"""Per-call wall time of the colour map at the shipped map_options (0.1 m voxels, 0.01 m fine cells; caps 20, 50 and 100 —
config/r3live.yaml uses 50, r3live_compressed.yaml 100) against the oracle's single-threaded time on the same inputs.
Prints one JSON line.

Workload: a stream of registered Livox frames from the synthetic street world (synth.make_sweep, the sensor driving along
+x, 1 m per frame), every frame fed to ColorVoxelMap.addPoints (add_point_step 1, to_rendering on) and then rendered
into a 640x480 BGR image by renderPointsInRecentVoxel from the sensor pose (camera looking along the boresight).  Both
calls end in a synchronising wait, so a call's time is its host wall time.  Before anything is timed the GPU map is
checked against the oracle on the first frame (stored count, stats and rendered count).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """Name and power limit of the GPU, read in the same run as the timings (read-only query)."""
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:   # the timings stand without it; say why it is missing
        out["power_limit_w"] = f"unavailable: {e!r}"
    return out


def camera_at(position, rows=480, cols=640):
    """camera at the sensor, looking along world +x (camera z = x, camera x = -y, camera y = -z)."""
    from sr_livo_b200 import capi
    pos = np.asarray(position, np.float64)
    R = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
    q = np.array([0.5, -0.5, 0.5, 0.5])                     # x, y, z, w of R
    t_cw = -R @ pos
    cam15 = np.concatenate([q, t_cw, pos, [300.0, 300.0, cols / 2.0, rows / 2.0, 0.01]])
    c = capi.Camera()
    c.q_camera_world[:] = q.tolist(); c.t_camera_world[:] = t_cw.tolist(); c.t_world_camera[:] = pos.tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = cam15[10:15].tolist()
    c.cols, c.rows = cols, rows
    return c, cam15


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed frames per cap")
    ap.add_argument("--warmup", type=int, default=5, help="untimed frames per cap")
    ap.add_argument("--points", type=int, default=20000, help="points per registered frame")
    ap.add_argument("--caps", type=str, default="20,50,100")
    ap.add_argument("--max-voxels", type=int, default=1 << 20)
    args = ap.parse_args()

    from oracle import oracle_py as O
    from sr_livo_b200 import lio, synth

    R_cam = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]])
    assert np.allclose(synth.quat_to_rot(np.array([0.5, -0.5, 0.5, 0.5])), R_cam)
    n_frames = args.warmup + args.steps
    frames = []
    for f in range(n_frames):
        sw = synth.make_sweep(args.points, seed=7000 + f, position=(1.0 * f, 3.0, 1.8))
        frames.append((synth.registered_points(sw), sw.t_true.copy()))
    rng = np.random.default_rng(1)
    images = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(n_frames)]

    ctx = lio.Context()
    result = {"bench": "color_map", "points_per_frame": args.points, "frames_timed": args.steps, "warmup": args.warmup,
              "size_voxel_map": 0.1, "min_distance_points": 0.01, "image": [640, 480], "gpu": card(), "caps": {}}
    for cap in [int(c) for c in args.caps.split(",")]:
        cmg = lio.ColorVoxelMap(ctx, voxel_size=0.1, max_num_points_in_voxel=cap, max_voxels=args.max_voxels, min_distance_points=0.01)
        cmo = O.OracleColorMap(voxel_size=0.1, max_num_points_in_voxel=cap, min_distance_points=0.01)
        add_g, add_o, ren_g, ren_o = [], [], [], []
        for f, (pts, pos) in enumerate(frames):
            kw = dict(add_point_step=1, time_sweep_end=1.0 + 0.1 * f, time_last_process=0.9 + 0.1 * f, to_rendering=True)
            cam, cam15 = camera_at(pos)
            obs = kw["time_sweep_end"] + 0.05
            t0 = time.perf_counter(); sg = cmg.addPoints(pts, **kw); t1 = time.perf_counter()
            so = cmo.add_points(pts, **kw); t2 = time.perf_counter()
            rg = cmg.renderPointsInRecentVoxel(cam, images[f], obs); t3 = time.perf_counter()
            ro = cmo.render(cam15, images[f], obs); t4 = time.perf_counter()
            if f == 0 or f == n_frames - 1:
                st, oc = cmg.stats(), cmo.counts()
                assert sg == so and rg == ro, (cap, f, sg, so, rg, ro)
                assert (st["voxels"], st["rgb_points"], st["recent"]) == (oc["voxels"], oc["rgb_points"], oc["recent"]), (cap, f)
            if f >= args.warmup:
                add_g.append((t1 - t0) * 1e3); add_o.append((t2 - t1) * 1e3); ren_g.append((t3 - t2) * 1e3); ren_o.append((t4 - t3) * 1e3)
        st = cmg.stats()
        result["caps"][str(cap)] = {"addPoints_gpu": stats(add_g), "addPoints_oracle_1thread": stats(add_o),
                                    "render_gpu": stats(ren_g), "render_oracle_1thread": stats(ren_o),
                                    "final_voxels": st["voxels"], "final_points": st["points"], "recent_last_frame": st["recent"]}
        cmg.close()
        del cmo
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
