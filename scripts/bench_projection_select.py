"""Per-call wall time of the map tracker's projection selection on the device (srl_color_map_select_for_projection) against the
oracle's single-threaded time on the same map and against the route a caller had before it: ColorVoxelMap.download() of the
whole colour map and a host selection over the downloaded arrays (the oracle's sequential rule restated in numpy).  Prints
one JSON line.

Workload, per cap (50 and 100, the shipped map_options): the bench_color_map.py stream, 35 registered 20k-point frames of the
synthetic street, each added (add_point_step 1, to_rendering on) and rendered into a 640x480 image.  After each rendering:
  * refresh: the recent voxels, 10 px cells, fov_margin -0.4 (refreshPointsForProjection after updatePoseForProjection)
  * first:   the recent voxels, 40 px cells (the first image's call, track_windows_size 40, image_scale_factor 1)
  * all:     use_all_points over the whole rgb list, 10 px cells
Once more on a 10M-point coloured map (the surface of bench_publish.py): use_all_points, 10 px cells.  Every call ends in a
synchronising wait, so its time is its host wall time.  The device is checked against the oracle on the first and the last
frame (and on the large map) before anything is timed.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_color_map import camera_at, card  # noqa: E402


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 4), "p10_ms": round(float(np.percentile(a, 10)), 4),
            "p90_ms": round(float(np.percentile(a, 90)), 4), "n": int(a.size)}


def with_fov(cam, cam15, fov):
    from sr_livo_b200 import capi
    c = capi.Camera()
    C = cam
    c.q_camera_world[:] = list(C.q_camera_world); c.t_camera_world[:] = list(C.t_camera_world); c.t_world_camera[:] = list(C.t_world_camera)
    c.fx, c.fy, c.cx, c.cy, c.fov_margin, c.cols, c.rows = C.fx, C.fy, C.cx, C.cy, fov, C.cols, C.rows
    c15 = np.array(cam15, np.float64)
    c15[14] = fov
    return c, c15


def old_route(cm, cam15, rows, cols, minimum_dis, use_all_points):
    """download() + the sequential selection on the host over the downloaded arrays (numpy projection, python cell walk)."""
    from sr_livo_b200 import synth
    d = cm.download()
    keys = d["keys"].astype(np.int64)
    packed = ((keys[:, 0] & 0xFFFF) << 32) | ((keys[:, 1] & 0xFFFF) << 16) | (keys[:, 2] & 0xFFFF)
    order = np.argsort(packed)
    if use_all_points or d["recent"].shape[0] == 0:
        lst = d["rgb_points"].astype(np.int64)
        lk = ((lst[:, 0] & 0xFFFF) << 32) | ((lst[:, 1] & 0xFFFF) << 16) | (lst[:, 2] & 0xFFFF)
        row = order[np.searchsorted(packed[order], lk)]
        idx = lst[:, 3]
    else:
        rec = d["recent"].astype(np.int64)
        rk = ((rec[:, 0] & 0xFFFF) << 32) | ((rec[:, 1] & 0xFFFF) << 16) | (rec[:, 2] & 0xFFFF)
        row = order[np.searchsorted(packed[order], rk)]
        idx = d["counts"][row] - 1
    p = d["xyz"][row, idx].astype(np.float64)
    R = synth.quat_to_rot(np.asarray(cam15[0:4]))
    t_cw, t_wc = np.asarray(cam15[4:7]), np.asarray(cam15[7:10])
    fx, fy, cx, cy, fov = cam15[10:15]
    dd = p - t_wc
    depth = np.sqrt(dd[:, 0] * dd[:, 0] + (dd[:, 1] * dd[:, 1] + dd[:, 2] * dd[:, 2]))
    pc = p @ R.T + t_cw
    with np.errstate(divide="ignore", invalid="ignore"):
        u = (pc[:, 0] * fx) / pc[:, 2] + cx
        v = (pc[:, 1] * fy) / pc[:, 2] + cy
    ok = (depth <= 200.0) & (depth >= 0.1) & (pc[:, 2] >= 0.001) & (u >= fov * cols + 1) & (np.ceil(u) < (1 - fov) * cols) & \
         (v >= fov * rows + 1) & (np.ceil(v) < (1 - fov) * rows)
    cu = np.trunc(np.sign(u[ok]) * np.floor(np.abs(u[ok] / minimum_dis) + 0.5) * minimum_dis).astype(np.int64)
    cv = np.trunc(np.sign(v[ok]) * np.floor(np.abs(v[ok] / minimum_dis) + 0.5) * minimum_dis).astype(np.int64)
    holder, stored = {}, {}
    for j, c, dpt in zip(np.nonzero(ok)[0].tolist(), zip(cu.tolist(), cv.tolist()), depth[ok].tolist()):
        if c not in stored or stored[c] > dpt:
            holder[c], stored[c] = j, float(np.float32(dpt))
    return len(holder)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=35)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--points", type=int, default=20000)
    ap.add_argument("--caps", type=str, default="50,100")
    ap.add_argument("--rgb-points", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--old-route-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from oracle import tracker_oracle as O
    from sr_livo_b200 import lio, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_projection_select: no CUDA device (these numbers are GPU measurements)")

    frames = []
    for f in range(args.frames):
        sw = synth.make_sweep(args.points, seed=7000 + f, position=(1.0 * f, 3.0, 1.8))
        frames.append((synth.registered_points(sw), sw.t_true.copy()))
    rng = np.random.default_rng(1)
    images = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8) for _ in range(args.frames)]
    calls = {"refresh": dict(minimum_dis=10.0, fov=-0.4, use_all_points=False), "first": dict(minimum_dis=40.0, fov=0.01, use_all_points=False),
             "all": dict(minimum_dis=10.0, fov=0.01, use_all_points=True)}

    ctx = lio.Context()
    result = {"bench": "projection_select", "points_per_frame": args.points, "frames": args.frames, "warmup": args.warmup,
              "image": [640, 480], "gpu": card(), "caps": {}}
    for cap in [int(c) for c in args.caps.split(",")]:
        cmg = lio.ColorVoxelMap(ctx, voxel_size=0.1, max_num_points_in_voxel=cap, max_voxels=1 << 20, min_distance_points=0.01, initial_voxels=4096)
        cmo = O.OracleColorMap(voxel_size=0.1, max_num_points_in_voxel=cap, min_distance_points=0.01)
        t = {f"{k}_{w}": [] for k in calls for w in ("gpu", "oracle_1thread")}
        t.update({f"{k}_old_route": [] for k in calls})
        sizes = {k: [] for k in calls}
        old_sizes = {k: [] for k in calls}   # (host selection, device) counts: numpy's projection is not the reference's arithmetic
        for f, (pts, pos) in enumerate(frames):
            kw = dict(add_point_step=1, time_sweep_end=1.0 + 0.1 * f, time_last_process=0.9 + 0.1 * f, to_rendering=True)
            cam, cam15 = camera_at(pos)
            obs = kw["time_sweep_end"] + 0.05
            cmg.addPoints(pts, **kw); cmo.add_points(pts, **kw)
            assert cmg.renderPointsInRecentVoxel(cam, images[f], obs) == cmo.render(cam15, images[f], obs)
            for name, c in calls.items():
                cc, c15 = with_fov(cam, cam15, c["fov"])
                sel = dict(minimum_dis=c["minimum_dis"], use_all_points=c["use_all_points"])
                if f == 0 or f == args.frames - 1:
                    ids, _, uv = cmg.selectPointsForProjection(cc, **sel)
                    ki, uvo = cmo.select(c15, 480, 640, **sel)
                    assert np.array_equal(cmg.gatherPoints(ids)["key_index"], ki) and np.array_equal(uv.view(np.uint32), uvo.view(np.uint32)), (cap, f, name)
                torch.cuda.synchronize()
                t0 = time.perf_counter(); ids, _, _ = cmg.selectPointsForProjection(cc, **sel); t1 = time.perf_counter()
                cmo.select(c15, 480, 640, **sel); t2 = time.perf_counter()
                if f >= args.warmup:
                    t[f"{name}_gpu"].append(1e3 * (t1 - t0)); t[f"{name}_oracle_1thread"].append(1e3 * (t2 - t1))
                    sizes[name].append(int(ids.shape[0]))
                if f >= args.frames - args.old_route_reps:
                    t3 = time.perf_counter(); n_old = old_route(cmg, c15, 480, 640, c["minimum_dis"], c["use_all_points"]); t4 = time.perf_counter()
                    t[f"{name}_old_route"].append(1e3 * (t4 - t3))
                    old_sizes[name].append((n_old, int(ids.shape[0])))
        st = cmg.stats()
        result["caps"][str(cap)] = {**{k: stats(v) for k, v in t.items()}, "selected_median": {k: int(np.median(v)) for k, v in sizes.items()},
                                    "old_route_vs_gpu_selected": old_sizes, "final_rgb_points": st["rgb_points"],
                                    "recent_last_frame": st["recent"]}
        cmg.close()
        del cmo

    # a 10M-point coloured map: the surface of bench_publish.py, camera 20 m above its centre looking down
    o = lio.r3live_map_options()
    side = int(np.ceil(np.sqrt(args.rgb_points)))
    cm = lio.ColorVoxelMap(ctx, o["size_voxel_map"], o["max_num_points_in_voxel"], 1 << 20, o["min_distance_points"], initial_voxels=4096)
    cmo = O.OracleColorMap(voxel_size=o["size_voxel_map"], max_num_points_in_voxel=o["max_num_points_in_voxel"], min_distance_points=o["min_distance_points"])
    g = (np.arange(side) * 0.02 + 0.005)
    for r0 in range(0, side, 512):
        gx, gy = np.meshgrid(g[r0:r0 + 512], g, indexing="ij")
        pts = np.stack([gx.ravel() - 32.0, gy.ravel() - 32.0, np.full(gx.size, 4.03)], axis=1)
        cm.addPoints(pts, o["add_point_step"], 1.0 + r0, float(r0), True)
        cmo.add_points(pts, o["add_point_step"], 1.0 + r0, float(r0), True)
    n = cm.stats()["rgb_points"]
    assert n >= args.rgb_points and n == cmo.num_rgb_points(), n
    from sr_livo_b200 import capi
    cam = capi.Camera()
    cam15 = np.concatenate([[0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 20.0], [0.0, 0.0, -20.0], [300.0, 300.0, 320.0, 240.0, -0.4]])
    cam.q_camera_world[:] = cam15[0:4].tolist(); cam.t_camera_world[:] = cam15[4:7].tolist(); cam.t_world_camera[:] = cam15[7:10].tolist()
    cam.fx, cam.fy, cam.cx, cam.cy, cam.fov_margin = cam15[10:15].tolist()
    cam.cols, cam.rows = 640, 480
    sel = dict(minimum_dis=10.0, use_all_points=True)
    ids, _, uv = cm.selectPointsForProjection(cam, **sel)
    t0 = time.perf_counter(); ki, uvo = cmo.select(cam15, 480, 640, **sel); t_oracle = 1e3 * (time.perf_counter() - t0)
    assert np.array_equal(cm.gatherPoints(ids)["key_index"], ki) and np.array_equal(uv.view(np.uint32), uvo.view(np.uint32))
    ids_dev = torch.empty(n, dtype=torch.int32, device="cuda"); uv_dev = torch.empty((n, 2), dtype=torch.float32, device="cuda")
    tg, td = [], []
    for r in range(args.reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter(); cm.selectPointsForProjection(cam, **sel); t1 = time.perf_counter()
        cm.selectPointsForProjection(cam, **sel, out=(ids_dev, None, uv_dev)); t2 = time.perf_counter()
        if r:
            tg.append(1e3 * (t1 - t0)); td.append(1e3 * (t2 - t1))
    t3 = time.perf_counter(); n_old = old_route(cm, cam15, 480, 640, 10.0, True); t_old = 1e3 * (time.perf_counter() - t3)
    result["large_map"] = {"rgb_points": n, "selected": int(ids.shape[0]), "old_route_selected": n_old, "all_gpu_host_out": stats(tg), "all_gpu_device_out": stats(td),
                           "all_oracle_1thread_ms": round(t_oracle, 2), "all_old_route_ms": round(t_old, 1)}
    cm.close(); ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
