"""Cost of publishing the maps from the device.  Prints one JSON line (and writes it to --out when given).

  * Registered cloud: srl_map_insert_published against srl_map_insert on 100k-point Livox sweeps (the bench's sweep size),
    registered into a map pre-filled with the synthetic street (80 m).  Two twins take the same sweeps, one with the plain
    insert and one with the published insert, and the order flips every sweep.  Host input / pageable host output, and device
    input / device output (torch tensors).  Wall time around each call, which ends in a synchronising wait.  Both twins must
    hold the same map at the end.
  * Coloured map: a colour map at r3live_map_options (0.1 m voxels, 50 points, 0.01 m fine cells) holding >= 10^7 rgb points
    (a 63 m x 63 m surface sampled every 0.02 m), exported with min_views = 0 (every rgb point kept: the output-heavy case) in
    both orders, to a device buffer, to page-locked host memory and to pageable numpy arrays, against the route a caller had
    before: srl_map_download + srl_color_map_download_state + srl_color_map_download_lists (ColorVoxelMap.download) and a
    numpy join of the list with the blocks.  The outputs of both routes must be equal.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": round(float(np.median(a)), 3), "p10_ms": round(float(np.percentile(a, 10)), 3),
            "p90_ms": round(float(np.percentile(a, 90)), 3), "n": int(a.size)}


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, 1e3 * (time.perf_counter() - t0)


def registered_cloud(args, torch, lio, synth):
    pts = synth.sample_map_points(80.0, 60.0, seed=1)
    A = lio.LioOptimization(max_voxels=1 << 21, sweep_capacity=args.points)
    B = lio.LioOptimization(max_voxels=1 << 21, sweep_capacity=args.points)
    A.addPointsToMap(pts); B.addPointsToMap(pts)
    sweeps = [synth.registered_points(synth.make_sweep(args.points, seed=7000 + i, yaw=0.3 * i, position=(0.5 * i - 10.0, 3.0, 1.8)))
              for i in range(args.sweeps)]
    t = {"plain_host": [], "published_host": [], "plain_device": [], "published_device": []}
    n_pub, out_h = [], np.empty((args.points, 4), np.float32)
    out_d = torch.empty((args.points, 4), dtype=torch.float32, device="cuda")
    for i, w in enumerate(sweeps):
        tz = 1.8 + 0.01 * i
        device = i % 2 == 1                              # alternate host and device transfers sweep by sweep
        src = torch.from_numpy(w).cuda() if device else w
        torch.cuda.synchronize()
        plain = (lambda: A.voxel_map.insert_device(src.data_ptr(), w.shape[0])) if device else (lambda: A.addPointsToMap(w))
        pub = lambda: B.addPointsToMapPublished(src, tz, out=out_d if device else out_h)
        order = [("plain", plain), ("published", pub)] if (i // 2) % 2 == 0 else [("published", pub), ("plain", plain)]
        res = {}
        for name, fn in order:
            res[name], ms = timed(fn)
            if i >= args.warmup:
                t[f"{name}_{'device' if device else 'host'}"].append(ms)
        assert res["plain"] == res["published"][0]
        n_pub.append(int(res["published"][1].shape[0]))
    ka, ca, xa = A.voxel_map.download()
    kb, cb, xb = B.voxel_map.download()
    assert np.array_equal(ka, kb) and np.array_equal(ca, cb) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))
    A.close(); B.close()
    return {"points_per_sweep": args.points, "sweeps": args.sweeps, "warmup": args.warmup, "published_per_sweep_median": int(np.median(n_pub)),
            **{k: stats(v) for k, v in t.items()}}


def color_map(args, torch, lio):
    o = lio.r3live_map_options()
    side = int(np.ceil(np.sqrt(args.rgb_points)))
    ctx = lio.Context()
    cm = lio.ColorVoxelMap(ctx, o["size_voxel_map"], o["max_num_points_in_voxel"], 1 << 20, o["min_distance_points"], initial_voxels=4096)
    g = (np.arange(side) * 0.02 + 0.005)
    for r0 in range(0, side, 512):                      # sweeps of 512 rows
        gx, gy = np.meshgrid(g[r0:r0 + 512], g, indexing="ij")
        pts = np.stack([gx.ravel() - 32.0, gy.ravel() - 32.0, np.full(gx.size, 4.03)], axis=1)
        cm.addPoints(pts, o["add_point_step"], 1.0 + r0, float(r0), True)
    n = cm.stats()["rgb_points"]
    assert n >= args.rgb_points, n
    res = {"rgb_points": n, "committed_bytes": cm.capacity()["committed_bytes"]}
    dx = torch.empty((n, 3), dtype=torch.float32, device="cuda"); dr = torch.empty((n, 3), dtype=torch.uint8, device="cuda")
    px = torch.empty((n, 3), dtype=torch.float32).pin_memory(); pr = torch.empty((n, 3), dtype=torch.uint8).pin_memory()
    hx = np.empty((n, 3), np.float32); hr = np.empty((n, 3), np.uint8)

    def old_route():
        d = cm.download()
        keys = d["keys"].astype(np.int64)
        packed = ((keys[:, 0] & 0xFFFF) << 32) | ((keys[:, 1] & 0xFFFF) << 16) | (keys[:, 2] & 0xFFFF)
        order = np.argsort(packed)
        lst = d["rgb_points"].astype(np.int64)
        lk = ((lst[:, 0] & 0xFFFF) << 32) | ((lst[:, 1] & 0xFFFF) << 16) | (lst[:, 2] & 0xFFFF)
        row = order[np.searchsorted(packed[order], lk)]
        idx = lst[:, 3]
        keep = d["n_rgb"][row, idx] >= 0
        return d["xyz"][row, idx][keep], d["rgb"][row, idx][keep][:, ::-1].astype(np.uint8)

    want, _ = timed(old_route)
    got = cm.exportColorPoints(0, 0, hx, hr)
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and np.array_equal(got[1], want[1])
    t = {"old_route": [], "device_publish": [], "device_save": [], "pinned_publish": [], "pageable_publish": [], "count_only": []}
    runs = {"device_publish": lambda: cm.exportColorPoints(0, 0, dx, dr), "device_save": lambda: cm.exportColorPoints(0, 1, dx, dr),
            "pinned_publish": lambda: cm.exportColorPoints(0, 0, px, pr), "pageable_publish": lambda: cm.exportColorPoints(0, 0, hx, hr),
            "count_only": lambda: cm.countColorPoints(0, 0)}
    for r in range(args.reps + 1):                      # the first round warms up every shape
        for name, fn in (list(runs.items()) if r % 2 == 0 else list(runs.items())[::-1]):
            torch.cuda.synchronize()
            _, ms = timed(fn)
            if r:
                t[name].append(ms)
        if r and r <= 3:
            _, ms = timed(old_route)
            t["old_route"].append(ms)
    res["old_route_bytes_d2h"] = int(cm.stats()["voxels"] * o["max_num_points_in_voxel"] * (12 + 6 + 2 + 12 + 8 + 8) + n * 8)
    res["export_bytes_out"] = int(n * 15)
    res.update({k: stats(v) for k, v in t.items()})
    cm.close(); ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--sweeps", type=int, default=24)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rgb-points", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from sr_livo_b200 import lio, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_publish: no CUDA device (these numbers are GPU measurements)")
    res = {"gpu": torch.cuda.get_device_name(0)}
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        res["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except OSError:
        pass
    res["registered_cloud"] = registered_cloud(args, torch, lio, synth)
    res["color_map_export"] = color_map(args, torch, lio)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
