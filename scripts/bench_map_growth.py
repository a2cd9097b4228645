"""Cost of growing the maps on demand, against twins committed at their limit up front.  Prints one JSON line.

  * LIO stream (config 4 shape: each sweep registered with 3 ESIKF passes, then inserted): the sensor drives along the
    synthetic street, 4 m per 100k-point Livox sweep, so the map keeps growing.  A growable map (initial_voxels 4096) and
    a fixed one (2^21 voxels) take the same sweeps, alternated sweep by sweep (the order flips every sweep).  Per-sweep
    time is CUDA-event time of register + insert; every sweep whose insert grew the map is listed with its insert time,
    the fixed twin's insert time on the same sweep and the slot count after growing.
  * Colour map at r3live_compressed's map_options (0.1 m voxels, 100 points, 0.01 m fine cells): the stream of registered
    street frames of scripts/bench_color_map.py, growable from 4096 voxels vs fixed at 2^20 voxels, alternated frame by
    frame: committed bytes at the end and addPoints wall time (the call ends in a synchronising wait).
Both twins must agree after every step (poses bit for bit, map stats), or the script stops.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def stats(ms):
    a = np.asarray(ms)
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90)), "n": int(a.size)}


def lio_stream(args, torch, lio, synth):
    prm = lio.r3live_params(max_num_residuals=2 ** 31 - 1)
    P = synth.prior_covariance()
    sweeps = [synth.make_sweep(args.points, seed=9000 + i, position=(4.0 * i, 3.0, 1.8)) for i in range(args.sweeps)]
    stream = torch.cuda.current_stream().cuda_stream or 1        # the events below are recorded on the maps' stream
    G = lio.LioOptimization(stream=stream, max_voxels=1 << 21, initial_voxels=4096, sweep_capacity=args.points)
    F = lio.LioOptimization(stream=stream, max_voxels=1 << 21, sweep_capacity=args.points)
    first = synth.registered_points(sweeps[0])
    assert G.addPointsToMap(first) == F.addPointsToMap(first)
    times = {"growable": [], "fixed": []}
    events = []
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for i, sw in enumerate(sweeps[1:]):
        order = [("growable", G), ("fixed", F)] if i % 2 == 0 else [("fixed", F), ("growable", G)]
        res, ins = {}, {}
        for name, L in order:
            before = L.voxel_map.capacity()
            e0, e1, e2 = ev(), ev(), ev()
            e0.record()
            L.setKeypoints(sw.raw_xyz)
            L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=P.copy())
            summ, fq, ft = L.updateIEKF(prm, sw.t_last)
            e1.record()
            L.addSweepToMap(fq, ft)
            e2.record()
            torch.cuda.synchronize()
            res[name] = (fq.tobytes(), ft.tobytes(), L.voxel_map.stats())
            ins[name] = e1.elapsed_time(e2)
            if i >= args.warmup:
                times[name].append(e0.elapsed_time(e2))
            after = L.voxel_map.capacity()
            if name == "growable" and after["committed_voxels"] != before["committed_voxels"]:
                events.append({"sweep": i + 1, "committed_voxels": [before["committed_voxels"], after["committed_voxels"]],
                               "slot_capacity": after["slot_capacity"], "voxels": res[name][2][0]})
        assert res["growable"] == res["fixed"], f"sweep {i + 1}: growable and fixed maps differ"
        for e in events:
            if e["sweep"] == i + 1:
                e["insert_ms_growable"], e["insert_ms_fixed"] = ins["growable"], ins["fixed"]
    out = {"workload": f"{args.sweeps} sweeps x ({args.points} keypoints, 3 passes + insert), 4 m apart; first sweep seeds the map",
           "growable_initial_voxels": 4096, "fixed_voxels": 1 << 21, "sweep_ms_growable": stats(times["growable"]),
           "sweep_ms_fixed": stats(times["fixed"]), "growth_events": events, "final_voxels": G.voxel_map.stats()[0],
           "committed_bytes_growable": G.voxel_map.capacity()["committed_bytes"], "committed_bytes_fixed": F.voxel_map.capacity()["committed_bytes"]}
    G.close(); F.close()
    return out


def color_stream(args, lio, synth):
    import time
    from bench_color_map import camera_at
    frames = []
    for f in range(args.frames):
        sw = synth.make_sweep(20000, seed=7000 + f, position=(1.0 * f, 3.0, 1.8))
        frames.append((synth.registered_points(sw), sw.t_true.copy()))
    rng = np.random.default_rng(1)
    ctx = lio.Context()
    G = lio.ColorVoxelMap(ctx, 0.1, 100, 1 << 20, 0.01, initial_voxels=4096)
    F = lio.ColorVoxelMap(ctx, 0.1, 100, 1 << 20, 0.01)
    add = {"growable": [], "fixed": []}
    for f, (pts, pos) in enumerate(frames):
        kw = dict(add_point_step=1, time_sweep_end=1.0 + 0.1 * f, time_last_process=0.9 + 0.1 * f, to_rendering=True)
        cam, _ = camera_at(pos)
        img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
        order = [("growable", G), ("fixed", F)] if f % 2 == 0 else [("fixed", F), ("growable", G)]
        got = {}
        for name, cm in order:
            t0 = time.perf_counter(); s = cm.addPoints(pts, **kw); t1 = time.perf_counter()
            r = cm.renderPointsInRecentVoxel(cam, img, kw["time_sweep_end"] + 0.05)
            got[name] = (s, r, cm.stats())
            if f >= args.warmup:
                add[name].append((t1 - t0) * 1e3)
        assert got["growable"] == got["fixed"], f"frame {f}: growable and fixed colour maps differ"
    st = G.stats()
    out = {"workload": f"{args.frames} registered street frames x 20000 points, cap 100, rendering after each",
           "final": {k: st[k] for k in ("voxels", "points", "rgb_points")},
           "growable": dict(G.capacity(), addPoints=stats(add["growable"])), "fixed_2p20": dict(F.capacity(), addPoints=stats(add["fixed"]))}
    G.close(); F.close(); ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=40)
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--frames", type=int, default=35)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from bench_color_map import card
    from sr_livo_b200 import lio, synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_map_growth.py needs a CUDA device")
    result = {"bench": "map_growth", "gpu": card(), "lio": lio_stream(args, torch, lio, synth), "color_map": color_stream(args, lio, synth)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
