"""Per-sweep wall time of the capped ESIKF update (max_num_residuals = 600, the value every shipped parameter file sets) on
the device-resident loop against the host-driven loop, in the same process.  Prints one JSON line.

Workload: bench config 2's ~10.28M-point map, 100k-point Livox sweeps grid-sampled at 1.5 m (L.gridSampling), the
keypoints registered by LioOptimization.optimize with lio.r3live_params() (yaml values).  Cases:
  steady  frame_id 100, convergence thresholds 0: all 6 passes run
  init    frame_id 5 (nb = 2): all 16 passes run
  chunk2  the steady case between 13000 keypoints far from the map (in front) and 20000 more (behind): k* lies in chunk 2
          of 4, so every pass runs three chunks and the device loop enqueues a fourth, which leaves at once
  skip4   the steady case followed by 64000 keypoints far from the map: k* lies in chunk 0 of 5, so the device loop
          enqueues four chunks per pass that leave at once (the price of the skipped chunks' launches); the host-driven
          loop never launches them
Keypoints far from the map have no neighbourhood: they never count toward the cap and do not change the result.
Per case: warm-up, then device_loop 1 and 0 alternate sweep by sweep; a sweep's time runs from the optimize() call to
its result (the call ends in a synchronising wait).  Before anything is timed, the two loops' states must agree to 1e-9.
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

FAR = np.array([5000.0, 0.0, 0.0])


def chunk_bounds(n, cap):
    """The capped pass's chunk schedule (srl_api.cu cap_chunk_bounds): 4096 keypoints (or 2 cap), then doubling."""
    b, chunk = [0], max(4096, 2 * max(cap, 1))
    while b[-1] < n:
        b.append(min(n, b[-1] + chunk))
        chunk *= 2
    return b


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="timed sweeps per loop and case")
    ap.add_argument("--warmup", type=int, default=5, help="untimed sweeps per loop and case")
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--map-extent", type=float, default=600.0, help="side of the square world in m (600 -> ~10M points)")
    ap.add_argument("--sweeps", type=int, default=4)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_capped.py needs a CUDA device: the capped update has no CPU fallback")
    from sr_livo_b200 import lio, synth

    L = lio.LioOptimization(max_voxels=1 << 21, sweep_capacity=1 << 17)
    L.addPointsToMap(synth.sample_map_points(args.map_extent, 60.0, seed=1))
    n_vox, n_pts = L.voxel_map.stats()
    P = synth.prior_covariance()
    sweeps = []
    for i in range(args.sweeps):   # bench.py's sensor positions
        pos = (40.0 * ((i % 5) - 2), 3.0 + 40.0 * ((i // 5) % 3 - 1), 1.8)
        sw = synth.make_sweep(args.points, seed=1000 + i, yaw=0.5 + 0.37 * i, position=pos)
        kp = np.ascontiguousarray(sw.raw_xyz[L.gridSampling(sw.raw_xyz, 1.5)])
        sweeps.append((sw, kp))
    far = sweeps[0][0].raw_xyz + FAR
    steady = lio.r3live_params(threshold_translation_norm=0.0, threshold_orientation_norm=0.0)
    cases = {   # parameters, keypoints far from the map in front of / behind the sweep's keypoints
        "steady": (steady, None, None),
        "init": (lio.r3live_params(frame_id=5, threshold_translation_norm=0.0, threshold_orientation_norm=0.0), None, None),
        "chunk2": (steady, far[:13000], far[13000:33000]),
        "skip4": (steady, None, far[:64000]),
    }

    def run(i, prm, prefix, suffix, mode):
        sw, kp = sweeps[i % len(sweeps)]
        raw = np.ascontiguousarray(np.concatenate([a for a in (prefix, kp, suffix) if a is not None]))
        L.ctx.set_option("device_loop", mode)
        L.eskf_pro = lio.EskfEstimator(p=sw.t_init.copy(), q=sw.q_init.copy(), cov=P.copy())
        t0 = time.perf_counter()
        summ, fq, ft, _ = L.optimize(raw, prm, sw.t_last, want_world=False)
        dt = time.perf_counter() - t0
        return dt, summ, L.eskf_pro, L.ctx.counter("cap_chunks_run"), raw.shape[0]

    result = {"card": card(), "map_points": int(n_pts), "map_voxels": int(n_vox), "cases": {}}
    for name, (prm, prefix, suffix) in cases.items():
        # the two loops agree on every sweep before anything is timed
        info = {}
        for i in range(len(sweeps)):
            _, sd, ed, cd, n = run(i, prm, prefix, suffix, 1)
            _, sh, eh, ch, _ = run(i, prm, prefix, suffix, 0)
            assert (sd.success, sd.passes_run, sd.num_residuals_used) == (sh.success, sh.passes_run, sh.num_residuals_used), name
            assert cd == ch, (name, cd, ch)
            for f in ("p", "q", "v", "ba", "bg", "g"):
                assert np.allclose(getattr(ed, f), getattr(eh, f), rtol=1e-9, atol=1e-9), (name, f)
            n_chunks = len(chunk_bounds(n, prm.max_num_residuals)) - 1
            if name in ("chunk2", "skip4"):   # the case prices chunks that are enqueued and skipped: there must be some
                assert cd < sd.passes_run * n_chunks, (name, cd, sd.passes_run, n_chunks)
            info.setdefault("keypoints", []).append(n)
            info.setdefault("passes", []).append(sd.passes_run)
            info.setdefault("cap_chunks_run", []).append(cd)
            info.setdefault("chunks_enqueued_device_loop", []).append(sd.passes_run * n_chunks)
        for i in range(args.warmup):
            for mode in (1, 0):
                run(i, prm, prefix, suffix, mode)
        times = {1: [], 0: []}
        for i in range(args.steps):
            for mode in ((1, 0) if i % 2 == 0 else (0, 1)):
                times[mode].append(run(i, prm, prefix, suffix, mode)[0] * 1e3)
        stats = {}
        for mode, key in ((1, "device_loop"), (0, "host_loop")):
            t = np.array(times[mode])
            stats[key] = {"median_ms": round(float(np.median(t)), 4), "p10_ms": round(float(np.percentile(t, 10)), 4),
                          "p90_ms": round(float(np.percentile(t, 90)), 4), "n": int(t.size)}
        stats["speedup_median"] = round(stats["host_loop"]["median_ms"] / stats["device_loop"]["median_ms"], 3)
        result["cases"][name] = {**info, **stats}
    L.ctx.set_option("device_loop", 1)
    L.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
