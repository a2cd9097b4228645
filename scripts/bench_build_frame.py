"""Time buildFrame (src/lioOptimization.cpp:786-893) on a bench-sized Livox sweep at r3live's parameters (config/r3live.yaml:
voxel_size 0.1, init_num_frames 20, CONSTANT_VELOCITY, point time given), by stage:

- srl_build_frame on the GPU (device shuffles), from host buffers and from device-resident buffers;
- the same with option "shuffle_on_host" (the shuffles as a host Fisher-Yates + upload);
- the compiled reference's own buildFrame on the host (oracle/_ref/libsrl_build_frame_ref.so), when it is built.

Usage: python scripts/bench_build_frame.py [--points 100000] [--reps 20] [--out results/bench_build_frame.json]
Prints one JSON line.  Stage times are host-clock intervals between the stage boundaries, each ending in a stream synchronise.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

STAGES = ("timestamps", "undistortion", "shuffle1", "subsample", "shuffle2", "transforms")


def sweep(n, seed=7):
    from sr_livo_b200 import synth
    import build_frame_model as M
    sw = synth.make_sweep(n, seed=seed)
    c = M.make_case("bench", n=0, seed=seed, index_frame=25, voxel_size=0.1, init_voxel_size=0.2, edges=False)
    rng = np.random.default_rng(seed)
    c["raw"] = np.ascontiguousarray(sw.raw_xyz, float)
    c["ts"] = np.sort(c["begin"] + rng.uniform(0.0, c["offset"], c["raw"].shape[0]))
    return c


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from sr_livo_b200 import capi, lio
    import build_frame_model as M
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    c = sweep(a.points)
    n = c["raw"].shape[0]
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=1024)
    L.R_imu_lidar, L.t_imu_lidar = c["R_il"], c["t_il"]
    frame = lio.CloudFrame(L.ctx, n)
    states = M.capi_imu_states(c["states"])
    args = (c["raw"], c["ts"], states, c["begin"], c["offset"], c["index_frame"], c["q_pred"], c["t_pred"], True, 1, 20, 0.2, 0.1,
            c["prev_time_sweep_end"])
    d_raw = torch.from_numpy(c["raw"]).cuda()
    d_ts = torch.from_numpy(c["ts"]).cuda()

    def run_device_input():
        p = capi.BuildFrameParams()
        p.timestamp_begin, p.timestamp_offset, p.point_time_enable, p.motion_compensation = c["begin"], c["offset"], 1, 1
        p.index_frame, p.init_num_frames, p.init_voxel_size, p.voxel_size = c["index_frame"], 20, 0.2, 0.1
        p.R_il[:] = list(np.ravel(c["R_il"])); p.t_il[:] = list(c["t_il"]); p.q_pred[:] = list(c["q_pred"]); p.t_pred[:] = list(c["t_pred"])
        info = capi.BuildFrameInfo()
        arr = (capi.ImuState * len(states))(*states)
        rc = capi.lib().srl_build_frame(L.ctx.h, d_raw.data_ptr(), d_ts.data_ptr(), n, arr, len(states), p, frame.h, info)
        assert rc == capi.SRL_OK
        return info

    def timed(fn, reps):
        fn()
        fn()   # warm-up: module load, first allocations
        tot, st = [], np.zeros(6)
        for _ in range(reps):
            t0 = time.perf_counter()
            info = fn()
            tot.append((time.perf_counter() - t0) * 1e3)
            st += np.array(list(info.stage_ms))
        return dict(ms_median=float(np.median(tot)), ms_min=float(np.min(tot)),
                    stage_ms_mean={k: round(float(v) / reps, 4) for k, v in zip(STAGES, st)}, points_out=int(info.n_points),
                    rejections=int(info.shuffle_rejections), engine_words=int(info.engine_words))

    res = dict(points_in=n, gpu=gpu_info(), reps=a.reps)
    res["device_shuffle_host_input"] = timed(lambda: L.buildFrame(*args, frame=frame).info, a.reps)
    res["device_shuffle_device_input"] = timed(run_device_input, a.reps)
    L.ctx.set_option("shuffle_on_host", 1)
    res["host_shuffle_host_input"] = timed(lambda: L.buildFrame(*args, frame=frame).info, a.reps)
    L.ctx.set_option("shuffle_on_host", 0)
    # the two shuffle forms give the same frame
    g0 = L.buildFrame(*args, frame=frame).download()["source_index"]
    L.ctx.set_option("shuffle_on_host", 1)
    g1 = L.buildFrame(*args, frame=frame).download()["source_index"]
    L.ctx.set_option("shuffle_on_host", 0)
    res["host_and_device_shuffle_agree"] = bool(np.array_equal(g0, g1))
    if M.reference_available():
        R = M.ReferenceBuildFrame()
        t = []
        for k in range(max(3, a.reps // 4) + 1):
            t0 = time.perf_counter()
            ref = R.build_frame(c)
            if k:
                t.append((time.perf_counter() - t0) * 1e3)
        res["reference_host"] = dict(ms_median=float(np.median(t)), ms_min=float(np.min(t)), points_out=int(len(ref["source_index"])),
                                     note="one host thread, includes the harness copying the sweep in and the frame out")
        res["reference_source_index_equal"] = bool(np.array_equal(ref["source_index"], g0))
    else:
        res["reference_host"] = "not built"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    frame.close()
    L.close()


if __name__ == "__main__":
    main()
