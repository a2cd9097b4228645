"""Per-image time of the optical-flow tracker's pyramidal Lucas-Kanade on the device (srl_lk_track_image,
lio.LKOpticalFlowKernel.trackImage) against the reference's own trackImage on one host thread (oracle/_ref/libsrl_lk_ref.so).
Prints one JSON line.

Workload: 30-frame sequences of tests/lk_cases.py at 1280x1024 (r3live's camera) and 752x480 (ntu), with 300 points (the shipped
maximum_tracked_points) and with 20 000 points, at the shipped parameters (lio.tracker_lk_params()).  Every frame tracks the
previous frame's output points.  The image comes from host memory (numpy) or from device memory (a CUDA tensor).
  * call time: host wall clock around trackImage, which ends in a synchronising read of the tracked count; median and p10-p90
    over the frames after the warm-up
  * device split (CUDA events on the ctx stream): image upload + pyramid + derivatives, then the point tracking
  * reference: the same sequence through the compiled reference on one host thread.  Its pyrDown and copyMakeBorder are the
    OpenCV stand-in's scalar restatements (oracle/shim_lk/srl_lk_cv.h), not OpenCV's vectorised ones, so its pyramid time is
    not OpenCV's.
The device output is checked against the reference on the first and the last frame (points as float bits, status, count).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


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


def stats(v):
    v = np.asarray(v, np.float64)
    return {"median": round(float(np.median(v)), 4), "p10": round(float(np.percentile(v, 10)), 4), "p90": round(float(np.percentile(v, 90)), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=str, default="300,20000")
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()

    import torch
    import lk_cases as K
    import lk_ref as R
    from sr_livo_b200 import lio
    if not torch.cuda.is_available():
        raise SystemExit("bench_lk_track: no CUDA device (these numbers are GPU measurements)")
    use_ref = R.available() and not args.no_reference
    kw = lio.tracker_lk_params()
    ctx = lio.Context()
    result = {"bench": "lk_track", "frames": args.frames, "warmup": args.warmup, "params": kw, "gpu": card(), "cases": {}}
    for name, size in (("r3live", K.R3LIVE), ("ntu", K.NTU)):
        frames = K.frames(*size, 51, args.frames)
        d_frames = [torch.from_numpy(f).cuda() for f in frames]
        for n in [int(x) for x in args.points.split(",")]:
            pts = K.points(*size, 51, n)
            case = {}
            outs = {}
            for src in ("host", "device"):
                dev = lio.LKOpticalFlowKernel(ctx, **kw)
                last = pts if src == "host" else torch.from_numpy(pts).cuda()
                wall, pyr, trk, out = [], [], [], []
                for k in range(args.frames):
                    img = frames[k] if src == "host" else d_frames[k]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    c, s, m = dev.trackImage(img, last)
                    t1 = time.perf_counter()
                    if k >= max(args.warmup, 1):   # the first image only builds its pyramid
                        a, b = dev.lastTimes()
                        wall.append((t1 - t0) * 1e3)
                        pyr.append(a)
                        trk.append(b)
                    if k in (1, args.frames - 1):
                        out.append((np.asarray(c.cpu() if src == "device" else c).copy(), np.asarray(s.cpu() if src == "device" else s).copy(), m))
                    last = c
                dev.close()
                case[src] = {"call_ms": stats(wall), "pyramid_ms": stats(pyr), "track_ms": stats(trk)}
                outs[src] = out
            same_src = all(np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1]) and a[2] == b[2]
                           for a, b in zip(outs["host"], outs["device"]))
            case["host_equals_device_input"] = bool(same_src)
            if use_ref:
                ref = R.LKReference(**kw)
                last, ref_ms, ref_out = pts, [], []
                for k in range(args.frames):
                    t0 = time.perf_counter()
                    c, s, m = ref.track(frames[k], last)
                    t1 = time.perf_counter()
                    if k >= max(args.warmup, 1):
                        ref_ms.append((t1 - t0) * 1e3)
                    if k in (1, args.frames - 1):
                        ref_out.append((c.copy(), s.copy(), m))
                    last = c
                ref.close()
                case["reference_1thread_ms"] = stats(ref_ms)
                case["equals_reference_first_last"] = bool(all(np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
                                                              and a[2] == b[2] for a, b in zip(outs["host"], ref_out)))
            case["tracked_last_frame"] = int(outs["host"][-1][2])
            result["cases"][f"{name}_{n}"] = case
            print(f"{name} {size} n={n}: " + json.dumps(case), file=sys.stderr)
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
