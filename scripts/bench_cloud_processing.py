"""cloudProcessing on the device (row N10): decode + sort + filter + append of one message, and the cut, timed with CUDA events
after warm-up; the upload it needs against the raw_xyz + timestamp upload (32 bytes per queued point) it replaces; and, when
oracle/_ref/libsrl_cloud_processing_ref.so is built, the reference's own handler on the host.  Prints one JSON line.

    python scripts/bench_cloud_processing.py [--reps 20]
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
import cloud_processing_ref as R  # noqa: E402


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception:
        return "unknown"


def workload(name, params, kind, msg, stamp, reps):
    import torch
    from sr_livo_b200 import lio
    ctx = lio.Context(0)
    cp = lio.CloudProcessing(ctx, **params)
    raw = np.frombuffer(msg.tobytes(), np.uint8)
    h = torch.from_numpy(raw.copy()).pin_memory()

    def handle(i):
        s = stamp + i * 0.1
        return cp.livoxHandler(h, s, stride=msg.dtype.itemsize) if kind == "livox" else \
            cp.process(h, R.cloud_layout(params["lidar_type"]), s)
    for i in range(3):
        handle(i)
        cp.cut(np.inf)
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    dec, cut, appended = [], [], 0
    for i in range(reps):
        e0.record()
        appended = handle(10 + i)
        e1.record()
        cp.cut(np.inf)
        e2.record()
        torch.cuda.synchronize()
        dec.append(e0.elapsed_time(e1))
        cut.append(e1.elapsed_time(e2))
    cp.close()
    out = dict(points_in=len(msg), points_appended=appended, decode_append_ms_median=float(np.median(dec)),
               cut_ms_median=float(np.median(cut)), upload_bytes=int(raw.nbytes), replaced_upload_bytes=32 * int(appended))
    if R.have_reference():
        lt, ns, rate, tu, blind, f = (params[k] for k in ("lidar_type", "n_scans", "scan_rate", "time_unit", "blind", "point_filter_num"))
        ref = R.ReferenceCP(lt, ns, rate, tu, blind, f)
        ts = []
        for i in range(max(3, reps // 4)):
            t0 = time.perf_counter()
            ref.livox(msg, stamp + i) if kind == "livox" else ref.process(msg, stamp + i)
            ts.append((time.perf_counter() - t0) * 1e3)
            ref.drain()
        ref.close()
        out["reference_host_ms_median"] = float(np.median(ts))
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    from sr_livo_b200 import lio
    res = {"gpu": gpu_name()}
    # a Livox Avia-size message (24k records, 10 Hz) at r3live's parameters; an Ouster-128 cloud (128 x 1024) at ntu's
    res.update([workload("livox_r3live", lio.r3live_lidar_params(), "livox", R.livox_records(1, 24000), 1.7e9, a.reps),
                workload("ouster128_ntu", lio.ntu_lidar_params(n_scans=128), "cloud", R.cloud2(R.OUST, 1, 128, 1024, scan_rate=20),
                         1.7e9, a.reps)])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
