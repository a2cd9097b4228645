"""Per-call device time of the two camera updates (srl_image_vio_esikf / srl_image_vio_photometric, CUDA events around the one
kernel) at n = 300 and 20 000 tracked points, from host and from device inputs, and the end-to-end call time; with the
reference's compiled vioEsikf / vioPhotometric (oracle/_ref/libsrl_vio_ref.so, over the stand-in Eigen: indicative only) on the
same inputs.  Prints one JSON line with the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import vio_cases as VC  # noqa: E402
import vio_ref as RF  # noqa: E402
from sr_livo_b200 import lio  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_vio needs a CUDA device")
    ctx = lio.Context(0)
    cam = VC.CAMERAS["ntu"]
    ip = lio.ImageProcessing(ctx, **cam)
    cols, rows = ip.output_size()
    res = {"card": card()}
    reps = 50
    for n in (300, 20000):
        c = VC.make_case(77, "ntu", n=int(n * 1.3))
        cm = lio.ColorVoxelMap(ctx, 1.0, 20, 1 << 16, 0.05)
        cm.addPoints(c["xyz"].astype(np.float64))
        st0 = lio.CameraState(c["state"][0:4], c["state"][4:7], c["state"][7:16].reshape(3, 3), c["state"][16:19], *c["state"][19:24])
        camera = st0.camera(cols, rows, 0.005)
        for k in range(3):
            cm.renderPointsInRecentVoxel(camera, c["img"], 1.0 + k)
        ids, _, uv = cm.selectPointsForProjection(camera, minimum_dis=1.0, use_all_points=True)
        ids, uv = np.ascontiguousarray(ids[:n]), np.ascontiguousarray(uv[:n])
        m = len(ids)
        g = cm.gatherPoints(ids)
        vel = np.random.default_rng(1).normal(scale=20.0, size=(m, 2))
        uvm = uv + np.float32(0.3)
        dev = dict(ids=torch.from_numpy(ids.view(np.int32)).cuda(), uv=torch.from_numpy(uvm).cuda(), vel=torch.from_numpy(vel).cuda(),
                   img=torch.from_numpy(c["img"]).cuda())
        host = dict(ids=ids, uv=uvm, vel=vel, img=c["img"])
        row = {"points": m}
        for kind, a in (("device", dev), ("host", host)):
            ke, kp, we, wp = [], [], [], []
            for r in range(reps + 5):
                ip.setCovariance(VC.initial_covariance())
                st = lio.CameraState(c["state"][0:4], c["state"][4:7], c["state"][7:16].reshape(3, 3), c["state"][16:19], *c["state"][19:24])
                t0 = time.perf_counter()
                ip.vioEsikf(cm, st, a["ids"], a["uv"], a["vel"], 40)
                t1 = time.perf_counter()
                ip.vioPhotometric(cm, st, a["ids"], a["vel"], 40, a["img"])
                t2 = time.perf_counter()
                e, p = ip.vio_last_times()
                if r >= 5:
                    ke.append(e); kp.append(p); we.append((t1 - t0) * 1e3); wp.append((t2 - t1) * 1e3)
            row[kind] = {"esikf_kernel_ms": float(np.median(ke)), "photometric_kernel_ms": float(np.median(kp)),
                         "esikf_call_ms": float(np.median(we)), "photometric_call_ms": float(np.median(wp))}
        if RF.available():
            te, tp = [], []
            for r in range(5):
                _, _, _, ns = RF.update(0, c["state"], VC.initial_covariance(), g["xyz"], uvm, vel, g["rgb"], g["cov"], g["n_rgb"], 40)
                te.append(ns / 1e6)
                if m <= 2000:
                    _, _, _, ns = RF.update(1, c["state"], VC.initial_covariance(), g["xyz"], uvm, vel, g["rgb"], g["cov"], g["n_rgb"], 40,
                                            c["img"])
                    tp.append(ns / 1e6)
            row["reference_cpu_ms"] = {"esikf": float(np.median(te)), "photometric": float(np.median(tp)) if tp else None}
        res[f"n{n}"] = row
        cm.close()
    ip.close()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
