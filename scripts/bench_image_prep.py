"""Per-image time of the camera image preparation on the device (srl_image_process, lio.ImageProcessing.process): undistortion,
grey conversion and both CLAHEs of imageProcessing::process (src/imageProcessing.cpp:120-125).  Prints one JSON line.

Workload: the textured images of tests/image_prep_cases.py at 1280x1024 (r3live's camera) and 752x480 (ntu), each processed
--frames times after --warmup calls, with the outputs on the device (what the renderer and the tracker take).
  * call time: host wall clock around process, which ends in a stream synchronise; median and p10-p90, from a pinned host
    image and from a device image
  * device split (CUDA events on the ctx stream): upload, remap + colour planes, both CLAHEs
  * cpu: the same per-image recipe through cv2 on one host thread, when cv2 is importable (it is not on every machine)
The device outputs are checked against the restatement (tests/image_prep_reference.py) once per camera.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_lk_track import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build()
    import image_prep_cases as IC
    import image_prep_reference as R
    from sr_livo_b200 import lio
    ctx = lio.Context(0)
    out = {"card": card(), "frames": args.frames, "cameras": {}}
    for name in ("r3live", "ntu"):
        case = IC.BY_NAME[name]
        bgr = case.bgr()
        ip = lio.ImageProcessing(ctx, **case.camera)
        oc, orows = ip.output_size()
        d_out = (torch.empty((orows, oc, 3), dtype=torch.uint8, device="cuda"), torch.empty((orows, oc), dtype=torch.uint8, device="cuda"))
        pinned = torch.from_numpy(bgr).pin_memory()
        device = pinned.cuda()
        rgb_w, gray_w = R.prepare(bgr, **case.camera)[:2]
        ip.process(device, out=d_out)
        assert np.array_equal(d_out[0].cpu().numpy(), rgb_w) and np.array_equal(d_out[1].cpu().numpy(), gray_w), name
        res = {"out": [oc, orows], "tiles": ip.tiles()}
        for src_name, src in (("pinned_host", pinned), ("device", device)):
            wall, split = [], []
            for k in range(args.warmup + args.frames):
                t0 = time.perf_counter()
                ip.process(src, out=d_out)
                t1 = time.perf_counter()
                if k >= args.warmup:
                    wall.append((t1 - t0) * 1e3)
                    split.append(ip.last_times())
            s = np.asarray(split)
            res[src_name] = {"call_ms": stats(wall), "upload_ms": stats(s[:, 0]), "remap_ms": stats(s[:, 1]), "clahe_ms": stats(s[:, 2])}
        try:
            import cv2
        except ImportError:
            res["cv2_one_thread_ms"] = "not measured: cv2 is not importable here"
        else:
            cv2.setNumThreads(1)
            s_, K, oc_, orows_, t = R.first_image(case.camera["image_width"], case.camera["image_height"], case.camera["camera_intrinsic"], case.cols)
            m1, m2 = cv2.initUndistortRectifyMap(K, np.array(case.camera["camera_dist_coeffs"]), None, K, (oc_, orows_), cv2.CV_16SC2)
            cpu = []
            for _ in range(20):   # process:120-125 per image; the map is built once, as the reference does
                t0 = time.perf_counter()
                und = cv2.remap(bgr, m1, m2, cv2.INTER_LINEAR)
                cv2.createCLAHE(3.0, (t, t)).apply(cv2.cvtColor(und, cv2.COLOR_RGB2GRAY))
                ch = list(cv2.split(cv2.cvtColor(und, cv2.COLOR_BGR2YCrCb)))
                ch[0] = cv2.createCLAHE(1.0, (t, t)).apply(ch[0])
                cv2.cvtColor(cv2.merge(ch), cv2.COLOR_YCrCb2BGR)
                cpu.append((time.perf_counter() - t0) * 1e3)
            res["cv2_one_thread_ms"] = stats(cpu)
        ip.close()
        out["cameras"][name] = res
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
