"""Per-step and per-image time of the optical-flow tracker's bookkeeping on the device (srl_flow_tracker_*, row N9,
lio.OpticalFlowTracker).  Prints one JSON line.

Workload, per camera (ntu 752 x 480 and r3live 1280 x 1024, images from tests/lk_cases.py): a colour map of 60 000 points in
front of the camera, 300 tracked points (the shipped maximum_tracked_points) seeded by the first image's selection, and every
image: trackImage -> rejectMatches (every third match rejected) -> removeOutlierUsingRansacPnp (every other current point) ->
refresh selection (minimum_dis 10, fov_margin -0.4: the full-size candidate list, about 10^4 ids, on the device) ->
updateAndAppendTrackPoints (mini_distance 40).  The camera drifts a little between images, so points are erased and appended.
  * per-step device time: CUDA events recorded on the tracker's stream (the context runs on torch's current stream) around
    each call.  trackImage includes the Lucas-Kanade call (pyramid and tracking, timed by row N6's bench).  Per image: the sum
    of the four steps (the selection is row N4's and is not included).  The host wall clock of each call (which ends in its
    count read-back) is reported beside it.
  * reference: the same calls on the same inputs through the reference's own compiled opticalFlowTracker
    (oracle/_ref/libsrl_flow_tracker_ref.so, one host thread), its Lucas-Kanade results taken from a second device tracker on
    the same images (the time inside that stand-in is subtracted).  Its sets are checked against the device's after every image.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import ctypes as C

    import torch
    import flow_tracker_ref as RF
    import lk_cases as K
    from bench_lk_track import card, stats
    from sr_livo_b200 import capi, lio
    if not torch.cuda.is_available():
        raise SystemExit("bench_flow_tracker: no CUDA device (these numbers are GPU measurements)")
    ctx = lio.Context(0, stream=torch.cuda.current_stream().cuda_stream)
    use_ref = RF.available()
    result = {"bench": "flow_tracker", "images": args.images, "warmup": args.warmup, "gpu": card(), "cases": {}}
    rng = np.random.default_rng(7)
    for name, (cols, rows) in (("ntu", K.NTU), ("r3live", K.R3LIVE)):
        fx = fy = 0.6 * cols
        cx, cy = cols / 2.0, rows / 2.0
        n = 60000
        z = rng.uniform(3.0, 30.0, n)
        u = rng.uniform(-0.6 * cols, 1.6 * cols, n)
        v = rng.uniform(-0.6 * rows, 1.6 * rows, n)
        xyz = np.stack([(u - cx) * z / fx, (v - cy) * z / fy, z], 1)

        def camera(tx, fov):
            return capi.Camera((C.c_double * 4)(0, 0, 0, 1), (C.c_double * 3)(tx, 0, 0), (C.c_double * 3)(-tx, 0, 0), fx, fy, cx, cy, fov,
                               cols, rows)

        cm = lio.ColorVoxelMap(ctx, 0.5, 20, 1 << 18, 0.05)
        cm.addPoints(torch.from_numpy(xyz).cuda(), time_sweep_end=1.0)
        frames = [torch.from_numpy(f).cuda() for f in K.frames(cols, rows, 61, args.images + 1)]
        lk = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
        t = lio.OpticalFlowTracker(ctx, cm, lk, 300)
        k0 = cm.countPointsForProjection(camera(0.0, 0.005), minimum_dis=40.0, use_all_points=True)
        ids0 = torch.empty(k0, dtype=torch.int32, device="cuda")
        uv0 = torch.empty((k0, 2), dtype=torch.float32, device="cuda")
        cm.selectPointsForProjection(camera(0.0, 0.005), minimum_dis=40.0, use_all_points=True, out=(ids0, None, uv0))
        t.init(frames[0], 1.0, ids0[:300].contiguous(), uv0[:300].contiguous())
        names = ["trackImage", "rejectMatches", "removeOutlierUsingRansacPnp", "updateAndAppendTrackPoints"]
        steps = {key: [] for key in names + ["image"]}
        wall = {key: [] for key in names}
        ref_steps = {key: [] for key in names + ["image"]}
        ref_same = True
        n_cand, n_last = [], []
        masks = {}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
        if use_ref:
            ref = RF.FlowTrackerReference(cm.download()["xyz"].reshape(-1, 3), 300)
            lk2 = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
            inside = [0.0]

            def lk_on(gray):
                def f(p):
                    t0 = time.perf_counter()
                    c, st, _ = lk2.trackImage(gray, np.ascontiguousarray(p, np.float32))
                    inside[0] += time.perf_counter() - t0
                    return c, st
                return f
            ref.init(1.0, ids0[:300].cpu().numpy().view(np.uint32), uv0[:300].cpu().numpy(), lk_on(frames[0]))
        for k in range(1, args.images + 1):
            tx = 0.01 * k
            cam_k = camera(tx, 0.005)
            kc = cm.countPointsForProjection(camera(tx, -0.4), minimum_dis=10.0, use_all_points=True)
            cand = torch.empty(kc, dtype=torch.int32, device="cuda")
            cm.selectPointsForProjection(camera(tx, -0.4), minimum_dis=10.0, use_all_points=True, out=(cand, None, None))
            torch.cuda.synchronize()
            w = []
            ev[0].record()
            t0 = time.perf_counter()
            t.trackImage(frames[k], 1.0 + 0.1 * k)
            w.append(time.perf_counter() - t0)
            ev[1].record()
            nm = t.counts()["match"]
            if nm not in masks:
                masks[nm] = torch.from_numpy((np.arange(nm) % 3 != 0).astype(np.uint8)).cuda()
            ev[2].record()
            t0 = time.perf_counter()
            t.rejectMatches(masks[nm])
            w.append(time.perf_counter() - t0)
            ev[3].record()
            nc = t.counts()["cur"]
            inl = torch.arange(0, nc, 2, dtype=torch.int32, device="cuda")
            ev[4].record()
            t0 = time.perf_counter()
            t.removeOutlierUsingRansacPnp(inl)
            w.append(time.perf_counter() - t0)
            ev[5].record()
            ev[6].record()
            t0 = time.perf_counter()
            t.updateAndAppendTrackPoints(cam_k, cand, 40.0)
            w.append(time.perf_counter() - t0)
            ev[7].record()
            torch.cuda.synchronize()
            dev = [ev[2 * j].elapsed_time(ev[2 * j + 1]) for j in range(4)]
            if use_ref:
                r_ns = []
                inside[0] = 0.0
                ref.track_image(1.0 + 0.1 * k, lk_on(frames[k]), cols, rows, lambda n: (np.arange(n) % 3 != 0).astype(np.uint8))
                r_ns.append(ref.ns * 1e-6 - inside[0] * 1e3)
                ref.remove_outliers(np.arange(0, len(ref.cur_arrays()[0]), 2, dtype=np.int32))
                r_ns.append(ref.ns * 1e-6)
                c15 = np.array([0, 0, 0, 1, tx, 0, 0, -tx, 0, 0, fx, fy, cx, cy, 0.005], np.float64)
                ref.update_and_append(c15, cols, rows, cand.cpu().numpy().view(np.uint32), 40.0)
                r_ns.append(ref.ns * 1e-6)
                a, b = t.last(), ref.last_arrays()
                ref_same &= all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))
            if k > args.warmup:
                for key, x, d in zip(names, w, dev):
                    wall[key].append(x * 1e3)
                    steps[key].append(d)
                steps["image"].append(sum(dev))
                if use_ref:
                    # the reference has no rejectMatches: its mask is applied inside trackImage
                    for key, x in zip(("trackImage", "removeOutlierUsingRansacPnp", "updateAndAppendTrackPoints"), r_ns):
                        ref_steps[key].append(x)
                    ref_steps["image"].append(sum(r_ns))
                n_cand.append(kc)
                n_last.append(t.counts()["last"])
        case = {"device_ms": {key: stats(v) for key, v in steps.items()}, "call_wall_ms": {key: stats(v) for key, v in wall.items()}}
        if use_ref:
            case["reference_1thread_ms"] = {key: stats(v) for key, v in ref_steps.items() if v}
            case["reference_equals_device_last"] = bool(ref_same)
            ref.close(); lk2.close()
        case["candidates_median"] = int(np.median(n_cand))
        case["tracked_median"] = int(np.median(n_last))
        result["cases"][name] = case
        print(f"{name}: " + json.dumps(case), file=sys.stderr)
        t.close(); lk.close(); cm.close()
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
