"""Handles may be destroyed before or after the ctx they were created on (include/srlivo_b200.h, srl_ctx_destroy).  One handle of
every kind is made on a ctx and made to allocate or grow once; then they are destroyed after the ctx, and in a second run before
it.  Each run is a subprocess with MALLOC_PERTURB_ set, so that a destroy reading the freed ctx reads poisoned memory instead of
the stale values it held; the subprocess must exit 0, and a fresh ctx in this process must still run a pass."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SCENARIO = r'''
import ctypes as C
import sys

import numpy as np

import cloud_processing_ref as R
import flow_tracker_cases as FC
from sr_livo_b200 import capi, lio, synth

ctx_first = sys.argv[1] == "ctx_first"
L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=8192, initial_voxels=64)
ctx = L.ctx
made = []

# map growth past its 64 initial voxels, then a debug pass and a capped pass over the sweep (its lazy buffers)
assert L.addPointsToMap(synth.sample_map_points(80.0, 60.0, seed=3)) > 0
assert L.voxel_map.capacity()["committed_voxels"] > 64
sw = synth.make_sweep(4000, seed=1003, yaw=0.5)
L.setKeypoints(sw.raw_xyz)
L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=2 ** 31 - 1), sw.q_init, sw.t_init, sw.t_last, debug=True)
L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=500), sw.q_init, sw.t_init, sw.t_last)

# a colour map with points the flow tracker can start from
cm = lio.ColorVoxelMap(ctx, 0.5, 20, 1 << 15, 0.01, initial_voxels=16)
front, _, exact = FC.scene_points()
cm.addPoints(np.r_[front, exact], time_sweep_end=1.0)
ids, _, uv = cm.selectPointsForProjection(FC.device_camera(capi, FC.cam15(fov=-0.4)), minimum_dis=1.0, use_all_points=True)
ids, uv = ids[:200], uv[:200]
assert len(ids) > 0
made.append(cm)

comm = C.c_void_p()
assert capi.lib().srl_comm_create(ctx.h, 0, 1, C.byref(comm)) == capi.SRL_OK

# a frame built beyond its capacity (at least 1024 points)
n = 3000
rng = np.random.default_rng(7)
raw = rng.uniform(-20.0, 20.0, (n, 3))
ts = np.sort(rng.uniform(0.0, 0.1, n))
frame = lio.CloudFrame(ctx, 16)
L.buildFrame(raw, ts, [capi.ImuState()], 0.0, 0.1, 1, voxel_size=0.0, frame=frame)
assert len(frame) > 1024
made.append(frame)

ip = lio.ImageProcessing(ctx, **lio.ntu_camera_params())
cols, rows = ip.input_size
ip.process(rng.integers(0, 256, (rows, cols, 3), dtype=np.uint8))
made.append(ip)

gray = rng.integers(0, 256, (FC.ROWS, FC.COLS), dtype=np.uint8)
lk = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
lk.trackImage(gray, np.asarray(uv, np.float32).reshape(-1, 2))
made.append(lk)
lk2 = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
ft = lio.OpticalFlowTracker(ctx, cm, lk2, 300)
ft.init(gray, 1.0, ids, uv)
made += [ft, lk2]

cp = lio.CloudProcessing(ctx, **lio.r3live_lidar_params(), capacity=16)
assert cp.livoxHandler(R.livox_records(5, 2000), 1.7e9) > 16
made.append(cp)
ctx.synchronize()

handles = [L.sweep, L.voxel_map] + made
if ctx_first:
    ctx.close()
for h in handles:
    h.close()
capi.lib().srl_comm_destroy(comm)
if not ctx_first:
    ctx.close()
print("ok")
'''


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["ctx_first", "ctx_last"])
def test_handles_outlive_or_precede_their_ctx(order):
    env = dict(os.environ, MALLOC_PERTURB_="165", PYTHONPATH=os.pathsep.join([ROOT, HERE, os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", SCENARIO, order], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), (r.returncode, r.stdout[-2000:], r.stderr[-4000:])

    from sr_livo_b200 import lio, synth
    L = lio.LioOptimization(max_voxels=1 << 16, sweep_capacity=8192)
    try:
        L.addPointsToMap(synth.sample_map_points(80.0, 60.0, seed=3))
        sw = synth.make_sweep(4000, seed=1003, yaw=0.5)
        L.setKeypoints(sw.raw_xyz)
        g = L.buildPlaneResiduals(lio.r3live_params(max_num_residuals=2 ** 31 - 1), sw.q_init, sw.t_init, sw.t_last)
        assert g.success and g.num_residuals > 0 and np.isfinite(g.HTH).all()
    finally:
        L.close()
