"""The pyramidal Lucas-Kanade on the GPU (srl_lk_*, lio.LKOpticalFlowKernel) bit for bit against the reference's own
LKOpticalFlowKernel::trackImage: against tests/golden/lk_track.npz always, and against oracle/_ref/libsrl_lk_ref.so when it
was built.  Points are compared as float bits, status and the return value exactly, pyramid levels byte for byte."""
import os

import numpy as np
import pytest

import lk_cases as K
import lk_ref as R
from sr_livo_b200 import capi, lio

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lk_track.npz")
needs_ref = pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_lk_ref.so not built (needs the reference tree)")


@pytest.fixture(scope="module")
def ctx():
    c = lio.Context(0)
    yield c
    c.close()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _levels(dev, max_level, which=0):
    return [dev.level(which, l) for l in range(max_level + 1)]


@pytest.mark.parametrize("run", K.GOLDEN_RUNS, ids=[r[0] for r in K.GOLDEN_RUNS])
def test_device_matches_golden(ctx, run):
    g = np.load(GOLDEN)
    frames, pts, kw = K.run_inputs(run)
    dev = lio.LKOpticalFlowKernel(ctx, **kw)
    key = run[0] + "/"
    last = pts
    for k, f in enumerate(frames):
        assert K.image_digest(f) == str(g[key + f"image{k}"]), "the case generator no longer makes the golden frames"
        curr, st, ret = dev.trackImage(f, last)
        assert np.array_equal(bits(curr), bits(g[key + f"pts{k}"])), (k, np.flatnonzero((bits(curr) != bits(g[key + f"pts{k}"])).any(1))[:10])
        assert np.array_equal(st, g[key + f"status{k}"]), k
        assert ret == int(g[key + f"ret{k}"]), k
        assert K.level_digest(_levels(dev, dev.getMaxLevel())) == str(g[key + f"levels{k}"]), k
        last = curr
    assert dev.getMaxLevel() == int(g[key + "max_level"])
    dev.close()


@needs_ref
@pytest.mark.parametrize("size", [K.R3LIVE, K.NTU, (161, 97), (330, 50)])
def test_every_level_against_reference(ctx, size):
    """Every padded level and derivative buffer of both buffer sets, byte for byte, after each of three images."""
    cols, rows = size
    kw = lio.tracker_lk_params()
    dev, ref = lio.LKOpticalFlowKernel(ctx, **kw), R.LKReference(**kw)
    pts = K.points(cols, rows, 4, 300)
    for k, f in enumerate(K.frames(cols, rows, 4, 3)):
        c_ref, s_ref, r_ref = ref.track(f, pts)
        c_dev, s_dev, r_dev = dev.trackImage(f, pts)
        assert dev.getMaxLevel() == ref.info()["max_level"]
        for which in ((0,) if k == 0 else (0, 1)):
            for l in range(dev.getMaxLevel() + 1):
                ri, rd = ref.level(which, l)
                di, dd = dev.level(which, l)
                assert np.array_equal(di, ri), (k, which, l)
                assert np.array_equal(dd, rd), (k, which, l)
        assert np.array_equal(bits(c_dev), bits(c_ref)) and np.array_equal(s_dev, s_ref) and r_dev == r_ref


@needs_ref
@pytest.mark.parametrize("case", K.PARAM_CASES, ids=[c[0] for c in K.PARAM_CASES])
def test_parameters_against_reference(ctx, case):
    """Windows that move the SSE chunk boundaries, max_level 0/3/5, max_count 1/10/30, epsilon 0 and 0.05, at r3live's size."""
    _, win, max_level, criteria, flags, min_eig = case
    kw = dict(win_size=win, max_level=max_level, criteria=criteria, flags=flags, min_eig_threshold=min_eig)
    dev, ref = lio.LKOpticalFlowKernel(ctx, **kw), R.LKReference(**kw)
    pts = K.points(*K.R3LIVE, 31, 2000)
    last_d = last_r = pts
    for f in K.frames(*K.R3LIVE, 31, 4):
        c_ref, s_ref, r_ref = ref.track(f, last_r)
        c_dev, s_dev, r_dev = dev.trackImage(f, last_d)
        assert np.array_equal(bits(c_dev), bits(c_ref)) and np.array_equal(s_dev, s_ref) and r_dev == r_ref
        last_d, last_r = c_dev, c_ref


@needs_ref
def test_20000_points_sequence_against_reference(ctx):
    kw = lio.tracker_lk_params()
    dev, ref = lio.LKOpticalFlowKernel(ctx, **kw), R.LKReference(**kw)
    pts = K.points(*K.NTU, 41, 20000)
    last_d = last_r = pts
    for f in K.frames(*K.NTU, 41):
        c_ref, s_ref, r_ref = ref.track(f, last_r)
        c_dev, s_dev, r_dev = dev.trackImage(f, last_d)
        assert np.array_equal(bits(c_dev), bits(c_ref)) and np.array_equal(s_dev, s_ref) and r_dev == r_ref
        last_d, last_r = c_dev, c_ref


def test_first_call_and_empty_calls(ctx):
    """First image (:762-773): curr = last, status untouched, 0.  n = 0 still consumes the image."""
    fr = K.frames(*K.NTU, 5, 4)
    pts = K.points(*K.NTU, 5, 300)
    dev = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    curr, st = np.full((300, 2), -7.0, np.float32), np.full(300, 9, np.uint8)
    c, s, n = dev.trackImage(fr[0], pts, out=(curr, st))
    assert n == 0 and np.array_equal(bits(c), bits(pts)) and (s == 9).all()
    c, s, n = dev.trackImage(fr[1], np.zeros((0, 2), np.float32))
    assert n == 0 and c.shape == (0, 2) and s.shape == (0,)
    # the next call tracks from fr[1], which the empty call consumed: same as a kernel that saw fr[1] first
    other = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    other.trackImage(fr[1], pts)
    a = dev.trackImage(fr[2], pts)
    b = other.trackImage(fr[2], pts)
    assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1]) and a[2] == b[2] > 0
    if R.available():
        ref = R.LKReference(**lio.tracker_lk_params())
        c_r, s_r, n_r = ref.track(fr[0], pts, status_in=np.full(300, 9, np.uint8))
        assert n_r == 0 and (s_r == 9).all() and np.array_equal(bits(c_r), bits(pts))
        ref.track(fr[1], np.zeros((0, 2), np.float32))
        c_r, s_r, n_r = ref.track(fr[2], pts)
        assert np.array_equal(bits(a[0]), bits(c_r)) and np.array_equal(a[1], s_r) and a[2] == n_r


def test_host_and_device_buffers(ctx):
    """numpy in / numpy out, CUDA tensors in and out (the selection's device uv straight in), a pitched device image."""
    torch = pytest.importorskip("torch")
    fr = K.frames(*K.NTU, 6, 3)
    pts = K.points(*K.NTU, 6, 3000)
    kw = lio.tracker_lk_params()
    host = lio.LKOpticalFlowKernel(ctx, **kw)
    dev = lio.LKOpticalFlowKernel(ctx, **kw)
    pitched = lio.LKOpticalFlowKernel(ctx, **kw)
    last_h = pts
    last_d = torch.from_numpy(pts).cuda()
    last_p = pts
    for f in fr:
        ch, sh, nh = host.trackImage(f, last_h)
        cd, sd, nd = dev.trackImage(torch.from_numpy(f).cuda(), last_d)
        big = torch.zeros((f.shape[0], f.shape[1] + 40), dtype=torch.uint8, device="cuda")
        big[:, 8:8 + f.shape[1]] = torch.from_numpy(f).cuda()
        out = (torch.empty((3000, 2), dtype=torch.float32, device="cuda"), np.ones(3000, np.uint8))
        cp, sp, n_p = pitched.trackImage(big[:, 8:8 + f.shape[1]], last_p, out=out)
        assert cd.is_cuda and sd.is_cuda
        assert np.array_equal(bits(ch), bits(cd.cpu().numpy())) and np.array_equal(sh, sd.cpu().numpy()) and nh == nd
        assert np.array_equal(bits(ch), bits(cp.cpu().numpy())) and np.array_equal(sh, sp) and nh == n_p
        last_h, last_d, last_p = ch, cd, ch


def test_bad_arguments(ctx):
    with pytest.raises(capi.SrlError) as e:
        lio.LKOpticalFlowKernel(ctx, win_size=(2, 21))
    assert e.value.code == capi.SRL_BAD_ARG
    with pytest.raises(capi.SrlError):
        lio.LKOpticalFlowKernel(ctx, win_size=(21, 33))
    with pytest.raises(capi.SrlError):
        lio.LKOpticalFlowKernel(ctx, max_level=9)
    dev = lio.LKOpticalFlowKernel(ctx, **lio.tracker_lk_params())
    with pytest.raises(capi.SrlError) as e:
        dev.trackImage(np.zeros((21, 100), np.uint8), np.zeros((1, 2), np.float32))   # not larger than the window
    assert e.value.code == capi.SRL_BAD_ARG
    fr = K.frames(161, 97, 2, 2)
    dev.trackImage(fr[0], np.zeros((4, 2), np.float32))
    with pytest.raises(capi.SrlError) as e:
        dev.trackImage(np.zeros((98, 161), np.uint8), np.zeros((4, 2), np.float32))   # another size than the first image
    assert e.value.code == capi.SRL_BAD_ARG
    c, s, n = dev.trackImage(fr[1], K.points(161, 97, 2, 50))   # the kernel is still usable
    assert n > 0
