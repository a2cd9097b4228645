"""The pyramidal Lucas-Kanade on the GPU (srl_lk_*, lio.LKOpticalFlowKernel) at its edges: on every crafted family of
tests/lk_edge_cases.py it equals the numpy restatement (tests/lk_track_reference.py) always, and the compiled reference
(oracle/_ref/libsrl_lk_ref.so) when it was built.  Point bits (NaN payloads included), status and the return value exactly;
the level count; every padded level and derivative buffer byte for byte on the shape family."""
import numpy as np
import pytest

import lk_edge_cases as E
import lk_ref as R
from sr_livo_b200 import lio

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:invalid value encountered:RuntimeWarning")]


@pytest.fixture(scope="module")
def ctx():
    c = lio.Context(0)
    yield c
    c.close()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _device(ctx, case):
    dev = lio.LKOpticalFlowKernel(ctx, **case.kw)
    c0, s0, r0 = dev.trackImage(case.frames[0], case.pts)
    assert r0 == 0 and np.array_equal(bits(c0), bits(case.pts)) and (s0 == 1).all()   # the first image: points copied bit for bit
    return dev, dev.trackImage(case.frames[1], case.pts)


def _same(got, want, name):
    (c, s, r), (cw, sw, rw) = got, want
    bad = np.flatnonzero((bits(c) != bits(cw)).any(1))
    assert not len(bad), (name, bad[:8], bits(c)[bad[:4]], bits(cw)[bad[:4]])
    assert np.array_equal(s, sw) and r == rw, name


@pytest.mark.parametrize("family", list(E.FAMILIES))
def test_device_matches_restatement_and_reference(ctx, family):
    for case in E.FAMILIES[family]():
        curr, st, ret, _, res = E.restate(case)
        dev, got = _device(ctx, case)
        _same(got, (curr, st, ret), case.name)
        assert dev.getMaxLevel() == res.max_level, case.name
        if family == "shapes":
            for which in (0, 1):
                for l in range(res.max_level + 1):
                    di, dd = dev.level(which, l)
                    ri, rd = res.level(which, l)
                    assert np.array_equal(di, ri) and np.array_equal(dd, rd), (case.name, which, l)
        if R.available():
            ref = R.LKReference(**case.kw)
            ref.track(case.frames[0], case.pts)
            _same(got, ref.track(case.frames[1], case.pts), case.name)
        dev.close()
