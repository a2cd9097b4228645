"""The LIO voxel map at its edges on the CPU: the plain restatement (tests/map_reference.py) against the oracle on every case
of tests/map_edge_cases.py (contents and order inside each voxel, counts, points stored, the published cloud and voxels
evicted), and against the reference's own compiled code where oracle/_ref was built.  Also the self-checks of the crafted
ties and of the mined hash collisions.

The reference's static_cast<short> is undefined for NaN, +-inf and |q| >= 2^31; the restatement drops such points, so the
oracle and the reference are fed the other points only (map_edge_cases.defined).
"""
import numpy as np
import pytest

from oracle import publish_oracle as PO
from oracle import reference_py as R

import map_edge_cases as E
import publish_ref as PR
from map_reference import MapRef, certify_pair, exact_sq, hash_key, short_key

CASES = {c.name: c for c in E.all_cases()}


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def map_dict(keys, counts, xyz):
    return {tuple(k): np.ascontiguousarray(x[:c]) for k, c, x in zip(np.asarray(keys).tolist(), np.asarray(counts).tolist(), xyz)}


def assert_same_map(got: dict, want: dict, where):
    assert got.keys() == want.keys(), where
    bad = [k for k in want if not np.array_equal(bits(got[k]), bits(want[k]))]
    assert not bad, (where, bad[:5])


def replay_restatement(case):
    """[(op, result, map after)] of the restatement: insert -> (added, cloud), remove -> voxels evicted."""
    m = MapRef(case.size, case.cap)
    out = []
    for op in case.ops:
        if op[0] == "upload":
            m.load(*op[1:])
            res = None
        elif op[0] == "insert":
            res = m.add_points(op[1], op[2], op[3], op[4])
        else:
            res = m.remove_far(op[1], op[2])
        out.append((op, res, m.as_dict()))
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_equals_oracle(name):
    case = CASES[name]
    om = PO.OracleMap()
    for i, (op, res, state) in enumerate(replay_restatement(case)):
        if op[0] == "upload":
            om.load(*op[1:])
        elif op[0] == "insert":
            added, cloud = om.add_points_published(E.defined(op[1], case.size), op[4], case.size, case.cap, op[2], op[3])
            assert added == res[0], (i, added, res[0])
            assert cloud.shape == res[1].shape and np.array_equal(bits(cloud), bits(res[1])), i
        else:
            assert not case.empty_voxels
            assert om.remove_far(op[1], op[2]) == res, i
        assert_same_map(map_dict(*om.snapshot(case.cap)), state, i)


@pytest.mark.skipif(not R.available(), reason="oracle/_ref/libsrl_reference.so not built (needs the reference tree)")
@pytest.mark.parametrize("name", list(CASES))
def test_restatement_equals_compiled_reference(name):
    case = CASES[name]
    ref = R.Reference()
    for i, (op, res, state) in enumerate(replay_restatement(case)):
        if op[0] == "upload":
            ref.load(*op[1:])
        elif op[0] == "insert":
            assert ref.add_points_to_map(E.defined(op[1], case.size), case.size, case.cap, op[2], op[3]) == res[0], i
        else:
            assert ref.remove_far(op[1], op[2]) == res, i
        s = ref.snapshot(0, case.cap)
        assert_same_map(map_dict(s["keys"], s["counts"], s["xyz"]), state, i)


@pytest.mark.skipif(not PR.available(), reason="oracle/_ref/libsrl_publish_ref.so not built (needs the reference tree)")
@pytest.mark.parametrize("name", [n for n, c in CASES.items() if all(op[0] == "insert" for op in c.ops)])
def test_published_cloud_equals_compiled_reference(name):
    case = CASES[name]
    ref = PR.PublishReference()
    for i, (op, res, _) in enumerate(replay_restatement(case)):
        added, cloud = ref.add_points_to_map(E.defined(op[1], case.size), op[4], case.size, case.cap, op[2], op[3])
        assert added == res[0] and cloud.shape == res[1].shape and np.array_equal(bits(cloud), bits(res[1])), i


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.certs])
def test_crafted_pairs_are_what_they_claim(name):
    case = CASES[name]
    for cert in case.certs:
        c = certify_pair(cert["a"], cert["b"], cert["md"])
        lim = 10 * case.size * case.size
        decided = min(lim, c["sq"]) > c["thr"]
        assert decided == cert["add"], cert
        if cert.get("exact"):          # a true tie: both sides exact in double, and equal
            assert c["sq_exact"] and c["thr_exact"] and c["ulps"] == 0, cert
        if "ulps" in cert:
            assert c["ulps"] == cert["ulps"], (cert, c)
        if cert.get("split"):          # the other reduction order would decide the opposite
            assert (c["other_order"] > c["thr"]) != cert["add"], (cert, c)
        if cert.get("clamp"):          # only the clamp decides
            assert exact_sq(cert["a"], cert["b"]) > lim and c["sq"] > c["thr"], cert
        # the restatement takes the same decision for the pair in an empty map
        m = MapRef(case.size, case.cap)
        m.add_points([cert["a"]], cert["md"])
        assert m.add_points([cert["b"]], cert["md"])[0] == int(cert["add"]), cert


def test_mined_chain_keys_collide():
    near, far = E.chain_keys()
    keys = near + far
    assert len(set(keys)) == len(keys) == 200
    for k in keys:
        h = hash_key(*k)
        assert h & 2047 >= 2044 and h & 1023 >= 1020, k
    assert all(max(abs(c) for c in k) <= 30 for k in near) and all(k[0] >= 100 or k[0] <= -100 for k in far)


def test_hash_key_is_uint32_arithmetic():
    # h = x*73856093 ^ y*19349669 ^ z*83492791 in uint32, then the avalanche steps; worked by hand for two keys
    def direct(x, y, z):
        h = ((x * 73856093) ^ (y * 19349669) ^ (z * 83492791)) % 2 ** 32
        h ^= h >> 16
        h = (h * 0x85EBCA6B) % 2 ** 32
        return h ^ (h >> 13)
    for k in [(0, 0, 0), (1, 0, 0), (-1, 0, 0), (32767, -32768, 5), (-12, 7, -30000)]:
        assert hash_key(*k) == direct(*k), k
    assert hash_key(0, 0, 0) == 0


def test_key_rule():
    assert [short_key(q) for q in (0.0, -0.0, 0.999, -0.999, 1.0, -1.0)] == [0, 0, 0, 0, 1, -1]
    assert [short_key(q) for q in (32767.5, 32768.0, -32768.5, -32769.0, 40000.0, 65541.5)] == [32767, -32768, -32768, 32767, -25536, 5]
    assert short_key(2.0 ** 31 - 1) == -1 and short_key(-(2.0 ** 31) + 1) == 1
    for q in (2.0 ** 31, -(2.0 ** 31), float("nan"), float("inf"), -float("inf")):
        assert short_key(q) is None
