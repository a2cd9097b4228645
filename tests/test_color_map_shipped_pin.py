"""Row N4 at the shipped map_options (config/r3live.yaml, config/ntu.yaml: 0.1 m / 50 / 0.01 m; r3live_compressed.yaml: 100
points): the reference's own addPointsToMap colour branch and renderPointsInRecentVoxel (compiled from its sources) against
the oracle, on dense surfaces that overfill the voxels and on points whose keys wrap (+-400 m, 655.36 m / 6553.6 m
aliasing pairs, beyond +-3276.8 m).  Also pins the oracle's keys to the wrap formula the GPU kernels implement.

CPU only; skipped when the reference library was not built.
"""
import numpy as np
import pytest

from oracle import oracle_py as O
from oracle import reference_py as Rf

from color_map_cases import FINE, SIZE, camera, model_lists, sweep, wrap_key

pytestmark = pytest.mark.skipif(not Rf.available(), reason="oracle/_ref/libsrl_reference.so not built (needs /root/reference)")

FIELDS = ("counts", "xyz", "rgb", "n_rgb", "cov", "obs_dist", "last_obs", "last_visited")


def test_wrap_key_is_the_low_16_bits_of_the_int32_truncation():
    x = np.array([327.6, 327.7, 400.0, -400.0, 655.36, 1000.0, 3276.8, -3276.9, 6553.6, 1e6])
    k = wrap_key(np.stack([x, x, x], axis=1), FINE)[:, 0].astype(np.int64)
    q = np.trunc(x.astype(np.float32).astype(np.float64) / FINE).astype(np.int64)
    assert np.array_equal(k, ((q + 32768) % 65536) - 32768)
    assert k[2] == -25536 and k[0] == 32760 and k[1] == -32766      # 400 m -> -25536; 327.7 m -> 32770 - 65536


@pytest.mark.parametrize("cap", [50, 100])
@pytest.mark.parametrize("step", [1, 4])
def test_shipped_color_map_reference_equals_oracle(cap, step):
    ref = Rf.Reference()
    oc = O.OracleColorMap(voxel_size=SIZE, max_num_points_in_voxel=cap, min_distance_points=FINE)
    rng = np.random.default_rng(100 * cap + step)
    fed = []
    for s, (t_end, t_proc) in enumerate([(1.0, 0.0), (1.1, 1.0)]):
        pts = sweep(seed=7 * cap + 31 * step + s)
        if s == 1:
            pts = pts + rng.normal(0, 0.003, pts.shape)              # the same surfaces again: full voxels refuse, fine cells dedupe
        ref.add_points_to_map(pts, 1.0, 20, 0.15, 0, color_voxel_size=SIZE, color_max_points=cap, color_min_distance=FINE,
                              add_point_step=step, time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        oc.add_points(pts, add_point_step=step, time_sweep_end=t_end, time_last_process=t_proc, to_rendering=True)
        fed.append((pts, step))
        assert ref.color_counts() == oc.counts()
        la, lb = ref.color_lists(), oc.lists()
        assert np.array_equal(la[0], lb[0]) and np.array_equal(la[1], lb[1])   # rgb_points_vec, voxels_recent_visited, in order
        for k, pos in enumerate([(0.0, 0.0, 0.0), (400.0, 0.0, 0.0)]):          # two renderings: near surfaces, then the +400 m ones
            img = rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)
            cam, obs = camera(pos), t_end + 0.01 * (k + 1)
            assert ref.color_render(cam, img, obs) == oc.render(cam, img, obs)
        sa, sb = ref.snapshot(which=1, cap=cap, color=True), oc.snapshot()
        da = {tuple(key): i for i, key in enumerate(sa["keys"].tolist())}
        assert da.keys() == {tuple(key) for key in sb["keys"].tolist()}
        for j, key in enumerate(sb["keys"].tolist()):
            i = da[tuple(key)]
            for f in FIELDS:
                assert np.array_equal(sa[f][i], sb[f][j]), (f, key)
    # the scene does what it is meant to: full voxels, wrapped keys, both aliasing kinds, and colours written
    assert sb["counts"].max() == cap and (sb["counts"] == cap).sum() > 20
    keys = sb["keys"].astype(np.int64)
    assert (np.abs(keys[:, 0]) > 3000).any() and (sb["n_rgb"] >= 2).any()
    # the oracle's keys are the wrap formula: voxel contents counts and rgb_points_vec from a plain model of the rule
    counts, rgb = model_lists(fed, cap)
    assert {tuple(k): c for k, c in zip(sb["keys"].tolist(), sb["counts"].tolist())} == counts
    assert np.array_equal(lb[0], rgb)
    # the 655.36 m partner of a near point never opens its own fine cell when the near point came first, so the fine keys wrap
    assert len(rgb) < sum(counts.values())
