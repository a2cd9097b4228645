"""buildFrame's edge cases for tests/test_build_frame_edges_pin.py and tests/test_build_frame_edges_device.py.

Every case is a tests/build_frame_model.make_case dict, with a reason.  Extra keys: "rule", the draw rule a rejection frame
is built for, and "first_rejection", the first draw of shuffle 1 that rule rejects on the default-seeded engine.
"""
from __future__ import annotations

import functools

import numpy as np

import build_frame_model as M

# The default-seeded mt19937_64 first fails a draw's rejection test at these draws (the range a draw has depends on the
# parity of n, so the rule-0 index does too); the next rejection is hundreds of thousands of draws later.  A shuffle of n
# takes num_draws(n) draws, so each frame is a few points larger than the smallest that reaches its draw: shuffle 1 is redone
# on the host from there, and shuffle 2 starts one word later than it would without the rejection.
#   (name, n, rule, first rejected draw)
REJECTION = [
    ("reject_rule0_odd", 6_041_101, 0, 3_020_545),    # smallest n: 6 041 093
    ("reject_rule0_even", 6_588_170, 0, 3_294_078),   # smallest n: 6 588 158
    ("reject_rule1_even", 5_159_560, 1, 2_579_772),   # smallest n: 5 159 546
    ("reject_rule1_odd", 5_159_561, 1, 2_579_772),    # smallest n: 5 159 547
]
REJECTION_NAMES = [r[0] for r in REJECTION] + ["reject_rule0_odd_no_subsample"]


@functools.lru_cache(maxsize=1)
def rejection_case(name: str) -> dict:
    """Point time on, constant velocity, voxel_size > 0 (both shuffles run), steady cell size; "_no_subsample": voxel_size 0,
    shuffle 1 alone."""
    base = name.replace("_no_subsample", "")
    _, n, rule, first = next(r for r in REJECTION if r[0] == base)
    c = M.make_case(name, n=n, seed=100 + n % 97, index_frame=25, voxel_size=0.0 if name != base else 0.5, scale=60.0)
    c.update(rule=rule, first_rejection=first)
    return c


def _stamps(c, ts):
    c = dict(c)
    c["ts"] = np.asarray(ts, float)
    return c


def edge_cases() -> list[dict]:
    out = []
    # index_frame against init_num_frames (20) and the frame-index branches: 0 and 1 have no dt_offset, <= 2 alpha 1 and the
    # identity pose, 19 the initial cell and 20 the steady one.  Dense points (scale 3 m), so the two cells keep different sets.
    for k, idx in enumerate((0, 1, 2, 3, 19, 20)):
        out.append(M.make_case(f"index{idx}", n=3000, seed=200 + k, index_frame=idx, scale=3.0, point_time_enable=k % 2 == 0))
    # makePointTimestamp's erase keeps nothing (every stamp before begin or after end), subsampling on
    c = M.make_case("erase_all", n=1000, seed=210, point_time_enable=False, edges=False)
    out.append(_stamps(c, np.where(np.arange(1000) % 2 == 0, c["begin"] - 0.5, c["begin"] + c["offset"] + 0.5)))
    # NaN stamps at the first, a middle and the last point: both comparisons false, so the erase keeps them as point time does
    for k, (pte, mc) in enumerate(((True, 1), (False, 1), (True, 0), (False, 0))):
        c = M.make_case(f"nan_stamp_pte{int(pte)}_mc{mc}", n=2000, seed=220 + k, point_time_enable=pte, motion_compensation=mc)
        ts = c["ts"].copy()
        ts[[0, 1000, 1999]] = np.nan
        out.append(_stamps(c, ts))
    # ±inf stamps: point time keeps them (alpha +inf clamped, -inf not), the erase drops them
    for pte in (True, False):
        c = M.make_case(f"inf_stamp_pte{int(pte)}", n=2000, seed=230 + pte, point_time_enable=pte)
        ts = c["ts"].copy()
        ts[[0, 1]] = -np.inf
        ts[[1998, 1999]] = np.inf
        ts[700] = np.inf
        out.append(_stamps(c, ts))
    # timestamp_offset 0: alpha = rel / 0 is +inf, -inf or NaN (0 / 0); the clamp turns +inf into 1 - 1e-5.  Without point
    # time only the stamps exactly at begin stay.  The IMU track spans 0.1 s so the interpolation stays defined.
    for k, (pte, mc) in enumerate(((True, 1), (False, 1), (True, 0))):
        c = M.make_case(f"zero_offset_pte{int(pte)}_mc{mc}", n=2000, seed=240 + k, offset=0.0, imu_span=0.1, point_time_enable=pte,
                        motion_compensation=mc, edges=False)
        b = c["begin"]
        ts = b + np.sort(np.random.default_rng(k).uniform(-0.005, 0.1, 2000))
        ts[[10, 11, 500, 1500]] = b
        ts[12] = np.nextafter(b, np.inf)
        ts[13] = np.nextafter(b, -np.inf)
        out.append(_stamps(c, np.sort(ts) if mc == 0 else ts))
    # stamps exactly at begin and end at Unix-epoch values, no point time: the erase keeps both ends (its comparisons are strict)
    for mc in (1, 0):
        c = M.make_case(f"epoch_ends_erase_mc{mc}", n=3000, seed=250 + mc, point_time_enable=False, motion_compensation=mc, edges=False)
        b, e = c["begin"], c["begin"] + c["offset"]
        ts = c["ts"].copy()
        ts[:300] = b
        ts[300:310] = np.nextafter(b, -np.inf)
        ts[-300:] = e
        ts[-310:-300] = np.nextafter(e, np.inf)
        out.append(_stamps(c, np.sort(ts)))
    # IMU state counts: one state (the IMU walk has no interval, the constant model one stamp), 4096 (the most the IMU walk
    # takes), 4097 with constant velocity (no limit there; the IMU walk refuses it, see the device file)
    for mc in (1, 0):
        out.append(M.make_case(f"one_state_mc{mc}", n=2000, seed=260 + mc, motion_compensation=mc, n_states=1))
        out.append(M.make_case(f"states4096_mc{mc}", n=2000, seed=262 + mc, motion_compensation=mc, n_states=4096,
                               edges=mc == 1, early=0.05 if mc == 1 else 0.0))
    out.append(M.make_case("states4097_mc1", n=2000, seed=264, n_states=4097))
    # init_voxel_size <= 0 is not used from init_num_frames on, and not at all with voxel_size <= 0
    out.append(M.make_case("init_size_zero_steady", n=2000, seed=270, index_frame=20, init_voxel_size=0.0))
    out.append(M.make_case("init_size_negative_no_subsample", n=2000, seed=271, index_frame=3, init_voxel_size=-1.0, voxel_size=0.0))
    return out


def reuse_sequence() -> list[dict]:
    """Frames built one after another into one object created for 4096 points: growth to 8192 (doubling), a smaller frame,
    growth to 16384, a small frame, growth straight to 40000 (more than double), an empty frame, then one that fits again."""
    sizes = (5000, 3000, 9000, 200, 40000, 0, 7000)
    return [M.make_case(f"reuse{k}_{n}", n=n, seed=300 + k, index_frame=1 + k, point_time_enable=k % 3 != 1,
                        motion_compensation=k % 2) for k, n in enumerate(sizes)]
