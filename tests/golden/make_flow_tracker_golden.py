"""Freeze the reference's own optical-flow tracker bookkeeping (oracle/_ref/libsrl_flow_tracker_ref.so) on the pin sequences
of tests/flow_tracker_cases.py into tests/golden/flow_tracker.npz: after every call, last (ids, uv), cur (ids, uv, velocity),
every point's is_out_lier_count and the number of Lucas-Kanade calls.  Run from the repository root after build()."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))   # tests/

import flow_tracker_cases as FC   # noqa: E402
import flow_tracker_ref as RF     # noqa: E402

FIELDS = ("last_ids", "last_uv", "cur_ids", "cur_uv", "cur_vel", "counts", "lk_calls")


def main():
    out = {}
    for max_points in FC.PIN_MAX_POINTS:
        r = RF.FlowTrackerReference(FC.pin_points(), max_points)
        for k, step in enumerate(FC.run_pin(r, False, max_points)):
            for f, a in zip(FIELDS, step[1:]):
                out[f"max{max_points}.{k:02d}.{step[0]}.{f}"] = np.asarray(a)
        r.close()
    np.savez_compressed(os.path.join(HERE, "flow_tracker.npz"), **out)
    print(f"wrote {len(out)} arrays")


if __name__ == "__main__":
    main()
