"""Record the reference's own cloudProcessing (oracle/_ref/libsrl_cloud_processing_ref.so, built by oracle/cloud_processing.mk)
over the seeded scenes of tests/cloud_processing_ref.py into tests/golden/cloud_processing.npz.  Only outputs are stored: after
every message, the points it appended (raw_point, relative_time, timestamp) and the handler state; the messages are regenerated
from their seeds.

    python tests/golden/make_cloud_processing_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import cloud_processing_ref as R  # noqa: E402


def main():
    out = {}
    for name, (lt, ns, rate, tu, blind, f, _) in R.SCENES.items():
        ref = R.ReferenceCP(lt, ns, rate, tu, blind, f)
        for m, (kind, msg, stamp) in enumerate(R.scene_messages(name)):
            ref.livox(msg, stamp) if kind == "livox" else ref.process(msg, stamp)
            xyz, rel, ts = ref.drain()
            le, given, sweep_id, _ = ref.state()
            key = f"{name}/{m}"
            out[key + "/xyz"], out[key + "/rel"], out[key + "/ts"] = xyz, rel, ts
            out[key + "/state"] = np.array([le, float(given), float(sweep_id)])
        ref.close()
    np.savez_compressed(os.path.join(HERE, "cloud_processing.npz"), **out)


if __name__ == "__main__":
    main()
