"""Generates tests/golden/lk_track.npz: the outputs of the reference's own LKOpticalFlowKernel::trackImage (src/lkpyramid.cpp,
compiled into oracle/_ref/libsrl_lk_ref.so by oracle/lk.mk) on the runs of tests/lk_cases.py GOLDEN_RUNS.  Per run and call k:
  <run>/pts<k>, <run>/status<k>, <run>/ret<k>   trackImage's outputs (status starts at ones)
  <run>/levels<k>                               sha256 of the last image's padded pyramid and derivative buffers after the call
  <run>/max_level                               getMaxLevel() after the first call
  <run>/image<k>                                sha256 of the generated frame (the generator's bytes are part of the pin)
Needs the reference tree (to build the library).  Run from the repo root:  python tests/golden/make_lk_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import lk_cases as K   # noqa: E402
import lk_ref as R     # noqa: E402


def reference_run(run):
    frames, pts, kw = K.run_inputs(run)
    ref = R.LKReference(**kw)
    out = {}
    last = pts
    for k, f in enumerate(frames):
        curr, st, ret = ref.track(f, last)
        out[f"pts{k}"], out[f"status{k}"], out[f"ret{k}"] = curr, st, np.int64(ret)
        ml = ref.info()["max_level"]
        out[f"levels{k}"] = np.array(K.level_digest([ref.level(0, l) for l in range(ml + 1)]))
        out[f"image{k}"] = np.array(K.image_digest(f))
        last = curr
    out["max_level"] = np.int64(ref.info()["max_level"])
    ref.close()
    return out


def main():
    assert R.available(), "oracle/_ref/libsrl_lk_ref.so is not built (it needs the reference tree)"
    data = {}
    for run in K.GOLDEN_RUNS:
        for key, v in reference_run(run).items():
            data[f"{run[0]}/{key}"] = v
    np.savez_compressed(os.path.join(HERE, "lk_track.npz"), **data)
    print("wrote", len(data), "arrays")


if __name__ == "__main__":
    main()
