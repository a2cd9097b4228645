"""Writes tests/golden/image_prep_edges.npz: OpenCV's own outputs of the camera image preparation for the edge cases of
tests/image_prep_edge_cases.py, by the reference's call sequence (make_image_golden.opencv_recipe).

Every case keeps SHA-256 digests of its input image, map1, gray and rgb, and of map2 at the unsaturated entries only (a
vectorised OpenCV may give a saturated entry's map2 another last bit, which no image can show).  Digests keep the file small;
the tests report where outputs differ by comparing the restatement with live cv2 and the device with the restatement.  The
tie-heavy map is left out: which way OpenCV rounds a 1/32 tie depends on its build.

    python tests/golden/make_image_edges_golden.py        (needs cv2)
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import image_prep_edge_cases as EC  # noqa: E402
import image_prep_reference as R  # noqa: E402
from make_image_golden import opencv_recipe  # noqa: E402


def main():
    cv2.setNumThreads(1)
    out = {}
    for c in EC.CASES:
        if not c.opencv:
            continue
        bgr = c.bgr()
        rgb, gray, map1, map2 = opencv_recipe(bgr, **c.camera)
        out[f"{c.name}/input_sha"] = np.array(EC.digest(bgr))
        out[f"{c.name}/shape"] = np.array(gray.shape, np.int64)
        for k, v in (("map1", map1), ("map2_unsat", map2[~R.saturated(map1)]), ("gray", gray), ("rgb", rgb)):
            out[f"{c.name}/{k}_sha"] = np.array(EC.digest(v))
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "image_prep_edges.npz"), **out)


if __name__ == "__main__":
    main()
