"""Writes tests/golden/image_prep.npz: OpenCV's own outputs of the camera image preparation for every case of
tests/image_prep_cases.py, by the call sequence of the reference:

  src/imageProcessing.cpp:93-104   image_scale_factor = image_width * 1.0 / cols; fx, cx, fy, cy /= it;
                                   initUndistortRectifyMap(K, dist, Mat(), K, Size(image_width / s, image_height / s), CV_16SC2)
  src/imageProcessing.cpp:121      remap(rgb_image, undist, map1, map2, INTER_LINEAR)
  src/imageProcessing.cpp:123,180  gray = cvtColor(undist, COLOR_RGB2GRAY)
  src/imageProcessing.cpp:124,169  createCLAHE(3, Size(t, t))->apply(gray), t = max(cols * 32.0 / 640, 4.0) truncated
  src/imageProcessing.cpp:185-200  rgb = YCrCb2BGR(merge(CLAHE(1, (t, t))(Y), Cr, Cb)) of BGR2YCrCb(undist)

Cases up to image_prep_cases.FULL_LIMIT output pixels keep the whole maps and images; larger ones keep SHA-256 digests of
map1, map2, gray and rgb.  Every case keeps the digest of its input image, so a change in the generator shows.

    python tests/golden/make_image_golden.py        (needs cv2)
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import image_prep_cases as IC  # noqa: E402


def opencv_recipe(bgr, image_width, image_height, camera_intrinsic, camera_dist_coeffs):
    s = image_width * 1.0 / bgr.shape[1]
    K = np.array(camera_intrinsic, np.float64).reshape(3, 3).copy()
    K[0, 0] /= s
    K[0, 2] /= s
    K[1, 1] /= s
    K[1, 2] /= s
    size = (int(image_width / s), int(image_height / s))
    map1, map2 = cv2.initUndistortRectifyMap(K, np.array(camera_dist_coeffs, np.float64), None, K, size, cv2.CV_16SC2)
    und = cv2.remap(bgr, map1, map2, cv2.INTER_LINEAR)
    t = int(max(und.shape[1] * 32.0 / 640, 4.0))
    gray = cv2.createCLAHE(3.0, (t, t)).apply(cv2.cvtColor(und, cv2.COLOR_RGB2GRAY))
    ch = list(cv2.split(cv2.cvtColor(und, cv2.COLOR_BGR2YCrCb)))
    ch[0] = cv2.createCLAHE(1.0, (t, t)).apply(ch[0])
    rgb = cv2.cvtColor(cv2.merge(ch), cv2.COLOR_YCrCb2BGR)
    return rgb, gray, map1, map2


def main():
    cv2.setNumThreads(1)
    out = {}
    for c in IC.CASES:
        bgr = c.bgr()
        rgb, gray, map1, map2 = opencv_recipe(bgr, **c.camera)
        out[f"{c.name}/input_sha"] = np.array(IC.digest(bgr))
        out[f"{c.name}/shape"] = np.array(gray.shape, np.int64)
        if gray.size <= IC.FULL_LIMIT:
            out[f"{c.name}/map1"], out[f"{c.name}/map2"] = map1, map2
            out[f"{c.name}/gray"], out[f"{c.name}/rgb"] = gray, rgb
        else:
            for k, v in (("map1", map1), ("map2", map2), ("gray", gray), ("rgb", rgb)):
                out[f"{c.name}/{k}_sha"] = np.array(IC.digest(v))
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "image_prep.npz"), **out)


if __name__ == "__main__":
    main()
