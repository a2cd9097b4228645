"""Generates tests/golden/vio_updates.npz: the outcomes of the reference's own imageProcessing::vioEsikf and vioPhotometric
(src/imageProcessing.cpp, compiled into oracle/_ref/libsrl_vio_ref.so by oracle/vio.mk) on the device scenes of
tests/vio_cases.py (device_scene), from the setInitialCov covariance.  Per scene:
  <scene>.ids, .xyz, .rgb, .cov_rgb, .n_rgb, .uv, .vel, .state   the inputs as the device scene produces them (the GPU test
                                                                checks that its scene is still this one, bit for bit)
  <scene>.img_digest                                            sha256 of the image the photometric update samples
  <scene>.esikf.state / .cov / .result, <scene>.photometric.state / .cov / .result   the reference's outputs
The scenes are built on the device (the colour state is the renderer's), so this needs a CUDA device and the reference
library.  Run from the repo root:  python tests/golden/make_vio_golden.py [output path]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import vio_cases as VC   # noqa: E402
import vio_ref as RF     # noqa: E402
from sr_livo_b200 import lio   # noqa: E402

SCENES = {"base_ntu": dict(camera="ntu"), "base_r3live": dict(camera="r3live", seed=502),
          "mixed": dict(camera="ntu", seed=503, n_usable=200, n_fresh=300)}


def main(path):
    if not RF.available():
        raise SystemExit("oracle/_ref/libsrl_vio_ref.so is missing: run __graft_entry__.build() with the reference tree present")
    ctx = lio.Context(0)
    out = {}
    for name, kw in SCENES.items():
        sc = VC.device_scene(lio, ctx, **kw)
        for k in ("ids", "xyz", "rgb", "cov_rgb", "n_rgb", "uv", "vel", "state"):
            out[f"{name}.{k}"] = sc[k]
        out[f"{name}.img_digest"] = np.frombuffer(VC.image_digest(sc["img"]), np.uint8)
        for which, w in ((0, "esikf"), (1, "photometric")):
            s, c, r, _ = RF.update(which, sc["state"], VC.initial_covariance(), sc["xyz"], sc["uv"], sc["vel"], sc["rgb"], sc["cov_rgb"],
                                   sc["n_rgb"], 40, sc["img"])
            out[f"{name}.{w}.state"], out[f"{name}.{w}.cov"], out[f"{name}.{w}.result"] = s, c, np.int32(r[which])
        sc["cm"].close(); sc["ip"].close()
    ctx.close()
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "vio_updates.npz"))
