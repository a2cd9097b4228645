"""Generates tests/golden/vio_edges.npz: the outcomes of the reference's own imageProcessing::vioEsikf and vioPhotometric
(compiled into oracle/_ref/libsrl_vio_ref.so by oracle/vio.mk) on the edge cases of tests/test_vio_edges_device.py:
  branch_<a>_<b>.ids, .xyz, .rgb, .cov_rgb, .n_rgb, .uv, .vel, .state    the rotation-branch scenes' inputs, as the device builds them
  branch_<a>_<b>.img_digest                                               sha256 of the image the photometric update samples
  branch_<a>_<b>.esikf.state / .cov / .result, ....photometric.*          the reference's outputs from the setInitialCov covariance
  pivot.<esikf|photometric>.<column>.cov / .state                         the pivot cases' covariances on the base scene, and the
                                                                          reference's state from them
  tiled.esikf.state                                                       vioEsikf over the 20 247-point tiled list
The scenes are built on the device, so this needs a CUDA device and the reference library.  Run from the repo root:
    python tests/golden/make_vio_edges_golden.py [output path]
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, ROOT)
import vio_cases as VC         # noqa: E402
import vio_edge_cases as EC    # noqa: E402
import vio_ref as RF           # noqa: E402
from sr_livo_b200 import lio   # noqa: E402
from test_vio_edges_device import SCENES   # noqa: E402


def _ref(which, sc, cov, idx=None):
    s = sc if idx is None else VC.subset(sc, idx)
    return RF.update(which, sc["state"], cov, s["xyz"], s["uv"], s["vel"], s["rgb"], s["cov_rgb"], s["n_rgb"], 40, s["img"])


def main(path):
    if not RF.available():
        raise SystemExit("oracle/_ref/libsrl_vio_ref.so is missing: run __graft_entry__.build() with the reference tree present")
    ctx = lio.Context(0)
    out = {}
    for a, b in EC.BRANCH_PAIRS:
        name = f"branch_{a}_{b}"
        sc = VC.device_scene(lio, ctx, **SCENES[name])
        for k in ("ids", "xyz", "rgb", "cov_rgb", "n_rgb", "uv", "vel", "state"):
            out[f"{name}.{k}"] = sc[k]
        out[f"{name}.img_digest"] = np.frombuffer(VC.image_digest(sc["img"]), np.uint8)
        for which, w in ((0, "esikf"), (1, "photometric")):
            s, c, r, _ = _ref(which, sc, VC.initial_covariance())
            out[f"{name}.{w}.state"], out[f"{name}.{w}.cov"], out[f"{name}.{w}.result"] = s, c, np.int32(r[which])
        sc["cm"].close(); sc["ip"].close()
    sc = VC.device_scene(lio, ctx, **SCENES["base"])
    for esikf in (True, False):
        for col in EC.PIVOT_TARGETS[esikf]:
            cov = EC.pivot_covariance(sc, esikf, col)
            key = f"pivot.{'esikf' if esikf else 'photometric'}.{col}"
            out[key + ".cov"] = cov
            out[key + ".state"] = _ref(0 if esikf else 1, sc, cov)[0]
    out["tiled.esikf.state"] = _ref(0, sc, VC.initial_covariance(), EC.tiled())[0]
    sc["cm"].close(); sc["ip"].close()
    ctx.close()
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(out)} arrays")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "vio_edges.npz"))
