"""tests/golden/singleview_cameras.json: the model-view-projection matrices of the reference's validation poses
`itr` = 0, 1, 17, 49 (DatasetMesh._rotate_scene, nvdiffrec/lib/dataset/dataset_mesh.py:67-76), computed by the UNMODIFIED
reference helpers `util.perspective / translate / rotate_x / rotate_y` (nvdiffrec/lib/render/util.py:193-243) with
RADIUS = 2 (fit_singleview.py:44), fovy = 45 degrees, a square image and cam_near_far = [0.1, 1000].

Run in the authoring container only (needs /root/reference). util.py imports nvdiffrast.torch and imageio at module level
and uses neither in these helpers, so both are replaced by empty stub modules for the import.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
GOLD = os.path.join(ROOT, "tests", "golden")
VIEWS = (0, 1, 17, 49)


def import_reference_util():
    nvdiffrast = types.ModuleType("nvdiffrast")
    nvdiffrast.torch = types.ModuleType("nvdiffrast.torch")
    sys.modules.setdefault("nvdiffrast", nvdiffrast)
    sys.modules.setdefault("nvdiffrast.torch", nvdiffrast.torch)
    sys.modules.setdefault("imageio", types.ModuleType("imageio"))
    spec = importlib.util.spec_from_file_location("_ref_render_util", os.path.join(REF, "nvdiffrec", "lib", "render", "util.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    util = import_reference_util()
    fovy, radius, near, far = np.deg2rad(45), 2.0, 0.1, 1000.0
    out = {"views": list(VIEWS), "mvp": []}
    for itr in VIEWS:
        proj = util.perspective(fovy, 1000 / 1000, near, far)
        ang = (itr / 50) * np.pi * 2
        mv = util.translate(0, 0, -radius) @ (util.rotate_x(-0.4) @ util.rotate_y(ang))
        out["mvp"].append([[float(x) for x in row] for row in (proj @ mv).numpy()])
    path = os.path.join(GOLD, "singleview_cameras.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1)
    print(path)


if __name__ == "__main__":
    main()
