"""Triangle meshes from `.obj` files for `--mode=fit_grids`, and the normalisation the reference applies before it fits a
grid (nvdiffrec/fit_dmtets.py:679-680, `center_by_reference(mesh, aabb_clean(mesh), 1.0)`). The writer is
mesh_ops.write_obj."""
import numpy as np


def _index(token, n_verts):
    """1-based OBJ index (negative: relative to the vertices read so far) -> 0-based."""
    k = int(token.split("/")[0])
    if k == 0:
        raise ValueError("OBJ vertex index 0")
    return k - 1 if k > 0 else n_verts + k


def read_obj(path):
    """-> (verts float64 [V, 3], faces int64 [F, 3]). Reads `v` lines and `f` lines in the forms `a`, `a/b`, `a//c` and
    `a/b/c` with positive or negative indices; polygons are fan-triangulated (a b c d -> a b c, a c d); every `o` / `g`
    group goes into the one mesh; every other line is ignored. A face naming a vertex that does not exist raises."""
    verts, faces = [], []
    with open(path, "r", errors="replace") as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f" and len(tok) >= 4:
                idx = [_index(t, len(verts)) for t in tok[1:]]
                if min(idx) < 0 or max(idx) >= len(verts):
                    raise ValueError(f"{path}: face {' '.join(tok[1:])} names a vertex that is not defined before it")
                faces.extend([idx[0], idx[i], idx[i + 1]] for i in range(1, len(idx) - 1))
    return np.asarray(verts, np.float64).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3)


def normalize(verts, faces, extent=1.0):
    """fit_dmtets.py:680: centre on the midpoint of the bounding box of the vertices the faces reference and scale so that
    the box's largest side is `extent` (float64) -> fp32 [V, 3]. Unreferenced vertices move along but do not count."""
    v = np.asarray(verts, np.float64)
    used = v[np.unique(np.asarray(faces).reshape(-1))]
    if used.shape[0] == 0:
        raise ValueError("the mesh has no faces")
    lo, hi = used.min(0), used.max(0)
    size = float((hi - lo).max())
    if not (size > 0 and np.isfinite(size)):
        raise ValueError("the mesh's faces span no volume")
    return ((v - (lo + hi) * 0.5) * (extent / size)).astype(np.float32)


def load_mesh(path):
    """read_obj + normalize -> (verts fp32 [V, 3], faces int64 [F, 3])."""
    v, f = read_obj(path)
    return normalize(v, f), f
