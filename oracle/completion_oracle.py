"""ORACLE (test infrastructure only): numpy restatement of the shape-completion metrics of diffusion/completion.py and of
`mdb_chamfer_pairs` (geometry/pointcloud.py `chamfer_pairs`).

The paired distances use the kernel's formula in fp64: d(x, y) = |x - y|^2, CD(a, b) = mean_x min_y d + mean_y min_x d,
the a->b mean and the a->b max of the row minima. TMD, UHD, accuracy and sign agreement are written as explicit loops over
completions and pairs, straight from their definitions (Wu et al. 2020, Multimodal Shape Completion via Conditional
GANs), so they check the driver's vectorised bookkeeping rather than restate it.
"""
import math

import numpy as np


def _sq(a, b):
    a = np.asarray(a, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    return ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1)


def pair_distances(a, b):
    """(CD(a, b), mean over x in a of min over y in b of d, max over x in a of the same minimum), fp64."""
    d = _sq(a, b)
    row, col = d.min(axis=1), d.min(axis=0)
    return float(row.mean() + col.mean()), float(row.mean()), float(row.max())


def chamfer(a, b):
    return pair_distances(a, b)[0]


def uhd(partial, completion):
    """max over x in the partial of min over y in the completion of |x - y| (Euclidean)."""
    best = 0.0
    for x in np.asarray(partial, np.float64):
        best = max(best, min(math.dist(x, y) for y in np.asarray(completion, np.float64)))
    return best


def tmd(completions):
    """(2 / (k - 1)) sum over i < j of CD(c_i, c_j)."""
    k = len(completions)
    s = 0.0
    for i in range(k):
        for j in range(i + 1, k):
            s += chamfer(completions[i], completions[j])
    return 2.0 * s / (k - 1)


def accuracy(completions, gt):
    """(min over j, mean over j) of CD(c_j, gt)."""
    cds = [chamfer(c, gt) for c in completions]
    return min(cds), sum(cds) / len(cds)


def sign_agreement(channel0_at_verts, partial_sdf, partial_vis):
    """Share of the vertices with vis > 0 where sign(channel 0) equals the partial's sdf."""
    n = agree = 0
    for c, s, v in zip(np.asarray(channel0_at_verts, np.float64), np.asarray(partial_sdf, np.float64),
                       np.asarray(partial_vis, np.float64)):
        if v > 0:
            n += 1
            agree += int(np.sign(c) == s)
    return agree / n if n else float("nan")


def visible_face_ids(face_id):
    """Sorted ids of the faces that own at least one pixel of a face-id buffer (-1 = empty)."""
    seen = set()
    for f in np.asarray(face_id).reshape(-1):
        if f >= 0:
            seen.add(int(f))
    return sorted(seen)
