"""numpy restatement of mdb_slerp_frames (csrc/interp.cu): spherical interpolation of endpoint pairs.

`slerp_sums` gives (a.b, a.a, b.b) in fp64 (numpy's summation order, not the kernel's fixed tree: the kernel's sums agree
to rounding). `slerp_coef` is phase 2 on given sums, so with the kernel's own sums it reproduces the kernel's weights
up to the last bit of the fp64 transcendentals. `slerp_combine` is phase 3 bit for bit: fl(fl(w_a a) + fl(w_b b)) in
float32, each product and the sum rounded on its own.
"""
import numpy as np


def slerp_sums(a, b):
    a = np.asarray(a, np.float64).reshape(-1)
    b = np.asarray(b, np.float64).reshape(-1)
    return np.array([a @ b, a @ a, b @ b], np.float64)


def slerp_coef(sums, alphas):
    """[F, 2] float32 (w_a, w_b) for the fp64 sums (a.b, a.a, b.b)."""
    ab, aa, bb = (float(v) for v in sums)
    out = np.empty((len(alphas), 2), np.float32)
    theta = st = None
    if aa > 0.0 and bb > 0.0:
        c = min(1.0, max(-1.0, ab / np.sqrt(aa * bb)))
        theta = np.arccos(c)
        st = np.sin(theta)
    for f, alpha in enumerate(alphas):
        alpha = float(alpha)
        if st is not None and st >= 1e-6:
            out[f] = (np.sin((1.0 - alpha) * theta) / st, np.sin(alpha * theta) / st)
        else:
            out[f] = (1.0 - alpha, alpha)
    return out


def slerp_combine(a, b, coef):
    """[F, *a.shape] float32 frames from float32 endpoints and [F, 2] float32 weights."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    coef = np.asarray(coef, np.float32)
    return np.stack([np.float32(wa) * a + np.float32(wb) * b for wa, wb in coef])


def slerp_frames(a, b, alphas):
    """The whole call for one pair: (frames [F, ...] float32, coef [F, 2] float32, sums [3] float64)."""
    sums = slerp_sums(a, b)
    coef = slerp_coef(sums, alphas)
    return slerp_combine(a, b, coef), coef, sums
