"""ORACLE (test infrastructure only): the Earth Mover's distance of geometry/pointcloud.py's `emd_matrix`.

EMD(X, Y) = min over bijections pi of (1/N) sum_i |x_i - y_pi(i)| (Euclidean, not squared), for clouds of equal size N.

* `emd_exact`: the ground truth, an fp64 cost matrix solved by `scipy.optimize.linear_sum_assignment`.
* `emd_auction`: a float32 numpy restatement of the device kernel (csrc/emd.cu): the same epsilon schedule, the same cost
  and bid arithmetic (each float32 operation rounds, as the kernel's `__fadd_rn` / `__fmul_rn` do) and the same tie rules,
  with vectorised Jacobi rounds. When it agrees with the device to 1e-12, both made the same decisions.
* `metrics`: MMD / COV / 1-NNA from three distance matrices, keyed by a suffix ("cd" or "emd").
"""
import numpy as np
from scipy.optimize import linear_sum_assignment

from . import pc_metrics_oracle as pco

EPS_FACTOR = 5            # epsilon divides by this between scaling phases
START_FRACTION = 0.25     # the first phase's epsilon, as a share of C_max
FLOOR = 2.0 ** -18        # eps must be at least FLOOR * C_max (fp32 prices resolve it)
MARGIN = 2.0 ** -19       # the last phase runs at eps - MARGIN * C_max, which absorbs the bids' fp32 rounding
MAX_ROUNDS = 1 << 18      # rounds per pair before the kernel gives up (NaN entry, +inf gap)


def _check(x, y):
    if x.ndim != 2 or x.shape[1] != 3 or y.ndim != 2 or y.shape[1] != 3:
        raise ValueError("clouds must be [N, 3]")
    if x.shape[0] != y.shape[0]:
        raise ValueError(f"EMD needs clouds of equal size, got {x.shape[0]} and {y.shape[0]}")
    if x.shape[0] < 1:
        raise ValueError("clouds need at least one point")


def emd_exact(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    _check(x, y)
    c = np.sqrt(((x[:, None, :] - y[None, :, :]) ** 2).sum(-1))
    r, k = linear_sum_assignment(c)
    return float(c[r, k].sum() / x.shape[0])


def costs32(x, y):
    """c_ij = sqrt((dx*dx + dy*dy) + dz*dz), every operation rounded to float32."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    d = [x[:, None, k] - y[None, :, k] for k in range(3)]
    return np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def c_max(x, y):
    """Diagonal of the joint bounding box, in float32."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    e = np.maximum(x.max(0), y.max(0)) - np.minimum(x.min(0), y.min(0))
    return np.float32(np.sqrt((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2]))


def eps_schedule(cmax, eps):
    """The phases' epsilons: C_max / 4, divided by EPS_FACTOR while above the last one, which is eps - MARGIN * C_max."""
    f32 = np.float32
    eps = f32(eps)
    if not eps >= f32(cmax * f32(FLOOR)):
        raise ValueError(f"eps = {float(eps):.3g} is below what fp32 prices resolve at this scale "
                         f"({FLOOR:.3g} x C_max = {float(cmax * f32(FLOOR)):.3g})")
    last = f32(eps - f32(cmax * f32(MARGIN)))
    out, e = [], f32(cmax * f32(START_FRACTION))
    while e > last:
        out.append(e)
        e = f32(e / f32(EPS_FACTOR))
    out.append(last)
    return out


def emd_auction(x, y, eps=1e-5, max_rounds=MAX_ROUNDS):
    """The kernel's algorithm -> (emd, certified gap, scan elements). The scan elements are the cost evaluations the kernel
    makes: sum over rounds of (unassigned bidders x N), plus N^2 for the dual bound."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    _check(x, y)
    N = x.shape[0]
    c = costs32(x, y)
    price = np.zeros(N, np.float32)
    rounds = scan = 0
    rows = np.arange(N)
    for e in eps_schedule(c_max(x, y), eps):
        price = price - price.min()
        owner = np.full(N, -1, np.int64)   # object -> bidder
        asg = np.full(N, -1, np.int64)     # bidder -> object
        while True:
            U = np.flatnonzero(asg < 0)
            if U.size == 0:
                break
            if rounds >= max_rounds:
                return float("nan"), float("inf"), scan
            rounds += 1
            scan += U.size * N
            v = c[U] + price[None, :]
            jb = v.argmin(axis=1)                      # lowest j among equal values
            r = rows[:U.size]
            best = v[r, jb]
            if N > 1:
                v[r, jb] = np.inf
                second = v.min(axis=1)
            else:
                second = best
            bid = (price[jb] + (second - best)) + e
            # per object: the highest bid, ties to the lowest bidder
            order = np.lexsort((U, -bid, jb))
            first = np.r_[True, jb[order][1:] != jb[order][:-1]]
            win = order[first]
            J, I = jb[win], U[win]
            prev = owner[J]
            asg[prev[prev >= 0]] = -1
            owner[J] = I
            asg[I] = J
            price[J] = bid[win]
    scan += N * N
    emd = c[owner, np.arange(N)].astype(np.float64).sum() / N
    lb = ((c.astype(np.float64) + price.astype(np.float64)[None, :]).min(axis=1).sum() - price.astype(np.float64).sum()) / N
    return float(emd), float(emd - lb), scan


def emd_matrix(A, B=None, eps=1e-5):
    """(emd, gap) float64 [nA, nB] from emd_auction; B None: the self matrix (i < j computed and mirrored, diagonal 0)."""
    self_ = B is None
    B = A if self_ else B
    emd = np.zeros((len(A), len(B)))
    gap = np.zeros((len(A), len(B)))
    for i in range(len(A)):
        for j in range(len(B)):
            if self_ and j <= i:
                continue
            emd[i, j], gap[i, j], _ = emd_auction(A[i], B[j], eps)
            if self_:
                emd[j, i], gap[j, i] = emd[i, j], gap[i, j]
    return emd, gap


def emd_exact_matrix(A, B=None):
    self_ = B is None
    B = A if self_ else B
    return np.array([[0.0 if self_ and i == j else emd_exact(a, b) for j, b in enumerate(B)] for i, a in enumerate(A)])


def metrics(d_gr, d_gg, d_rr, suffix="cd"):
    """pc_metrics_oracle.metrics (loop by loop, lowest-index ties) with its keys renamed to the given distance."""
    return {k.replace("_cd", "_" + suffix): v for k, v in pco.metrics(d_gr, d_gg, d_rr).items()}
