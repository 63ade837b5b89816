"""ORACLE (test infrastructure only -- never imported by the product path).

float64 restatement of progressive distillation (Salimans & Ho, ICLR 2022) on the halving DDIM grid, written from the
paper's formulas rather than from the solver's step form:

  * grid      l_i = round((N - 1)(1 - i / K)), halves rounded up, in exact rational arithmetic
  * DDIM      x0 = (z_s - sigma_s eps) / alpha_s;  z_t = alpha_t x0 + sigma_t eps
  * target    eps~ = (z_e - (alpha_e / alpha_s) z_s) / (sigma_e - alpha_e sigma_s / alpha_s), the eps whose DDIM step
              s -> e from z_s lands on z_e
  * rows      mdb_distill_row's 13 columns for a teacher grid of K_T steps

`abar` is alphas_cumprod as a float64 array (the product computes it in float32 and widens it, so the oracle takes it
as given).
"""
from fractions import Fraction
import math

import numpy as np


def grid(N, K):
    return [math.floor(Fraction((N - 1) * (K - i), K) + Fraction(1, 2)) for i in range(K + 1)]


def alpha_sigma(abar, n):
    return math.sqrt(abar[n]), math.sqrt(1.0 - abar[n])


def ddim_step(abar, s, t, z, eps):
    a_s, s_s = alpha_sigma(abar, s)
    a_t, s_t = alpha_sigma(abar, t)
    x0 = (z - s_s * eps) / a_s
    return a_t * x0 + s_t * eps


def target(abar, s, e, z_s, z_e):
    a_s, s_s = alpha_sigma(abar, s)
    a_e, s_e = alpha_sigma(abar, e)
    return (z_e - (a_e / a_s) * z_s) / (s_e - a_e * s_s / a_s)


def rows(abar, K_T):
    """[K_T / 2, 13]: labels s, m, e; (sigma, 1 / alpha, c_x, c_0) of the DDIM steps s -> m and m -> e written as
    z' = c_x z + c_0 x0; r = alpha_e / alpha_s; 1 / (sigma_e - alpha_e sigma_s / alpha_s)."""
    N = len(abar)
    l = grid(N, K_T)
    out = []
    for i in range(K_T // 2):
        s, m, e = l[2 * i:2 * i + 3]
        row = [s, m, e]
        for a, b in ((s, m), (m, e)):
            a_a, s_a = alpha_sigma(abar, a)
            a_b, s_b = alpha_sigma(abar, b)
            # alpha_b x0 + sigma_b (z - alpha_a x0) / sigma_a
            row += [s_a, 1.0 / a_a, s_b / s_a, a_b - s_b * a_a / s_a]
        a_s, s_s = alpha_sigma(abar, s)
        a_e, s_e = alpha_sigma(abar, e)
        row += [a_e / a_s, 1.0 / (s_e - a_e * s_s / a_s)]
        out.append(row)
    return np.array(out, dtype=np.float64)


def teacher_target(abar, s, m, e, z_s, eps_s, eps_m):
    """Two teacher DDIM steps s -> m -> e with the given predictions, then the target: (z_m, z_e, eps~)."""
    z_m = ddim_step(abar, s, m, z_s, eps_s)
    z_e = ddim_step(abar, m, e, z_m, eps_m)
    return z_m, z_e, target(abar, s, e, z_s, z_e)
