"""Pins oracle/interp_oracle.py against the UNMODIFIED reference `slerp` (lib/diffusion/evaler.py:63-71) and writes
tests/golden/slerp_reference.npz.

Run in the authoring container only (needs the reference tree; its import goes through oracle/make_golden.py):

    python oracle/make_interp_golden.py

Inputs: 3 pairs of [4, 16, 16, 16] float32 endpoints drawn from numpy's default_rng(seed) and rounded to float16 values
(so the file stores them exactly in half the bytes); pair 1's second endpoint is zero on x-slabs 4..11. Each pair is
slerped into 8 frames, alpha = f / 7, by the reference in float32 on the CPU. Stored: the seeds, the endpoints (float16),
the alphas, the reference's angle per pair, and every frame at the elements `SUBSET` selects (every 4th element of the
flattened grid), which keeps the file small; the reference computes its angle over the whole tensor.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import interp_oracle  # noqa: E402
from oracle.make_golden import GOLD, import_reference  # noqa: E402

SEEDS = (101, 202, 303)
SHAPE = (4, 16, 16, 16)
FRAMES = 8
STRIDE = 4


def endpoints(seed, pair):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(SHAPE).astype(np.float16)
    b = rng.standard_normal(SHAPE).astype(np.float16)
    if pair == 1:
        b[:, 4:12] = 0
    return a, b


def main():
    import_reference()
    from lib.diffusion.evaler import slerp
    alphas = np.array([f / float(FRAMES - 1) for f in range(FRAMES)])
    za, zb, frames, thetas = [], [], [], []
    worst = 0.0
    for p, seed in enumerate(SEEDS):
        a16, b16 = endpoints(seed, p)
        a, b = torch.from_numpy(a16.astype(np.float32)), torch.from_numpy(b16.astype(np.float32))
        ref = torch.stack([slerp(a, b, f / float(FRAMES - 1)) for f in range(FRAMES)]).numpy()
        theta = torch.acos(torch.sum(a * b) / (torch.norm(a) * torch.norm(b))).item()
        got, _, _ = interp_oracle.slerp_frames(a.numpy(), b.numpy(), alphas)
        err = np.abs(got - ref).max() / np.abs(ref).max()
        print(f"pair {p}: theta {np.degrees(theta):.4f} deg, oracle vs reference {err:.3e} of max |frame|")
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[-1], ref[-1])
        worst = max(worst, err)
        za.append(a16)
        zb.append(b16)
        frames.append(ref.reshape(FRAMES, -1)[:, ::STRIDE])
        thetas.append(theta)
    assert worst <= 2.5e-7, worst
    path = os.path.join(GOLD, "slerp_reference.npz")
    np.savez_compressed(path, seeds=np.array(SEEDS), za=np.stack(za), zb=np.stack(zb), alphas=alphas,
                        theta=np.array(thetas), stride=np.array(STRIDE), frames=np.stack(frames).astype(np.float32))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
