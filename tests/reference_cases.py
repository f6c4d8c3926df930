"""Deterministic inputs of the host-side tests that compare with the reference's own classes.  The tests and the
generator of their golden data (tests/golden/make_reference_golden.py) both build their inputs here."""

import hashlib

import numpy as np

from tests import fixtures as fx

WS0 = (2, 6, 12)
WINDOW_CHUNKS = 4
REGRID_RES = (5.0, 11.25, 7.3)


def sample(v):
    """The fixed sub-grid of a field that the golden files store: every 5th latitude row, every 9th longitude."""
    return v[..., ::5, ::9]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def batch_case():
    """`tiny_air` on a 16 x 30 grid with 13 levels: one latitude row too many for patch size 3."""
    return fx.make_batch(fx.CONFIGS["tiny_air"], 16, 30, levels=fx.LEVELS13, b=1)


def regrid_case():
    return fx.make_batch(fx.CONFIGS["tiny"], 17, 32, levels=fx.LEVELS4, b=2)


def random_geometries(n, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n):
        res = (int(rng.integers(1, 7)), int(rng.integers(1, 41)), int(rng.integers(1, 61)))
        out.append((res, bool(rng.integers(0, 2)), bool(rng.integers(0, 2))))
    return out


def window_geometries(chunk):
    return random_geometries(30, 200 + chunk)
