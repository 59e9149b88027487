"""Float64 numpy restatement of the device neighbour list's open directions: the bounding box and grid that
``nqb_nl_bbox`` writes into the parameter block and the bins ``k_nl_bin`` then gives each atom.

Every operation is one IEEE-rounded float64 operation in the kernels' order, so the results are bitwise those of the
device: fractional coordinates ``x / diag`` for an orthorhombic cell, ``(x inv[0, d] + y inv[1, d]) + z inv[2, d]``
otherwise; ``width = max(fmax - fmin, 1e-9) (1 + 1e-9)`` (a NaN difference takes 1e-9);
``nb = min(cap, max(1, floor(perp width / r_max)))``.
"""
from __future__ import annotations

import math

import numpy as np


def bin_cap(n_atoms: int) -> int:
    """Most bins per direction: round((4 N)^(1/3)), at least 1 (``ops._nl_bin_cap``)."""
    return max(1, int(round((4 * max(n_atoms, 1)) ** (1.0 / 3.0))))


def frac_coords(pos, cell) -> np.ndarray:
    pos = np.asarray(pos, dtype=np.float64)
    cell = np.eye(3) if cell is None else np.asarray(cell, dtype=np.float64).reshape(3, 3)
    if np.count_nonzero(cell - np.diag(np.diagonal(cell))) == 0:
        return pos / np.diagonal(cell)
    inv = np.linalg.inv(cell)
    return (pos[:, 0:1] * inv[0] + pos[:, 1:2] * inv[1]) + pos[:, 2:3] * inv[2]


def open_grid(fmin: float, fmax: float, perp: float, r_max: float, cap: int):
    """(lo, width, nb) of one open direction from the min / max of its fractional coordinates."""
    w = fmax - fmin
    w = w if w > 1e-9 else 1e-9
    w = w * (1 + 1e-9)
    t = math.floor(perp * w / r_max) if math.isfinite(perp * w / r_max) else perp * w / r_max
    nb = (int(t) if t < cap else cap) if t >= 1.0 else 1
    return fmin, w, nb


def bbox(frac: np.ndarray):
    """Per-direction min / max skipping NaN; (+inf, -inf) for a direction without any number."""
    fin = ~np.isnan(frac)
    lo = np.where(fin, frac, np.inf).min(0)
    hi = np.where(fin, frac, -np.inf).max(0)
    return lo, hi


def bins(pos, cell, pbc, r_max: float, periodic_nb) -> np.ndarray:
    """cidx [N, 3] of ``k_nl_bin`` after ``nqb_nl_bbox``: ``periodic_nb`` bins along the periodic directions (the
    plan's host grid), the device grid over the bounding box along the open ones."""
    frac = frac_coords(pos, cell)
    c = np.eye(3) if cell is None else np.asarray(cell, dtype=np.float64).reshape(3, 3)
    perp = 1.0 / np.linalg.norm(np.linalg.inv(c), axis=0)
    cap = bin_cap(frac.shape[0])
    lo, hi = bbox(frac)
    out = np.zeros(frac.shape, dtype=np.int64)
    for d in range(3):
        if pbc[d]:
            nb = int(periodic_nb[d])
            w = frac[:, d] + (-np.floor(frac[:, d]))
            q = np.trunc(w * nb)
            out[:, d] = np.minimum(q, nb - 1).astype(np.int64)
        else:
            l0, width, nb = open_grid(lo[d], hi[d], perp[d], r_max, cap)
            q = np.floor(((frac[:, d] - l0) / width) * nb)
            q = np.nan_to_num(q, nan=0.0)
            out[:, d] = np.clip(q, 0, nb - 1).astype(np.int64)
    return out
