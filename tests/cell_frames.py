"""Frames in general periodic cells (triclinic, left-handed, smaller than the cutoff, partly periodic) and a float64
brute-force neighbour list for any cell, shared by the cell tests.

``brute_list`` is the reference every list is compared with: it tries every image that can reach the cutoff, so it
does not share the cell-list code (bins, search ranges, bounding boxes) of ``ops.neighbor_list``.  It refuses frames
with a pair within 1e-10 relative of the cutoff, where two correct lists could disagree by rounding alone.
"""
from __future__ import annotations

import numpy as np
import torch

from nequip_b200 import data as D

#: shapes of the named cells (rows = lattice vectors, in units of the lattice length ``n_side * a``)
_TILTED = np.array([[1.0, 0.0, 0.0], [0.3, 1.0, 0.0], [-0.2, 0.15, 1.0]])  # LAMMPS-style tilts xy, xz, yz
CELL_SHAPES = {
    "cubic": np.eye(3),
    "tilted": _TILTED,
    # tilts of 0.5 and more of the length: not basis-reduced, the faces are far from the lattice vectors
    "skewed": np.array([[1.0, 0.0, 0.0], [0.6, 1.0, 0.0], [0.55, -0.5, 1.0]]),
    # tilted with rows 0 and 1 swapped: det < 0
    "left": _TILTED[[1, 0, 2]],
    # with n_side = 2 every perpendicular width is below r_max = 5: a neighbour appears under several shifts
    "small": np.array([[1.0, 0.0, 0.0], [0.16, 0.92, 0.0], [-0.07, 0.11, 0.96]]),
}


def pbc3(pbc):
    return (bool(pbc),) * 3 if isinstance(pbc, (bool, np.bool_)) else tuple(bool(b) for b in pbc)


def perp_widths(cell) -> np.ndarray:
    """Distance between opposite faces along each lattice direction: 1 / |column d of the inverse|."""
    return 1.0 / np.linalg.norm(np.linalg.inv(np.asarray(cell, dtype=np.float64)), axis=0)


def brute_list(pos, cell, pbc, r_max: float, max_pairs: int = 20_000_000):
    """Full neighbour list within ``r_max`` (float64, numpy) for any cell and per-direction periodicity: edge_index
    [2, E] int64 and shifts [E, 3] float64 with ``pos[j] - pos[i] + shift @ cell`` the edge vector, no self edge
    at zero shift, sorted by (i, j, shift) like the device list.  Atoms may lie outside the cell.

    Atoms are wrapped along the periodic directions, every image within ``ceil(r_max / perp_d) + 1`` cells is
    tried along periodic direction d (0 along open ones), and the shifts are expressed for the positions as given.
    Centres are processed in chunks of at most ``max_pairs`` (centre, neighbour, image) candidates."""
    pos = np.asarray(pos, dtype=np.float64)
    flags = np.array(pbc3(pbc))
    N = pos.shape[0]
    if cell is None:
        assert not flags.any(), "periodic directions need a cell"
        cell = np.eye(3)
    cell = np.asarray(cell, dtype=np.float64).reshape(3, 3)
    if np.count_nonzero(cell - np.diag(np.diagonal(cell))) == 0:
        frac = pos / np.diagonal(cell)  # as the host and device lists compute it for a diagonal cell
    else:
        frac = pos @ np.linalg.inv(cell)
    base = np.where(flags, np.floor(frac), 0.0)  # pos - base @ cell is wrapped along the periodic directions
    w = pos - base @ cell
    k = np.where(flags, np.ceil(r_max / perp_widths(cell)) + 1, 0).astype(int)
    imgs = np.array([(a, b, c) for a in range(-k[0], k[0] + 1) for b in range(-k[1], k[1] + 1)
                     for c in range(-k[2], k[2] + 1)], dtype=np.float64)
    # torch on the host only for its threads: elementwise float64 arithmetic, rounded as numpy would round it
    wt, off = torch.from_numpy(w), torch.from_numpy(imgs @ cell)
    home = torch.from_numpy(np.all(imgs == 0, axis=1))
    r2 = r_max * r_max
    chunk = max(1, max_pairs // max(1, N * len(imgs)))
    ii, jj, mm = [], [], []
    for s in range(0, N, chunk):
        c = torch.arange(s, min(N, s + chunk))
        vec = (wt[None, :, None, :] + off[None, None]) - wt[c, None, None, :]  # [centre, j, image, 3]
        d2 = (vec[..., 0] * vec[..., 0] + vec[..., 1] * vec[..., 1]) + vec[..., 2] * vec[..., 2]
        near = (d2 - r2).abs() < 1e-10 * r2
        assert not bool(near.any()), "a pair lies within 1e-10 relative of the cutoff: membership is ill-defined"
        ok = d2 < r2
        ok[torch.arange(c.numel()), c, :] &= ~home
        i, j, m = (t.numpy() for t in torch.nonzero(ok, as_tuple=True))
        ii.append(c.numpy()[i])
        jj.append(j)
        mm.append(m)
    i, j, m = np.concatenate(ii), np.concatenate(jj), np.concatenate(mm)
    sh = imgs[m] + base[i] - base[j]
    order = np.lexsort((sh[:, 2], sh[:, 1], sh[:, 0], j, i))
    return np.stack([i[order], j[order]]).astype(np.int64), sh[order]


def named_cell(name: str, n_side: int, kind: str = "li3po4") -> np.ndarray:
    """The named cell for ``n_side``^3 atoms at the density of preset ``kind``."""
    a = (1.0 / D.PRESETS[kind]["density"]) ** (1.0 / 3.0)
    return n_side * a * CELL_SHAPES[name]


def cell_frame(kind: str, n_side: int, cell, seed: int = 0, outside: bool = False, pbc=True, r_max: float = 5.0):
    """AtomicDataDict-shaped frame (CPU tensors, ``_meta`` as in ``data.make_system``) of ``n_side``^3 atoms in
    ``cell`` (a name of ``CELL_SHAPES`` or a [3, 3] array): the jittered lattice of ``data.jittered_lattice`` in
    fractional coordinates, mapped through the cell; types drawn as in ``make_system``; edges from ``brute_list``.

    ``outside=True`` moves each atom by a random integer combination (-2..3) of the periodic lattice vectors, so the
    lists need non-zero base shifts, and moves the whole frame back by half a lattice vector along each open
    direction, so that its atoms reach below fractional 0 there."""
    pr = D.PRESETS[kind]
    cell = named_cell(cell, n_side, kind) if isinstance(cell, str) else np.asarray(cell, dtype=np.float64)
    flags = np.array(pbc3(pbc))
    lat_pos, lat_cell = D.jittered_lattice(n_side, pr["density"], seed=seed)
    frac = lat_pos / np.diagonal(lat_cell)
    rng = np.random.default_rng(seed + 1)
    ratios = np.asarray(pr["ratios"], dtype=np.float64)
    types = rng.choice(len(ratios), size=frac.shape[0], p=ratios / ratios.sum())
    if outside:
        moves = np.random.default_rng(seed + 2).integers(-2, 4, size=frac.shape)
        frac = frac + np.where(flags, moves, 0) - np.where(flags, 0.0, 0.5)
    pos = frac @ cell
    ei, sh = brute_list(pos, cell, flags, r_max)
    return {
        "pos": torch.from_numpy(pos),
        "cell": torch.from_numpy(cell.copy()),
        "atom_types": torch.from_numpy(types.astype(np.int64)),
        "edge_index": torch.from_numpy(ei),
        "edge_cell_shift": torch.from_numpy(sh),
        "_meta": dict(kind=kind, type_names=list(pr["type_names"]), r_max=r_max,
                      avg_num_neighbors=float(ei.shape[1]) / pos.shape[0]),
    }
