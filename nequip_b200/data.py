"""Synthetic AtomicDataDict-shaped inputs (host side; numpy) for tests and bench.

No ASE / matscipy in this image, so structures and neighbour lists are generated
here.  The neighbour list follows the reference's contract
(nequip/data/_nl.py:102-152, "ijS" lists): a FULL list (both directions), no
self-edges at zero shift, ``edge_index[0]`` = centre atom, ``edge_index[1]`` =
neighbour, ``edge_cell_shift`` = integer lattice shifts such that
``r_ij = pos[j] - pos[i] + shift @ cell`` (nequip/nn/utils.py:86-118), sorted by
(centre, neighbour) like ``SortedNeighborListTransform``
(nequip/data/transforms/neighborlist.py:120-157).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

#: density (atoms / A^3), type ratios -- SURVEY.md section 8d
PRESETS = {
    "water": dict(density=0.100, type_names=("H", "O"), ratios=(2, 1)),
    "li3po4": dict(density=0.104, type_names=("Li", "P", "O"), ratios=(3, 1, 4)),
    "asi": dict(density=0.0489, type_names=("Si",), ratios=(1,)),
}


def jittered_lattice(n_side: int, density: float, jitter: float = 0.22, seed: int = 0):
    """n_side^3 atoms on a simple-cubic lattice (spacing from density), uniformly jittered.
    Returns (pos [N,3] f64, cell [3,3] f64).  Min distance >= (1 - 2*jitter*sqrt(3)) a > 0."""
    rng = np.random.default_rng(seed)
    a = (1.0 / density) ** (1.0 / 3.0)
    g = np.arange(n_side, dtype=np.float64)
    # x fastest within y within z: raster order keeps spatial neighbours close in index
    zz, yy, xx = np.meshgrid(g, g, g, indexing="ij")
    pos = np.stack([xx.ravel(), yy.ravel(), zz.ravel()], axis=1) + 0.5
    pos = (pos + rng.uniform(-jitter, jitter, size=pos.shape)) * a
    cell = np.eye(3) * (n_side * a)
    return pos, cell


def edge_type_rc2(atom_types, cutoffs, r_max: float) -> np.ndarray:
    """[T, T] float64 ``rc * rc`` of a per-edge-type cutoff table ``cutoffs[source, target]`` (0 < rc <= r_max), after
    checking the table and the types."""
    rc = np.asarray(cutoffs.detach().cpu() if torch.is_tensor(cutoffs) else cutoffs, dtype=np.float64)
    if rc.ndim != 2 or rc.shape[0] != rc.shape[1]:
        raise ValueError(f"cutoffs must be a [T, T] table, got shape {rc.shape}")
    if not (np.all(rc > 0) and np.all(rc <= r_max)):
        raise ValueError(f"cutoffs: every entry must satisfy 0 < rc <= r_max = {r_max}")
    t = np.asarray(atom_types).reshape(-1)
    if t.size and (t.min() < 0 or t.max() >= rc.shape[0]):
        raise ValueError(f"atom_types must lie in [0, {rc.shape[0]})")
    return rc * rc


def neighbor_list(pos: np.ndarray, cell: Optional[np.ndarray], r_max: float, pbc: bool = True, atom_types=None,
                  cutoffs=None):
    """Full neighbour list within r_max.  Orthorhombic cells only.  Returns
    (edge_index [2,E] int64, shifts [E,3] float64) sorted by (centre, neighbour).

    Per-edge-type cutoffs (nequip/data/transforms/neighborlist.py:9-117): ``cutoffs`` [T, T] (``rc[source, target]``)
    with ``atom_types`` [N] keeps the pair (i, j) when ``dist2 < rc[t_i, t_j]^2`` (``rc * rc`` in float64) instead of
    ``dist2 < r_max^2``, in both paths below.  A table of r_max everywhere gives the list without it."""
    N = pos.shape[0]
    thr = None  # [N, N] squared cutoff of each (centre, neighbour) pair, or None for r_max
    if cutoffs is not None:
        if atom_types is None:
            raise ValueError("cutoffs need atom_types")
        t = np.asarray(atom_types).reshape(-1).astype(np.int64)
        if t.size != N:
            raise ValueError(f"atom_types must hold {N} types")
        thr = edge_type_rc2(t, cutoffs, r_max)[t[:, None], t[None, :]]
    if not isinstance(pbc, (bool, np.bool_)):  # per-direction flags (mixed boundary conditions, e.g. a slab)
        flags = [bool(b) for b in pbc]
        if cell is not None and any(flags) and not all(flags):
            assert np.allclose(cell, np.diag(np.diag(cell))), "orthorhombic cells only"
            return _nl_bruteforce(pos, np.diag(cell).copy(), r_max, periodic=np.array(flags), thr=thr)
        pbc = all(flags)
    if cell is None or not pbc:
        L = None
    else:
        assert np.allclose(cell, np.diag(np.diag(cell))), "orthorhombic cells only"
        L = np.diag(cell).copy()
    if L is None or np.any(np.floor(L / r_max) < 3) or N < 64:
        return _nl_bruteforce(pos, L, r_max, thr=thr)
    nc = np.floor(L / r_max).astype(np.int64)
    frac = pos / L
    wrapped = frac - np.floor(frac)
    base_shift = -np.floor(frac)  # pos + base_shift*L is inside the box
    cidx = np.minimum((wrapped * nc).astype(np.int64), nc - 1)
    cid = (cidx[:, 2] * nc[1] + cidx[:, 1]) * nc[0] + cidx[:, 0]
    order = np.argsort(cid, kind="stable")
    counts = np.bincount(cid, minlength=int(nc.prod()))
    starts = np.concatenate([[0], np.cumsum(counts)])
    maxocc = int(counts.max())
    # padded table cell -> atom ids
    table = -np.ones((int(nc.prod()), maxocc), dtype=np.int64)
    rank = np.arange(N) - starts[cid[order]]
    table[cid[order], rank] = order
    wpos = wrapped * L
    ii_all, jj_all, sh_all = [], [], []
    chunk = max(1, 2_000_000 // (27 * maxocc))
    offs = np.array([(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)], dtype=np.int64)
    for s in range(0, N, chunk):
        sl = slice(s, min(N, s + chunk))
        ci = cidx[sl]  # [n,3]
        nb = ci[:, None, :] + offs[None, :, :]  # [n,27,3]
        img = np.floor_divide(nb, nc)  # -1,0,1 image of the neighbour cell
        nbw = nb - img * nc
        ncid = (nbw[..., 2] * nc[1] + nbw[..., 1]) * nc[0] + nbw[..., 0]  # [n,27]
        cand = table[ncid]  # [n,27,maxocc]
        valid = cand >= 0
        cj = np.where(valid, cand, 0)
        d = wpos[cj] + (img[:, :, None, :] * L) - wpos[sl][:, None, None, :]
        dist2 = (d * d).sum(-1)
        ai = np.broadcast_to(np.arange(sl.start, sl.stop)[:, None, None], cand.shape)
        ok = valid & (dist2 < (r_max * r_max if thr is None else thr[ai, cj]))
        ok &= ~((cj == ai) & (img == 0).all(-1)[:, :, None])
        i_sel = ai[ok]
        j_sel = cj[ok]
        img_sel = np.broadcast_to(img[:, :, None, :], cand.shape + (3,))[ok]
        # shift such that pos[j] - pos[i] + shift*L == wrapped difference
        sh = img_sel + base_shift[j_sel] - base_shift[i_sel]
        ii_all.append(i_sel)
        jj_all.append(j_sel)
        sh_all.append(sh)
    ii = np.concatenate(ii_all)
    jj = np.concatenate(jj_all)
    sh = np.concatenate(sh_all).astype(np.float64)
    o = np.lexsort((jj, ii))
    return np.stack([ii[o], jj[o]]).astype(np.int64), sh[o]


def _nl_bruteforce(pos, L, r_max, periodic=None, thr=None):
    """``periodic`` (optional bool[3]): directions without periodic images (their cell length is ignored).
    ``thr`` (optional [N, N]): squared cutoff of each (centre, neighbour) pair in place of r_max^2."""
    r2 = r_max * r_max if thr is None else thr
    if L is not None and periodic is not None:
        per = np.asarray(periodic, dtype=bool)
        Lp = np.where(per, L, 1.0)
        cells = np.where(per, np.floor(pos / Lp), 0.0)  # wrap along the periodic directions only
        w = pos - cells * Lp
        reps = np.where(per, np.ceil(r_max / Lp), 0).astype(int)
        rng = [np.arange(-r, r + 1) for r in reps]
        shifts = np.array([(a, b, c) for a in rng[0] for b in rng[1] for c in rng[2]], dtype=np.float64)
        ii, jj, ss = [], [], []
        for s in shifts:
            d = w[None, :, :] + s * Lp - w[:, None, :]
            ok = (d * d).sum(-1) < r2
            if not np.any(s):
                ok &= ~np.eye(pos.shape[0], dtype=bool)
            i, j = np.nonzero(ok)
            ii.append(i)
            jj.append(j)
            ss.append(np.broadcast_to(s, (i.size, 3)))
        ii, jj, ss = np.concatenate(ii), np.concatenate(jj), np.concatenate(ss).astype(np.float64)
        o = np.lexsort((jj, ii))
        ei = np.stack([ii[o], jj[o]]).astype(np.int64)
        return ei, ss[o] + cells[ei[0]] - cells[ei[1]]
    if L is not None:
        cells = np.floor(pos / L)
        if np.any(cells != 0):
            # atoms outside the home cell (unwrapped trajectories, nequip/utils/unittests/model_tests_basic.py:326-383):
            # search among the wrapped images, then express the shifts for the positions as given --
            # pos[j] - pos[i] + shift * L is the same vector as for the wrapped atoms
            ei, sh = _nl_bruteforce(pos - cells * L, L, r_max, thr=thr)
            return ei, sh + cells[ei[0]] - cells[ei[1]]
    N = pos.shape[0]
    if L is None:
        shifts = np.zeros((1, 3))
    else:
        reps = np.ceil(r_max / L).astype(int)
        rng = [np.arange(-r, r + 1) for r in reps]
        shifts = np.array([(a, b, c) for a in rng[0] for b in rng[1] for c in rng[2]], dtype=np.float64)
    ii, jj, ss = [], [], []
    for s in shifts:
        off = (s * L) if L is not None else 0.0
        d = pos[None, :, :] + off - pos[:, None, :]
        dist2 = (d * d).sum(-1)
        ok = dist2 < r2
        if not np.any(s):
            ok &= ~np.eye(N, dtype=bool)
        i, j = np.nonzero(ok)
        ii.append(i)
        jj.append(j)
        ss.append(np.broadcast_to(s, (i.size, 3)))
    ii, jj, ss = np.concatenate(ii), np.concatenate(jj), np.concatenate(ss)
    o = np.lexsort((jj, ii))
    return np.stack([ii[o], jj[o]]).astype(np.int64), ss[o].astype(np.float64)


def make_system(kind: str, n_side: int, r_max: float = 5.0, seed: int = 0) -> Dict[str, torch.Tensor]:
    """AtomicDataDict-shaped dict (CPU tensors): pos f64, cell f64 [3,3], atom_types i64,
    edge_index i64 [2,E], edge_cell_shift f64 [E,3]; plus python metadata under '_meta'."""
    pr = PRESETS[kind]
    pos, cell = jittered_lattice(n_side, pr["density"], seed=seed)
    rng = np.random.default_rng(seed + 1)
    ratios = np.asarray(pr["ratios"], dtype=np.float64)
    types = rng.choice(len(ratios), size=pos.shape[0], p=ratios / ratios.sum())
    ei, sh = neighbor_list(pos, cell, r_max)
    return {
        "pos": torch.from_numpy(pos),
        "cell": torch.from_numpy(cell),
        "atom_types": torch.from_numpy(types.astype(np.int64)),
        "edge_index": torch.from_numpy(ei),
        "edge_cell_shift": torch.from_numpy(sh),
        "_meta": dict(kind=kind, type_names=list(pr["type_names"]), r_max=r_max,
                      avg_num_neighbors=float(ei.shape[1]) / pos.shape[0]),
    }


def replicate_frame(data: Dict[str, torch.Tensor], copies: int, r_max: float = 5.0, axis: int = 0) -> Dict[str, torch.Tensor]:
    """``copies``-fold periodic supercell of an orthorhombic frame along ``axis``: atom ``c * n + b`` is base atom ``b``
    shifted by ``c`` cell lengths, the cell grows ``copies`` times along ``axis``, the neighbour list is rebuilt.
    By periodicity every copy of an atom has the energy and force of the base atom -- the property bench.py uses to
    check a frame sharded over N GPUs against the unsharded base frame (weak scaling = the N-fold supercell)."""
    pos = data["pos"].double().numpy()
    cell = data["cell"].double().numpy().reshape(3, 3)
    if copies < 1 or np.abs(cell - np.diag(np.diagonal(cell))).max() > 0:
        raise ValueError("replicate_frame: needs copies >= 1 and an orthorhombic (diagonal) cell")
    n = pos.shape[0]
    step = np.zeros(3)
    step[axis] = cell[axis, axis]
    big = np.concatenate([pos + c * step for c in range(copies)], 0)
    big_cell = cell.copy()
    big_cell[axis, axis] *= copies
    ei, sh = neighbor_list(big, big_cell, r_max)
    return {
        "pos": torch.from_numpy(big),
        "cell": torch.from_numpy(big_cell),
        "atom_types": data["atom_types"].repeat(copies),
        "edge_index": torch.from_numpy(ei),
        "edge_cell_shift": torch.from_numpy(sh),
    }


def oscillating_positions(pos0: torch.Tensor, t: int, period: int = 50, amplitude: float = 0.2, seed: int = 0) -> torch.Tensor:
    """Step ``t`` of a bounded MD-like trajectory: ``pos0 + amplitude * sin(2 pi t / period + phi)``, one seeded phase
    per atom and direction.  Edges cross the cutoff at most steps, and unlike a trajectory integrated with a
    random-weight model's forces, it stays physical for any number of steps."""
    g = torch.Generator().manual_seed(seed)
    phi = (2 * np.pi) * torch.rand(tuple(pos0.shape), generator=g, dtype=torch.float64).to(pos0.device)
    return pos0 + amplitude * torch.sin(2 * np.pi * t / period + phi)


def oscillating_strain(t: int, period: int = 50, diagonal: float = 0.02, shear: float = 0.03) -> torch.Tensor:
    """``I + eps(t)`` [3,3] float64 of a bounded variable-cell trajectory: ``eps`` is symmetric, its diagonal
    oscillates with amplitude ``diagonal`` and its off-diagonal pairs with amplitude ``shear``, each with its own fixed
    phase.  Step t of the trajectory is ``cell0 @ S`` and ``oscillating_positions(pos0, t) @ S`` (rows = vectors), so
    the cell is triclinic at most steps.  The diagonal phases are pi/3 apart, so the trace of eps swings by
    2 * diagonal: the volume swings by about +-4 % for diagonal = 0.02 (phases 2 pi/3 apart would keep it fixed)."""
    w = 2 * np.pi * t / period
    eps = np.zeros((3, 3))
    for d in range(3):
        eps[d, d] = diagonal * np.sin(w + np.pi * d / 3)
    for k, (a, b) in enumerate(((0, 1), (0, 2), (1, 2))):
        eps[a, b] = eps[b, a] = shear * np.sin(w + np.pi / 4 + 2 * np.pi * k / 3)
    return torch.from_numpy(np.eye(3) + eps)


def to_device(data: Dict, device) -> Dict:
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in data.items()}
