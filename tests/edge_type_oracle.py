"""Per-edge-type cutoffs for the float64 oracles and the brute-force list (TEST INFRASTRUCTURE ONLY).

With ``per_edge_type_cutoff`` the reference normalises each edge length by its own type pair's cutoff
(nequip/nn/embedding/_edge.py:65-80): ``x_e = r_e * rmax_recip[T * t_src + t_tgt]`` with ``t_src`` the type of
``edge_index[0, e]`` (the centre).  The Bessel prefactor keeps the global ``r_max`` (model/nequip_models.py:318-322) and
the ZBL envelope reads the same ``x_e`` (nn/pair_potential.py:374), while the ZBL physics keeps ``r``.

``per_edge_cutoffs(recip_e)`` is a context manager under which ``oracle.model`` (and so ``oracle.pair`` and
``preset_oracle``, which call it) evaluate exactly that: the radial embedding and the ZBL per-atom energy are restated
below with ``x_e = r_e * recip_e`` in place of ``r_e * (1 / r_max)``, everything else of the oracles is unchanged.
``recip_e`` [E, 1] belongs to the one edge list evaluated inside the block (``edge_recip``).  It shares no code with
the product.
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch

from cell_frames import brute_list
from oracle import model as om
from oracle import pair as opair

#: the reference's test configuration (nequip/utils/unittests/minimal_aspirin.yaml:4-13), types [C, O, H], r_max 5
ASPIRIN_TYPES = ["C", "O", "H"]
ASPIRIN_CUTOFFS = {"H": 2.0, "C": {"H": 4.0, "C": 3.5, "O": 3.7}, "O": 3.9}
ASPIRIN_TABLE = [[3.5, 3.7, 4.0], [3.9, 3.9, 3.9], [2.0, 2.0, 2.0]]  # rc[source, target], written out by hand


def edge_recip(types: torch.Tensor, edge_index: torch.Tensor, table) -> torch.Tensor:
    """[E, 1] float64: ``1 / rc[type(edge_index[0, e]), type(edge_index[1, e])]`` (the reciprocal in float64, as the
    reference's ``_rmax_recip``)."""
    table = torch.as_tensor(table, dtype=torch.float64)
    T = table.shape[0]
    recip = table.reciprocal().reshape(-1)
    t = types.view(-1).long()
    return recip[T * t[edge_index[0].long()] + t[edge_index[1].long()]].view(-1, 1)


@contextlib.contextmanager
def per_edge_cutoffs(recip_e: torch.Tensor):
    """Inside the block the oracles normalise edge e's length by ``recip_e[e]`` (see the module docstring)."""
    recip_e = recip_e.view(-1, 1).to(torch.float64)

    def radial_embedding(r, r_max, num_bessels, p, model_dtype):
        x = r.view(-1, 1) * recip_e
        bw = torch.linspace(1.0, num_bessels, num_bessels, dtype=torch.float64).unsqueeze(0)
        bessel = (torch.sinc(x * bw) * bw).to(model_dtype)
        cutoff = om.polynomial_cutoff(x, p).to(model_dtype)
        return ((2 * math.pi) / (r_max * r_max)) * (bessel * cutoff)

    def zbl_atom_energy(atomic_numbers, qqr2exesquare, p, r_max, vec, atom_types, edge_index, num_nodes, model_dtype):
        r = vec.square().sum(1).sqrt()
        eng = opair.zbl_edge_energy(atomic_numbers.to(model_dtype), r, atom_types, edge_index, qqr2exesquare)
        eng = eng.unsqueeze(-1) * om.polynomial_cutoff(r.view(-1, 1) * recip_e, p).to(model_dtype)
        return torch.zeros((num_nodes, 1), dtype=eng.dtype, device=eng.device).index_add(0, edge_index[0], eng)

    saved = om.radial_embedding, opair.zbl_atom_energy
    om.radial_embedding, opair.zbl_atom_energy = radial_embedding, zbl_atom_energy
    try:
        yield
    finally:
        om.radial_embedding, opair.zbl_atom_energy = saved


def pruned_brute_list(pos, cell, pbc, r_max: float, types, table):
    """``brute_list`` within ``r_max``, filtered by ``d2 < rc[t_i, t_j]^2`` (d2 of ``pos[j] - pos[i] + shift @ cell``).
    Refuses frames with a pair within 1e-10 relative of its rc, where two correct lists could disagree by rounding."""
    pos = np.asarray(pos, dtype=np.float64)
    ei, sh = brute_list(pos, cell, pbc, r_max)
    c = np.eye(3) if cell is None else np.asarray(cell, dtype=np.float64).reshape(3, 3)
    vec = pos[ei[1]] - pos[ei[0]] + sh @ c
    d2 = (vec * vec).sum(1)
    t = np.asarray(types).reshape(-1)
    rc2 = np.square(np.asarray(table, dtype=np.float64))[t[ei[0]], t[ei[1]]]
    assert not np.any(np.abs(d2 - rc2) < 1e-10 * rc2), "a pair lies within 1e-10 relative of its cutoff"
    keep = d2 < rc2
    return ei[:, keep], sh[keep]


def random_table(T: int, r_max: float, seed: int) -> np.ndarray:
    """[T, T] asymmetric table with entries in [0.55, 1] * r_max, a quarter of them exactly r_max."""
    rng = np.random.default_rng(seed)
    tab = r_max * rng.uniform(0.55, 1.0, size=(T, T))
    tab[rng.random((T, T)) < 0.25] = r_max
    return tab
