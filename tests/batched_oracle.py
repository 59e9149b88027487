"""The reference's batched formulation restated in float64 on top of the frame-by-frame oracle, and a helper that
concatenates frames into one batch.

A batch holds independent frames, each with its own cell (torch-sim's input: ``cell`` [F, 3, 3], ``pbc`` [F, 3],
``batch``, ``num_atoms``).  ``with_edge_vectors_`` takes the cell of an edge from ``batch[edge_index[0]]``
(nequip/nn/utils.py:96-106), and ``ForceStressOutput`` applies one symmetric displacement per frame to the positions
of that frame's atoms and to its cell, and divides each frame's virial by its own volume
(nequip/nn/grad_output.py:117-260).
"""
from __future__ import annotations

from typing import Dict, List

import torch

from oracle import model as omodel
from oracle import pair as opair


def concat_frames(frames: List[Dict[str, torch.Tensor]], pbcs=None) -> Dict[str, torch.Tensor]:
    """One batch from frames (CPU dicts with ``pos``, ``atom_types``, ``edge_index``, ``edge_cell_shift`` and ``cell``
    or none): atoms and edges concatenated with the edge indices offset by each frame's first atom, ``cell`` [F, 3, 3]
    (the identity for a frame without one), ``pbc`` [F, 3] (``pbcs``, or periodic when the frame has a cell),
    ``batch`` [N] and ``num_atoms`` [F]."""
    pos, types, ei, sh, cells, batch, counts = [], [], [], [], [], [], []
    off = 0
    for f, d in enumerate(frames):
        n = d["pos"].shape[0]
        pos.append(d["pos"].double())
        types.append(d["atom_types"].view(-1).long())
        ei.append(d["edge_index"].long() + off)
        sh.append(d["edge_cell_shift"].double() if "edge_cell_shift" in d
                  else torch.zeros((d["edge_index"].shape[1], 3), dtype=torch.float64))
        cells.append(d["cell"].double().view(3, 3) if d.get("cell") is not None else torch.eye(3, dtype=torch.float64))
        batch.append(torch.full((n,), f, dtype=torch.int64))
        counts.append(n)
        off += n
    if pbcs is None:
        pbcs = [[d.get("cell") is not None] * 3 for d in frames]
    return {
        "pos": torch.cat(pos),
        "atom_types": torch.cat(types),
        "edge_index": torch.cat(ei, 1),
        "edge_cell_shift": torch.cat(sh),
        "cell": torch.stack(cells),
        "pbc": torch.tensor(pbcs, dtype=torch.bool).view(-1, 3),
        "batch": torch.cat(batch),
        "num_atoms": torch.tensor(counts, dtype=torch.int64),
    }


def edge_vectors(pos, edge_index, cell, shift, batch):
    """Edge vectors of a batch: ``pos[j] - pos[i] + shift @ cell[batch[i]]``, i = ``edge_index[0]``."""
    vec = torch.index_select(pos, 0, edge_index[1]) - torch.index_select(pos, 0, edge_index[0])
    return vec + torch.sum(shift.view(-1, 3, 1) * cell[batch[edge_index[0]]], 1)


def energy_forces_stress(sd, cfg, data, model_dtype=torch.float64):
    """(per-frame energies [F, 1], per-atom energies [N, 1], forces [N, 3], stress [F, 3, 3], virial [F, 3, 3]) of a
    batch: a displacement ``disp_f`` per frame, symmetrised, moves ``pos_i -> pos_i (1 + sym_f)`` for the atoms of
    frame f and ``cell_f -> cell_f (1 + sym_f)``; virial_raw_f = dE/d(disp_f), stress_f = virial_raw_f / |det cell_f|,
    virial_f = -virial_raw_f.  The network (and ZBL when ``cfg`` has a pair potential) is the frame-by-frame oracle
    fed with the batch's edge vectors."""
    batch = data["batch"].view(-1).long()
    cell = data["cell"].double().view(-1, 3, 3)
    F = cell.shape[0]
    pos = data["pos"].detach().clone().double().requires_grad_(True)
    disp = torch.zeros((F, 3, 3), dtype=torch.float64, requires_grad=True)
    sym = 0.5 * (disp + disp.transpose(1, 2))
    pos_d = pos + torch.sum(pos.view(-1, 3, 1) * sym[batch], 1)
    cell_d = cell + torch.sum(cell.view(F, 3, 3, 1) * sym.view(F, 1, 3, 3), 2)
    vec = edge_vectors(pos_d, data["edge_index"], cell_d, data["edge_cell_shift"].double(), batch)
    inputs = {"pos": pos_d, "atom_types": data["atom_types"], "edge_index": data["edge_index"], "edge_vectors": vec,
              "batch": batch, "num_atoms": torch.ones(F, dtype=torch.int64)}
    energy = opair.energy if "pair_potential" in cfg else omodel.energy
    e_tot, e_atom = energy(sd, cfg, inputs, model_dtype)
    g, v = torch.autograd.grad([e_tot.sum()], [pos, disp])
    vol = torch.linalg.det(cell).abs().view(F, 1, 1)
    return e_tot.detach(), e_atom.detach(), -g, v / vol, -v
