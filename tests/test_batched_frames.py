"""Batches of frames with per-frame cells, on the host: the float64 batched formulation (``batched_oracle``) against
the oracle run frame by frame, and the argument checks of the batched neighbour list."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from nequip_b200 import ops
from nequip_b200.nn.model import NequIPEnergyModel
from oracle import model as omodel
from oracle import pair as opair

from batched_oracle import concat_frames, edge_vectors, energy_forces_stress
from cell_frames import cell_frame

R_MAX = 5.0
ZBL = {"units": "metal", "chemical_species": ["Li", "P", "O"]}


def _frames():
    """A cubic, a tilted, a left-handed and a small cell (each with atoms outside the cell) and a slab."""
    out = [cell_frame("li3po4", 2, name, seed=s, outside=True) for s, name in enumerate(["cubic", "tilted", "left"])]
    out.append(cell_frame("li3po4", 2, "small", seed=5))
    out.append(cell_frame("li3po4", 2, "skewed", seed=6, pbc=(True, True, False)))
    pbcs = [[True] * 3] * 4 + [[True, True, False]]
    meta = out[0]["_meta"]
    return [{k: v for k, v in d.items() if k != "_meta"} for d in out], pbcs, meta


@pytest.mark.parametrize("zbl", [False, True], ids=["plain", "zbl"])
def test_batched_oracle_matches_frame_by_frame(zbl):
    frames, pbcs, meta = _frames()
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=2, num_layers=2, num_features=8,
                              model_dtype=torch.float64, avg_num_neighbors=meta["avg_num_neighbors"],
                              pair_potential=ZBL if zbl else None, seed=3)
    sd, cfg = model.state_dict(), model.config
    single = opair.energy_forces_stress if zbl else omodel.energy_forces_stress
    batch = concat_frames(frames, pbcs)
    e, e_atom, f, s, v = energy_forces_stress(sd, cfg, batch, torch.float64)
    assert e.shape == (len(frames), 1) and s.shape == v.shape == (len(frames), 3, 3)
    off = 0
    for k, d in enumerate(frames):
        n = d["pos"].shape[0]
        ek, fk, sk, vk = single(sd, cfg, d, torch.float64)
        _ek, ea = (opair.energy if zbl else omodel.energy)(sd, cfg, d, torch.float64)
        scale = float(fk.abs().max())
        assert abs(float(e[k, 0]) - float(ek)) <= 1e-12 * max(1.0, abs(float(ek)))
        assert torch.allclose(e_atom[off:off + n], ea.detach(), rtol=0, atol=1e-12)
        assert torch.allclose(f[off:off + n], fk, rtol=0, atol=1e-12 * max(1.0, scale))
        assert torch.allclose(s[k], sk[0], rtol=0, atol=1e-12 * max(1.0, float(sk.abs().max())))
        assert torch.allclose(v[k], vk[0], rtol=0, atol=1e-12 * max(1.0, float(vk.abs().max())))
        off += n


def test_batched_oracle_keeps_frames_apart():
    """The gradient of frame 0's energy is exactly zero on every other frame's atoms."""
    frames, pbcs, meta = _frames()
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=1, num_layers=2, num_features=8,
                              model_dtype=torch.float64, seed=4)
    batch = concat_frames(frames, pbcs)
    pos = batch["pos"].clone().requires_grad_(True)
    vec = edge_vectors(pos, batch["edge_index"], batch["cell"], batch["edge_cell_shift"], batch["batch"])
    e, _ = omodel.energy(model.state_dict(), model.config,
                         {"pos": pos, "atom_types": batch["atom_types"], "edge_index": batch["edge_index"],
                          "edge_vectors": vec, "batch": batch["batch"], "num_atoms": batch["num_atoms"]},
                         torch.float64)
    (g,) = torch.autograd.grad([e[0, 0]], [pos])
    n0 = frames[0]["pos"].shape[0]
    assert bool(g[:n0].abs().max() > 0)
    assert bool((g[n0:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# argument checks of ops.neighbor_list(..., batch=) -- raised on the host, before any device work
# ---------------------------------------------------------------------------------------------------------------
def _pos(n=6):
    return torch.zeros((n, 3), dtype=torch.float64)


def _cells(F):
    return torch.eye(3, dtype=torch.float64).expand(F, 3, 3) * 10.0


def test_neighbor_list_rejects_a_decreasing_batch():
    with pytest.raises(ValueError, match="non-decreasing"):
        ops.neighbor_list(_pos(), _cells(2), True, R_MAX, batch=torch.tensor([0, 0, 1, 1, 0, 1]))


def test_neighbor_list_rejects_a_batch_of_the_wrong_length_or_type():
    with pytest.raises(ValueError, match="batch must be"):
        ops.neighbor_list(_pos(), _cells(2), True, R_MAX, batch=torch.tensor([0, 0, 1, 1]))
    with pytest.raises(ValueError, match="batch must be"):
        ops.neighbor_list(_pos(), _cells(2), True, R_MAX, batch=torch.zeros(6))


@pytest.mark.parametrize("batch", [[0, 0, 1, 1, 2, 2], [-1, 0, 0, 1, 1, 1]])
def test_neighbor_list_rejects_a_cell_count_other_than_the_frame_count(batch):
    with pytest.raises(ValueError, match="outside"):
        ops.neighbor_list(_pos(), _cells(2), True, R_MAX, batch=torch.tensor(batch))
    with pytest.raises(ValueError, match="rows for"):
        ops.neighbor_list(_pos(), _cells(2), torch.ones((3, 3), dtype=torch.bool), R_MAX,
                          batch=torch.tensor([0, 0, 1, 1, 1, 1]))
    with pytest.raises(ValueError, match=r"\[F, 3, 3\]"):
        ops.neighbor_list(_pos(), torch.eye(3, dtype=torch.float64), True, R_MAX,
                          batch=torch.tensor([0, 0, 0, 0, 0, 0]))


@pytest.mark.parametrize("pbc", [np.ones((2, 2), dtype=bool), np.ones(2, dtype=bool), np.ones((2, 3, 1), dtype=bool)])
def test_neighbor_list_rejects_a_pbc_of_the_wrong_shape(pbc):
    with pytest.raises(ValueError, match="pbc must be"):
        ops.neighbor_list(_pos(), _cells(2), pbc, R_MAX, batch=torch.tensor([0, 0, 1, 1, 1, 1]))


def test_neighbor_list_rejects_a_periodic_frame_without_a_cell():
    with pytest.raises(ValueError, match="no cell"):
        ops.neighbor_list(_pos(), None, torch.tensor([[False] * 3, [True, False, False]]), R_MAX,
                          batch=torch.tensor([0, 0, 1, 1, 1, 1]))
    with pytest.raises(ValueError, match="no cell"):
        ops.neighbor_list(_pos(), None, True, R_MAX, batch=torch.tensor([0, 0, 1, 1, 1, 1]))


def test_frame_args_give_open_frames_the_identity_cell():
    cells = _cells(3).clone()
    cells[1] = torch.tensor([[3.0, 0.0, 0.0], [1.0, 4.0, 0.0], [0.0, 0.5, 5.0]])
    pbc = np.array([[True] * 3, [False] * 3, [True, True, False]])
    F, p, c = ops._nl_frame_args(cells, pbc, torch.tensor([0, 1, 1, 2]), 4)
    assert F == 3 and p.tolist() == pbc.tolist()
    assert np.array_equal(c[1], np.eye(3)) and np.array_equal(c[0], cells[0].numpy())
    assert np.array_equal(c[2], cells[2].numpy())
    F, p, c = ops._nl_frame_args(None, False, torch.tensor([0, 0, 2]), 3)  # a frame may hold no atoms
    assert F == 3 and not p.any() and np.array_equal(c, np.broadcast_to(np.eye(3), (3, 3, 3)))
