"""Captured MD steps of a batch of frames, on the host: the argument checks of ``NeighborListPlan(batch=)``, the
per-frame blocks of ``nqb_nl_frames_pack_capacity`` read back through ctypes, and on the float64 batched oracle that
each frame's null edges with that frame's own shift change nothing, while one shift for every frame can."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from nequip_b200 import _capi
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel

from batched_oracle import concat_frames, energy_forces_stress
from cell_frames import brute_list, cell_frame

R_MAX = 5.0


def _pos(n=6):
    return torch.zeros((n, 3), dtype=torch.float64)


def _cells(F):
    return torch.eye(3, dtype=torch.float64).expand(F, 3, 3) * 10.0


# ------------------------------------------------------------------------------------------------------------------
# argument checks of NeighborListPlan(batch=) -- raised on the host, before any device work
# ------------------------------------------------------------------------------------------------------------------
def test_plan_rejects_a_malformed_or_decreasing_batch():
    with pytest.raises(ValueError, match="non-decreasing"):
        ops.NeighborListPlan(6, _cells(2), True, R_MAX, 100, batch=torch.tensor([0, 0, 1, 1, 0, 1]))
    with pytest.raises(ValueError, match="batch must be"):
        ops.NeighborListPlan(6, _cells(2), True, R_MAX, 100, batch=torch.tensor([0, 0, 1, 1]))
    with pytest.raises(ValueError, match="batch must be"):
        ops.NeighborListPlan(6, _cells(2), True, R_MAX, 100, batch=torch.zeros(6))
    with pytest.raises(ValueError, match="outside"):
        ops.NeighborListPlan(6, _cells(2), True, R_MAX, 100, batch=torch.tensor([0, 0, 1, 1, 2, 2]))


def test_plan_rejects_a_cell_shape_that_does_not_match_the_frames():
    with pytest.raises(ValueError, match=r"\[F, 3, 3\]"):
        ops.NeighborListPlan(6, torch.eye(3, dtype=torch.float64), True, R_MAX, 100, batch=torch.zeros(6, dtype=torch.long))
    with pytest.raises(ValueError, match="rows for"):
        ops.NeighborListPlan(6, _cells(2), torch.ones((3, 3), dtype=torch.bool), R_MAX, 100,
                             batch=torch.tensor([0, 0, 1, 1, 1, 1]))


def test_plan_rejects_open_frames_without_the_opt_in_and_with_variable_cell():
    pbc = torch.tensor([[True] * 3, [True, True, False]])
    b = torch.tensor([0, 0, 0, 1, 1, 1])
    with pytest.raises(ValueError, match="open_boundaries"):
        ops.NeighborListPlan(6, _cells(2), pbc, R_MAX, 100, batch=b)
    with pytest.raises(ValueError, match="open_boundaries"):
        ops.NeighborListPlan(6, None, False, R_MAX, 100, batch=b)
    with pytest.raises(ValueError, match="variable_cell"):
        ops.NeighborListPlan(6, _cells(2), pbc, R_MAX, 100, batch=b, variable_cell=True, open_boundaries=True)


def test_plan_rejects_a_singular_frame_cell():
    cells = _cells(2).clone()
    cells[1, 2] = cells[1, 1]
    with pytest.raises(ValueError, match="singular"):
        ops.NeighborListPlan(6, cells, True, R_MAX, 100, batch=torch.tensor([0, 0, 0, 1, 1, 1]))


def test_graphed_md_step_reads_per_frame_periodicity():
    ex = {"pbc": torch.tensor([[True, True, False], [False] * 3]), "batch": torch.tensor([0, 1])}
    assert GraphedMDStep._periodicity(ex) == ((True, True, False), (False, False, False))
    # without a batch the [F, 3] form is not a frame's periodicity
    with pytest.raises(ValueError, match="3 flags"):
        GraphedMDStep._periodicity({"pbc": ex["pbc"]})
    assert GraphedMDStep._periodicity({"pbc": torch.tensor([True, True, False]), "batch": ex["batch"]}) == (
        True, True, False)


# ------------------------------------------------------------------------------------------------------------------
# the packed blocks
# ------------------------------------------------------------------------------------------------------------------
class _Block(ctypes.Structure):
    """``NlBlock`` of nqb_nl.cu (``NlParams`` then the capacity and open-direction fields)."""
    _fields_ = [("cell", ctypes.c_double * 9), ("inv", ctypes.c_double * 9), ("diag", ctypes.c_double * 3),
                ("orthorhombic", ctypes.c_int), ("pbc", ctypes.c_int * 3), ("nb", ctypes.c_int * 3),
                ("sr", ctypes.c_int * 3), ("lo", ctypes.c_double * 3), ("width", ctypes.c_double * 3),
                ("r2", ctypes.c_double), ("pad_shift", ctypes.c_double * 3), ("open", ctypes.c_int * 3),
                ("cap", ctypes.c_int), ("perp", ctypes.c_double * 3), ("r_max", ctypes.c_double)]


def _frame_args(cells, pbc):
    F = cells.shape[0]
    invs = np.linalg.inv(cells)
    I3, D9, D3 = ctypes.c_int * (3 * F), ctypes.c_double * (9 * F), ctypes.c_double * (3 * F)
    nb = [2 + (k % 3) for k in range(3 * F)]
    sr = [1 + (k % 2) for k in range(3 * F)]
    lo = [0.25 * k for k in range(3 * F)]
    width = [1.0 + k for k in range(3 * F)]
    return (F, D9(*cells.reshape(-1)), D9(*invs.reshape(-1)), I3(*[int(b) for b in pbc.reshape(-1)]), I3(*nb),
            I3(*sr), D3(*lo), D3(*width), R_MAX)


def _pack_cells():
    cells = np.stack([np.diag([20.0, 10.0, 10.0]), np.diag([2.4, 12.0, 12.0]),
                      np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]]), np.eye(3)])
    pbc = np.array([[True] * 3, [True] * 3, [True, True, False], [False] * 3])
    return cells, pbc


def test_pack_capacity_holds_each_frames_null_shift_and_open_fields():
    L = _capi.lib()
    nbytes = int(L.nqb_nl_params_bytes())
    assert ctypes.sizeof(_Block) == nbytes
    cells, pbc = _pack_cells()
    F = cells.shape[0]
    pad = np.stack([ops.null_edge_shift(c, R_MAX) for c in cells])
    perp = np.stack([1.0 / np.linalg.norm(np.linalg.inv(c), axis=0) for c in cells])
    caps = [3, 5, 7, 2]
    args = _frame_args(cells, pbc)
    out = ctypes.create_string_buffer(F * nbytes)
    _capi.check(L.nqb_nl_frames_pack_capacity(*args, (ctypes.c_double * (3 * F))(*pad.reshape(-1)),
                                              (ctypes.c_int * F)(*caps), (ctypes.c_double * (3 * F))(*perp.reshape(-1)),
                                              out), "nqb_nl_frames_pack_capacity")
    plain = ctypes.create_string_buffer(F * nbytes)
    _capi.check(L.nqb_nl_frames_pack(*args, plain), "nqb_nl_frames_pack")
    for f in range(F):
        b = _Block.from_buffer_copy(out.raw[f * nbytes:(f + 1) * nbytes])
        assert list(b.pad_shift) == pad[f].tolist()
        assert list(b.open) == [0 if p else 1 for p in pbc[f]]
        assert b.cap == caps[f] and b.r_max == R_MAX and list(b.perp) == perp[f].tolist()
        # the parameters the kernels read are those of nqb_nl_frames_pack, byte for byte
        off = _Block.pad_shift.offset
        assert out.raw[f * nbytes:f * nbytes + off] == plain.raw[f * nbytes:f * nbytes + off]
    # frames 0 and 1 need different shifts: (2, 0, 0) would be 4.8 long in frame 1
    assert pad[0].tolist() == [2.0, 0.0, 0.0] and pad[1].tolist() == [0.0, 2.0, 0.0]


def test_pack_capacity_rejects_bad_arguments():
    L = _capi.lib()
    nbytes = int(L.nqb_nl_params_bytes())
    cells, pbc = _pack_cells()
    F = cells.shape[0]
    out = ctypes.create_string_buffer(F * nbytes)
    D, I = ctypes.c_double * (3 * F), ctypes.c_int * F
    pad, perp, caps = D(*([7.0] * 3 * F)), D(*([1.0] * 3 * F)), I(*([2] * F))
    assert L.nqb_nl_frames_pack_capacity(*_frame_args(cells, pbc), pad, caps, perp, out) == 0
    assert L.nqb_nl_frames_pack_capacity(*_frame_args(cells, pbc), pad, I(2, 0, 2, 2), perp, out) != 0
    bad = [1.0] * 3 * F
    bad[4] = float("nan")
    assert L.nqb_nl_frames_pack_capacity(*_frame_args(cells, pbc), pad, caps, D(*bad), out) != 0
    assert L.nqb_nl_frames_pack_capacity(*_frame_args(cells, pbc), None, caps, perp, out) != 0


# ------------------------------------------------------------------------------------------------------------------
# null edges on the float64 batched oracle
# ------------------------------------------------------------------------------------------------------------------
def _pad_rows(b, shifts_of_frame, seed):
    """The batch with 0 to 3 null edges (i, i, shifts_of_frame[frame of i]) appended to each row."""
    rng = np.random.default_rng(seed)
    ei, sh = b["edge_index"].numpy(), b["edge_cell_shift"].numpy()
    frame = b["batch"].numpy()
    rows, shs = [], []
    extra = rng.integers(0, 4, b["pos"].shape[0])
    for i in range(b["pos"].shape[0]):
        sel = ei[0] == i
        rows.append(np.concatenate([ei[:, sel], np.full((2, extra[i]), i, dtype=np.int64)], 1))
        shs.append(np.concatenate([sh[sel], np.tile(shifts_of_frame[frame[i]], (extra[i], 1))], 0))
    assert extra.sum() > 0
    return dict(b, edge_index=torch.from_numpy(np.concatenate(rows, 1)),
                edge_cell_shift=torch.from_numpy(np.concatenate(shs, 0)))


def _model(type_names, E_over_N, zbl=False):
    kw = dict(pair_potential={"units": "metal", "chemical_species": list(type_names)}) if zbl else {}
    return NequIPEnergyModel(r_max=R_MAX, type_names=type_names, parity=True, l_max=2, num_layers=2, num_features=8,
                             radial_mlp_depth=1, radial_mlp_width=16, avg_num_neighbors=E_over_N,
                             model_dtype=torch.float64, seed=7, **kw)


@pytest.mark.parametrize("zbl", [False, True], ids=["plain", "zbl"])
def test_each_frames_own_null_edges_change_nothing(zbl):
    frames, pbcs = [], []
    for s, (name, pbc) in enumerate([("cubic", True), ("tilted", True), ("left", True), ("small", True),
                                     ("skewed", (True, True, False))]):
        d = cell_frame("li3po4", 2, name, seed=s, outside=True, pbc=pbc)
        meta = d.pop("_meta")
        frames.append(d)
        pbcs.append([bool(v) for v in (pbc if isinstance(pbc, tuple) else (pbc,) * 3)])
    b = concat_frames(frames, pbcs)
    pads = np.stack([ops.null_edge_shift(c, R_MAX) for c in b["cell"].numpy()])
    model = _model(meta["type_names"], b["edge_index"].shape[1] / b["pos"].shape[0], zbl)
    sd, cfg = model.state_dict(), model.config
    e0, ea0, f0, s0, _ = energy_forces_stress(sd, cfg, b)
    e1, ea1, f1, s1, _ = energy_forces_stress(sd, cfg, _pad_rows(b, pads, 3))
    assert float(f0.abs().max()) > 0
    assert float((e1 - e0).abs().max()) <= 1e-13 * float(ea0.abs().sum())
    assert float((ea1 - ea0).abs().max()) <= 1e-13 * float(ea0.abs().max())
    assert float((f1 - f0).abs().max()) <= 1e-13 * float(f0.abs().max())
    assert float((s1 - s0).abs().max()) <= 1e-13 * float(s0.abs().max())


def test_one_shift_for_every_frame_changes_the_energy():
    """Frame 0 in diag(20, 10, 10) has the null shift (2, 0, 0); in frame 1's diag(2.4, 12, 12) that shift is an edge
    of 4.8 < r_max, which adds energy, while frame 1's own shift (0, 2, 0) adds none."""
    rng = np.random.default_rng(11)
    frames = []
    for cell, n in ((np.diag([20.0, 10.0, 10.0]), 6), (np.diag([2.4, 12.0, 12.0]), 4)):
        pos = rng.uniform(0.0, 1.0, (n, 3)) * np.diagonal(cell)
        ei, sh = brute_list(pos, cell, True, R_MAX)
        frames.append({"pos": torch.from_numpy(pos), "cell": torch.from_numpy(cell.copy()),
                       "atom_types": torch.from_numpy(rng.integers(0, 3, n)), "edge_index": torch.from_numpy(ei),
                       "edge_cell_shift": torch.from_numpy(sh)})
    b = concat_frames(frames)
    own = np.stack([ops.null_edge_shift(c, R_MAX) for c in b["cell"].numpy()])
    assert own.tolist() == [[2.0, 0.0, 0.0], [0.0, 2.0, 0.0]]
    model = _model(["Li", "P", "O"], b["edge_index"].shape[1] / b["pos"].shape[0])
    sd, cfg = model.state_dict(), model.config
    e0, ea0, f0, _s, _v = energy_forces_stress(sd, cfg, b)
    e_own = energy_forces_stress(sd, cfg, _pad_rows(b, own, 5))[0]
    e_one = energy_forces_stress(sd, cfg, _pad_rows(b, own[[0, 0]], 5))[0]
    assert float((e_own - e0).abs().max()) <= 1e-13 * float(ea0.abs().sum())
    assert float(e_one[0, 0]) == float(e_own[0, 0])  # frame 0 keeps its own shift
    assert abs(float(e_one[1, 0]) - float(e0[1, 0])) > 1e-6
