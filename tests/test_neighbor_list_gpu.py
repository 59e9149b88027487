"""GPU cell-list neighbour list (nqb_nl_*, nequip_b200/ops.py neighbor_list) vs the host lists of
nequip_b200/data.py (cell list / brute force with images) and, in triclinic, left-handed, small and partly periodic
cells, vs the float64 brute force of tests/cell_frames.py -- same contract as the reference's backends
(nequip/data/_nl.py:60-152): the edge set, the shifts and the (centre, neighbour) order must be identical."""
import numpy as np
import pytest
import torch

from cell_frames import brute_list, cell_frame, named_cell, perp_widths
from nequip_b200 import data as D
from nequip_b200 import ops

pytestmark = pytest.mark.gpu


def _check(pos_np, cell_np, r_max, pbc=True, ref=None):
    """The device list against ``ref`` (edge_index, shifts), by default the host list of data.py: identical edges,
    shifts and order, the destination CSR and the (neighbour, centre) transpose order.  Returns the device list."""
    ei_ref, sh_ref = D.neighbor_list(pos_np, cell_np, r_max, pbc=pbc) if ref is None else ref
    out = ops.neighbor_list(torch.from_numpy(pos_np).cuda(), None if cell_np is None else torch.from_numpy(cell_np), pbc, r_max,
                            transpose_perm=True)
    ei, sh = out["edge_index"].cpu().numpy(), out["edge_cell_shift"].cpu().numpy()
    assert ei.shape == ei_ref.shape, (ei.shape, ei_ref.shape)
    np.testing.assert_array_equal(ei, ei_ref)
    np.testing.assert_array_equal(sh, sh_ref)
    N = pos_np.shape[0]
    rp = out["row_ptr"].cpu().numpy()
    np.testing.assert_array_equal(rp, np.concatenate([[0], np.cumsum(np.bincount(ei_ref[0], minlength=N))]))
    tp = out["edge_transpose_perm"].cpu().numpy()
    np.testing.assert_array_equal(tp, np.lexsort((ei_ref[0], ei_ref[1])))
    return out


@pytest.mark.parametrize("kind,n_side", [("li3po4", 12), ("water", 10), ("asi", 16)])
def test_matches_host_cell_list(kind, n_side):
    pr = D.PRESETS[kind]
    pos, cell = D.jittered_lattice(n_side, pr["density"], seed=3)
    pos = pos + np.array([3.7, -11.2, 0.4])  # atoms outside the home cell: base shifts are exercised
    assert _check(pos, cell, 5.0)["edge_index"].shape[1] > 0


def test_small_cells_need_several_images():
    rng = np.random.default_rng(0)
    for L in (3.0, 6.5, 9.0):  # r_max = 5 > L/2: the same neighbour appears under several shifts
        cell = np.diag([L, L * 1.1, L * 0.9])
        pos = rng.uniform(0, 1, (11, 3)) @ cell
        _check(pos, cell, 5.0)


def test_non_periodic_and_empty():
    rng = np.random.default_rng(1)
    pos = rng.uniform(0, 14, (200, 3))
    _check(pos, None, 5.0, pbc=False)
    out = ops.neighbor_list(torch.tensor([[0.0, 0, 0], [100.0, 0, 0]], dtype=torch.float64).cuda(), None, False, 5.0)
    assert out["edge_index"].shape == (2, 0) and out["row_ptr"].tolist() == [0, 0, 0]


def test_triclinic_cell_against_bruteforce():
    rng = np.random.default_rng(2)
    cell = np.array([[11.0, 0.0, 0.0], [3.0, 10.0, 0.0], [-2.0, 1.5, 12.0]])
    pos = rng.uniform(0, 1, (150, 3)) @ cell
    _check(pos, cell, 4.0, ref=brute_list(pos, cell, True, 4.0))


def test_model_runs_on_the_device_list():
    from nequip_b200.nn.model import NequIPEnergyModel

    sysd = D.make_system("water", 6, r_max=5.0, seed=0)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=5.0, type_names=meta["type_names"], l_max=2, num_layers=3, num_features=32,
                              avg_num_neighbors=meta["avg_num_neighbors"]).cuda()
    dev = D.to_device(sysd, "cuda")
    ref = model(dev)
    nl = ops.neighbor_list(dev["pos"], sysd["cell"], True, 5.0)
    d2 = dict(dev)
    d2["edge_index"], d2["edge_cell_shift"] = nl["edge_index"], nl["edge_cell_shift"]
    out = model(d2)
    assert torch.equal(out["forces"], ref["forces"]) or float((out["forces"] - ref["forces"]).abs().max()) <= 1e-6 * float(ref["forces"].abs().max())


# ------------------------------------------------------------------------------------------------------------------
# general cells against the float64 brute force of tests/cell_frames.py
# ------------------------------------------------------------------------------------------------------------------
PBC = {"TTT": (True, True, True), "TTF": (True, True, False), "TFT": (True, False, True), "FFT": (False, False, True)}


@pytest.mark.parametrize("outside", [False, True], ids=["inside", "outside"])
@pytest.mark.parametrize("pbc", list(PBC))
@pytest.mark.parametrize("name", ["tilted", "skewed", "left", "small"])
def test_general_cells_against_bruteforce(name, pbc, outside):
    """Every named cell (triclinic, not basis-reduced, left-handed, smaller than r_max) with full, slab and partial
    periodicity; ``outside``: atoms several cells away along the periodic directions (base shifts) and below
    fractional 0 along the open ones."""
    f = cell_frame("li3po4", 2 if name == "small" else 6, name, seed=11, outside=outside, pbc=PBC[pbc])
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    out = _check(pos, cell, 5.0, pbc=PBC[pbc], ref=(f["edge_index"].numpy(), f["edge_cell_shift"].numpy()))
    sh = out["edge_cell_shift"].cpu().numpy()
    assert sh.shape[0] > 0
    for d in range(3):
        if not PBC[pbc][d]:
            assert not sh[:, d].any()
        elif outside:
            assert np.abs(sh[:, d]).max() >= 2, "base shifts are exercised"
    if name == "small":  # a neighbour appears under several shifts
        ei = out["edge_index"].cpu().numpy()
        assert perp_widths(cell).max() < 5.0 and np.unique(ei[0] * pos.shape[0] + ei[1]).size < ei.shape[1]


def test_skewed_cell_with_several_bins_per_direction():
    """~1 300 atoms in a cell with tilts of 0.5 to 0.6 of its lengths and at least 3 bins along every direction."""
    f = cell_frame("li3po4", 11, "skewed", seed=5, outside=True)
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    _pbc, cell_np, inv_np = ops._nl_cell(cell, True)
    nb = ops._NlArgs(pos.shape[0], cell_np, inv_np, [True] * 3, 5.0, np.zeros(3), np.ones(3)).nb
    assert min(nb) >= 3, tuple(nb)
    _check(pos, cell, 5.0, ref=(f["edge_index"].numpy(), f["edge_cell_shift"].numpy()))


@pytest.mark.parametrize("name", ["cubic", "tilted"])
def test_perfect_lattice_on_bin_faces(name):
    """An unjittered lattice: atoms at fractional 0 and exactly on bin faces (8 lattice planes over 4 bins), with
    r_max in the middle of the gap between two neighbour shells."""
    n = 8
    cell = 2.5 * n * (np.eye(3) if name == "cubic" else np.array([[1.0, 0.0, 0.0], [0.125, 1.0, 0.0], [-0.125, 0.125, 1.0]]))
    g = np.arange(n, dtype=np.float64)
    frac = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) / n
    pos = frac @ cell
    # neighbour shells of the lattice: |u @ cell / n| for small integer u
    u = np.stack(np.meshgrid(*[np.arange(-4, 5)] * 3, indexing="ij"), -1).reshape(-1, 3)
    shells = np.unique(np.round(np.linalg.norm(u @ cell / n, axis=1), 9))
    k = int(np.searchsorted(shells, 5.0))
    r_max = 0.5 * (shells[k - 1] + shells[k])
    assert shells[k] - shells[k - 1] > 0.05
    _pbc, cell_np, inv_np = ops._nl_cell(cell, True)
    nb = ops._NlArgs(pos.shape[0], cell_np, inv_np, [True] * 3, r_max, np.zeros(3), np.ones(3)).nb
    assert min(nb) >= 3 and all(n % b == 0 for b in nb), tuple(nb)
    out = _check(pos, cell, r_max, ref=brute_list(pos, cell, True, r_max))
    assert np.all(np.diff(out["row_ptr"].cpu().numpy()) == np.diff(out["row_ptr"].cpu().numpy())[0])


def _bins(monkeypatch, pos, cell, pbc, r_max=5.0):
    """The device list plus the bin grid and per-atom bins (cidx) that ops.neighbor_list used for it."""
    seen = {}
    rows = ops._nl_rows

    def spy(pos_, a, s, params_dev=None):
        rows(pos_, a, s, params_dev)
        seen.update(nb=tuple(a.nb), cidx=s["cidx"].cpu().numpy())

    monkeypatch.setattr(ops, "_nl_rows", spy)
    out = ops.neighbor_list(torch.from_numpy(pos).cuda(), torch.from_numpy(cell), pbc, r_max)
    return out, seen["nb"], seen["cidx"]


@pytest.mark.parametrize("pbc", ["TTF", "FFT"])
def test_open_directions_are_binned_over_the_bounding_box(monkeypatch, pbc):
    """Along an open direction the bins divide the atoms' bounding box: the lowest atom is in bin 0, the highest in
    the last bin, and the bin grows with the fractional coordinate.  (A grid that missed the box would still give
    the exact list -- any grid of bins at least r_max wide does -- but with most atoms piled into one bin.)"""
    f = cell_frame("li3po4", 9, "tilted", seed=3, outside=True, pbc=PBC[pbc])
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    out, nb, cidx = _bins(monkeypatch, pos, cell, PBC[pbc])
    np.testing.assert_array_equal(out["edge_index"].cpu().numpy(), f["edge_index"].numpy())
    frac = pos @ np.linalg.inv(cell)
    for d in range(3):
        if PBC[pbc][d]:
            continue
        assert frac[:, d].min() < -0.4, "the frame reaches below fractional 0"
        assert nb[d] >= 3, nb
        o = np.argsort(frac[:, d], kind="stable")
        assert cidx[o[0], d] == 0 and cidx[o[-1], d] == nb[d] - 1, (d, nb, cidx[o[[0, -1]], d])
        assert np.all(np.diff(cidx[o, d]) >= 0)
        assert np.all(np.bincount(cidx[:, d], minlength=nb[d]) > 0)


def test_slab_equals_a_periodic_cell_with_vacuum():
    """pbc = (T, T, F) and the same frame with pbc = True in a cell whose third vector is long enough to leave more
    than r_max of vacuum: identical lists, shifts included (no edge crosses the vacuum)."""
    f = cell_frame("li3po4", 6, "tilted", seed=4, outside=True, pbc=PBC["TTF"])
    pos, cell = f["pos"].numpy(), f["cell"].numpy()
    tall = cell.copy()
    tall[2] *= 4.0
    frac = pos @ np.linalg.inv(tall)
    vacuum = (1.0 - (frac[:, 2].max() - frac[:, 2].min())) * perp_widths(tall)[2]
    assert vacuum > 5.0, vacuum
    slab = ops.neighbor_list(torch.from_numpy(pos).cuda(), torch.from_numpy(cell), PBC["TTF"], 5.0)
    per = ops.neighbor_list(torch.from_numpy(pos).cuda(), torch.from_numpy(tall), True, 5.0)
    for k in ("edge_index", "edge_cell_shift", "row_ptr"):
        assert torch.equal(slab[k], per[k]), k
    assert slab["edge_index"].shape[1] == f["edge_index"].shape[1]


def test_open_frame_equals_a_large_periodic_box():
    """pbc = False and a periodic box far larger than the frame plus r_max: the same edges, every shift 0."""
    f = cell_frame("li3po4", 6, "skewed", seed=6, outside=False, pbc=False)
    pos = torch.from_numpy(f["pos"].numpy()).cuda()
    box = torch.from_numpy(named_cell("tilted", 40))
    open_ = ops.neighbor_list(pos, None, False, 5.0)
    per = ops.neighbor_list(pos, box, True, 5.0)
    assert torch.equal(open_["edge_index"], per["edge_index"]) and torch.equal(open_["row_ptr"], per["row_ptr"])
    assert not per["edge_cell_shift"].any() and not open_["edge_cell_shift"].any()
    np.testing.assert_array_equal(open_["edge_index"].cpu().numpy(), f["edge_index"].numpy())
