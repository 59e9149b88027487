"""Reverse-edge pair map of the radial MLP (nqb_edge_pairs, ops.edge_pairs) and the forward that computes one row
per pair (nqb_mlp_hidden_fwd_rows + nqb_gemm_grouped_pairs): the map against a host restatement, the edge weights
bitwise equal to the per-edge forward, the write contracts, and whole models against the same model without pairs."""
import math

import numpy as np
import pytest
import torch

from cell_frames import cell_frame
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.nn import dense
from nequip_b200.nn.model import NequIPEnergyModel, ScalarLinearLayer

pytestmark = pytest.mark.gpu

R_MAX = 5.0


# ---------------------------------------------------------------------------------------------------------------
# host restatement
# ---------------------------------------------------------------------------------------------------------------
def host_pairs(ei: np.ndarray, sh, emb: np.ndarray):
    """Slots (representative, partner or -1) of the contract in nqb.h, from a dict on (i, j, shift, emb bits)."""
    E = ei.shape[1]
    order = np.argsort(ei[0], kind="stable")  # CSR order
    bits = np.ascontiguousarray(emb.astype(np.float32)).view(np.uint32)
    shv = np.zeros((E, 3)) if sh is None else np.asarray(sh, dtype=np.float64)
    rows = {}
    for f in order:  # value keys: -0.0 == 0.0 hashes and compares as 0.0
        rows.setdefault((int(ei[0, f]), int(ei[1, f]), tuple(float(v) for v in shv[f]), bits[f].tobytes()), []).append(int(f))
    cand = np.full(E, -1, dtype=np.int64)
    for e in range(E):
        for f in rows.get((int(ei[1, e]), int(ei[0, e]), tuple(float(-v) for v in shv[e]), bits[e].tobytes()), ()):
            if f != e:
                cand[e] = f
                break
    slots = []
    for e in range(E):
        c = cand[e]
        p = c if (c >= 0 and cand[c] == e) else -1
        if p < 0 or e < p:
            slots.append((e, p))
    return np.array(slots, dtype=np.int64).reshape(-1, 2)


def _embed(d):
    pos, ei = d["pos"].cuda(), d["edge_index"].cuda()
    cell = d.get("cell")
    shift = d.get("edge_cell_shift")
    if cell is not None:
        cell, shift = cell.cuda(), shift.cuda()
    _v, _y, emb = ops.edge_embed(pos, ei, shift, cell, lmax=2, num_bessel=8, r_max=R_MAX,
                                 prefactor=2 * math.pi / R_MAX ** 2)
    return ei, shift, emb


def _pairs(ei, shift, emb, N):
    csr = ops.build_csr(ei[0], N)
    return ops.edge_pairs(ei, shift, emb, csr), csr


def _mlp(W, seed=0):
    g = torch.Generator().manual_seed(seed)
    l1, l2 = ScalarLinearLayer(8, 128, 1 / math.sqrt(8)).cuda(), ScalarLinearLayer(128, W, 1 / math.sqrt(128)).cuda()
    with torch.no_grad():
        l1.weight.copy_(torch.randn(8, 128, generator=g))
        l2.weight.copy_(torch.randn(128, W, generator=g))
    return dense.RadialMLPGemm(l1, l2, "cuda")


def _frames():
    out = {}
    out["bench"] = D.make_system("li3po4", 22, r_max=R_MAX)
    out["tilted"] = cell_frame("li3po4", 4, "tilted")
    out["left"] = cell_frame("li3po4", 4, "left", outside=True)
    out["small_self_images"] = cell_frame("li3po4", 2, "small")
    base = D.make_system("li3po4", 6, r_max=R_MAX)
    E = base["edge_index"].shape[1]
    g = torch.Generator().manual_seed(5)
    p = torch.randperm(E, generator=g)
    out["shuffled"] = dict(base, edge_index=base["edge_index"][:, p].contiguous(),
                           edge_cell_shift=base["edge_cell_shift"][p].contiguous())
    # some reverse edges deleted; atom 0 loses every edge
    keep = (torch.rand(E, generator=g) > 0.1) & (base["edge_index"][0] != 0) & (base["edge_index"][1] != 0)
    out["deleted"] = dict(base, edge_index=base["edge_index"][:, keep].contiguous(),
                          edge_cell_shift=base["edge_cell_shift"][keep].contiguous())
    # a duplicated edge (its copy follows it in the same row)
    dup = torch.cat([torch.arange(0, 7), torch.tensor([6]), torch.arange(7, E)])
    out["duplicated"] = dict(base, edge_index=base["edge_index"][:, dup].contiguous(),
                             edge_cell_shift=base["edge_cell_shift"][dup].contiguous())
    # padded capacity list of the device neighbour list: null edges (i, i, pad_shift) stay unpaired
    plan = ops.NeighborListPlan(base["pos"].shape[0], base["cell"], True, R_MAX, E + 999, device="cuda")
    nl = plan.run(base["pos"].cuda())
    out["capacity"] = dict(base, edge_index=nl["edge_index"].cpu(), edge_cell_shift=nl["edge_cell_shift"].cpu(),
                           pad_shift=torch.tensor([float(v) for v in plan.pad_shift], dtype=torch.float64))
    # no edges at all
    out["empty"] = dict(base, edge_index=torch.zeros((2, 0), dtype=torch.int64),
                        edge_cell_shift=torch.zeros((0, 3), dtype=torch.float64))
    for d in out.values():
        d.pop("_meta", None)
    return out


_FRAMES = None


def frames():
    global _FRAMES
    if _FRAMES is None:
        _FRAMES = _frames()
    return _FRAMES


FRAME_NAMES = ["bench", "tilted", "left", "small_self_images", "shuffled", "deleted", "duplicated", "capacity", "empty"]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", FRAME_NAMES)
def test_pair_map_matches_host_and_w_is_bitwise_per_edge(name):
    d = frames()[name]
    N = d["pos"].shape[0]
    ei, shift, emb = _embed(d)
    E = ei.shape[1]
    (rows, count), csr = _pairs(ei, shift, emb, N)
    if name == "shuffled":
        assert csr.perm is not None
    torch.cuda.synchronize()
    U = int(count.item())
    ref = host_pairs(ei.cpu().numpy(), None if shift is None else shift.cpu().numpy(), emb.cpu().numpy())
    assert U == ref.shape[0]
    assert np.array_equal(rows[:U].cpu().numpy(), ref)
    if name == "bench":
        assert U * 2 == E
    if name == "small_self_images":
        eic = ei.cpu()
        self_e = (eic[0] == eic[1]).nonzero().flatten()
        assert self_e.numel() > 0
        assert set(self_e.tolist()) <= set(rows[:U].cpu().flatten().tolist())
    if name == "capacity":  # null edges (i, i, pad_shift): one slot each, no partner
        null_edges = ((ei[0] == ei[1]) & (shift == d["pad_shift"].cuda()).all(1)).nonzero().flatten().cpu()
        assert null_edges.numel() > 0
        r = rows[:U].cpu()
        assert not bool(torch.isin(null_edges, r[:, 1]).any())
        assert bool(torch.isin(null_edges, r[:, 0]).all())
    for W in (864, 1728):
        mlp = _mlp(W, seed=W)
        w_pair = mlp(emb, (rows, count))
        h = torch.empty((E, 128), device="cuda")
        if E:
            ops.mlp_hidden_fwd(emb, mlp.w1s, h, None)
        w_edge = torch.empty((E, W), device="cuda")
        mlp.fwd.run(h, w_edge, E)
        assert torch.equal(w_pair, w_edge), (name, W)


# ---------------------------------------------------------------------------------------------------------------
# write contracts
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("name", ["bench", "deleted", "capacity", "empty"])
def test_edge_pairs_write_contract(name):
    d = frames()[name]
    N = d["pos"].shape[0]
    ei, shift, emb = _embed(d)
    E = ei.shape[1]
    csr = ops.build_csr(ei[0], N)
    rows, ck_rows = guarded(max(E, 1), 2, torch.int64)
    cnt, ck_cnt = guarded(1, 1, torch.int64)
    L = _capi.lib()
    work = torch.empty(int(L.nqb_edge_pairs_work_size(E)), dtype=torch.int64, device="cuda")
    _capi.check(L.nqb_edge_pairs(ei.data_ptr(), E, N, 0 if shift is None else shift.data_ptr(), emb.data_ptr(), 8,
                                 csr.row_ptr.data_ptr(), 0 if csr.perm is None else csr.perm.data_ptr(),
                                 work.data_ptr(), rows.data_ptr(), cnt.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream), "nqb_edge_pairs")
    torch.cuda.synchronize()
    ck_rows("pair_rows")
    ck_cnt("count")
    U = int(cnt.item())
    assert not bool(is_poison(rows[:U]).any())
    assert bool(is_poison(rows[U:]).all()), "slots >= U written"
    if E == 0:
        assert U == 0


def _synthetic_pairs(E, U, seed):
    """U slots over E rows: slot u = (r[u], r[U + u] or -1), rows distinct."""
    g = torch.Generator().manual_seed(seed)
    r = torch.randperm(E, generator=g)
    rows = torch.full((E, 2), -7, dtype=torch.int64)
    rows[:U, 0] = r[:U]
    rows[:U, 1] = -1
    npair = min(U, E - U)
    rows[:npair, 1] = r[U:U + npair]
    return rows


@pytest.mark.timeout(300)
@pytest.mark.parametrize("U", [0, 1, 63, 129, "half", "all"])
def test_paired_gemm_and_gathered_hidden_write_contracts(U):
    E, W = 4099, 260
    U = {"half": E // 2, "all": E}.get(U, U)
    g = torch.Generator().manual_seed(U + 1)
    emb = (torch.rand(E, 8, generator=g) * 2 - 0.7).cuda()
    mlp = _mlp(W, seed=3)
    rows = _synthetic_pairs(E, U, U).cuda()
    count = torch.tensor([U], dtype=torch.int64, device="cuda")
    # gathered hidden layer: rows < U only, each the per-edge row of its representative
    hflat, ck_h = guarded(E, 128, torch.float32)
    ops.mlp_hidden_fwd_rows(emb, mlp.w1s, (rows, count), hflat)
    h_edge = torch.empty((E, 128), device="cuda")
    ops.mlp_hidden_fwd(emb, mlp.w1s, h_edge, None)
    torch.cuda.synchronize()
    ck_h("h")
    assert torch.equal(hflat[:U], h_edge[rows[:U, 0]])
    assert bool(is_poison(hflat[U:]).all()), "gathered hidden layer wrote rows >= U"
    # paired GEMM into a guarded, poisoned C: every listed row once, columns < N, nothing else
    Cp, ck_C = guarded(E, W, torch.float32)
    mlp.fwd.run_pairs(hflat, Cp, (rows, count))
    ref = torch.empty((E, W), device="cuda")
    mlp.fwd.run(h_edge, ref, E)
    torch.cuda.synchronize()
    ck_C("C")
    listed = torch.cat([rows[:U, 0], rows[:U, 1][rows[:U, 1] >= 0]])
    assert listed.numel() == listed.unique().numel()
    written = ~is_poison(Cp).all(1)
    mask = torch.zeros(E, dtype=torch.bool, device="cuda")
    mask[listed] = True
    assert torch.equal(written, mask)
    assert not bool(is_poison(Cp[listed]).any())
    # row r of a slot holds the result of the slot's representative (bitwise the per-edge GEMM row)
    src = torch.empty(E, dtype=torch.int64, device="cuda")
    src[rows[:U, 0]] = rows[:U, 0]
    sel = rows[:U, 1] >= 0
    src[rows[:U, 1][sel]] = rows[:U, 0][sel]
    assert torch.equal(Cp[listed], ref[src[listed]])


def test_paired_gemm_rejects_non_plain_problems():
    l2 = ScalarLinearLayer(128, 64, 1.0).cuda()
    gg = ops.GroupedGemm([ops.GemmProblem(0, 128, 0, 64, l2.weight.detach(), act="silu")], "cuda")
    rows = torch.zeros((4, 2), dtype=torch.int64, device="cuda")
    count = torch.ones(1, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        gg.run_pairs(torch.zeros(4, 128, device="cuda"), torch.zeros(4, 64, device="cuda"), (rows, count))


# ---------------------------------------------------------------------------------------------------------------
# whole models: with pairs vs the same model with a map without pairs (U = E)
# ---------------------------------------------------------------------------------------------------------------
def _no_pairs(edge_index, shift, emb, csr):
    E = edge_index.shape[1]
    ar = torch.arange(E, dtype=torch.int64, device=emb.device)
    return torch.stack([ar, torch.full_like(ar, -1)], 1).contiguous(), torch.full((1,), E, dtype=torch.int64,
                                                                                     device=emb.device)


def _model(n_side=8):
    sysd = D.make_system("li3po4", n_side, r_max=R_MAX, seed=1)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=2, num_layers=4, num_features=64,
                              parity=True, avg_num_neighbors=meta["avg_num_neighbors"], strict_fast_path=True).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    return model, D.to_device(sysd, "cuda")


def _same(a, b, keys=("total_energy", "atomic_energy"), vec=("forces", "stress", "virial")):
    for k in keys:
        if k in a:
            assert torch.equal(a[k], b[k]), k
    for k in vec:
        if k in a and a[k] is not None:
            scale = float(b[k].abs().max())
            assert float((a[k] - b[k]).abs().max()) <= 2e-6 * scale + 1e-12, k


def _both(fn, monkeypatch):
    calls = []
    real = ops.edge_pairs

    def counted(*a):
        calls.append(1)
        return real(*a)

    monkeypatch.setattr(ops, "edge_pairs", counted)
    a = {k: v.clone() for k, v in fn().items() if torch.is_tensor(v)}
    assert calls, "the model did not build the pair map"
    monkeypatch.setattr(ops, "edge_pairs", _no_pairs)
    b = {k: v.clone() for k, v in fn().items() if torch.is_tensor(v)}
    monkeypatch.setattr(ops, "edge_pairs", real)
    return a, b


@pytest.mark.timeout(600)
def test_model_eager_and_edge_vectors_match_no_pairs(monkeypatch):
    model, dev = _model()
    for compute_stress in (False, True):
        a, b = _both(lambda: model(dev, compute_stress=compute_stress), monkeypatch)
        _same(a, b)
    # ML-IAP: edge vectors in, edge forces out
    vec = ops.edge_embed(dev["pos"], dev["edge_index"], dev["edge_cell_shift"], dev["cell"], lmax=0, num_bessel=8,
                         r_max=R_MAX)[0]
    d2 = {k: v for k, v in dev.items() if k not in ("edge_cell_shift", "cell")}
    d2["edge_vectors"] = vec.clone()
    a, b = _both(lambda: model(d2), monkeypatch)
    _same(a, b, vec=("edge_forces",))


@pytest.mark.timeout(900)
def test_graphed_steps_match_no_pairs(monkeypatch):
    from nequip_b200.graph import GraphedEnergyForces, GraphedMDStep

    model, dev = _model()

    # each graph is captured under the map it replays with: the map is part of the captured step
    real = ops.edge_pairs
    ga = GraphedEnergyForces(model, dev)
    a = {k: v.clone() for k, v in ga.replay().items() if torch.is_tensor(v)}
    monkeypatch.setattr(ops, "edge_pairs", _no_pairs)
    gb = GraphedEnergyForces(model, dev)
    b = {k: v.clone() for k, v in gb.replay().items() if torch.is_tensor(v)}
    monkeypatch.setattr(ops, "edge_pairs", real)
    _same(a, b)
    del ga, gb

    pos1 = D.oscillating_positions(dev["pos"], 7, seed=3)
    for variable in (False, True):
        outs = []
        for fn in (real, _no_pairs):
            monkeypatch.setattr(ops, "edge_pairs", fn)
            kw = dict(variable_cell=True) if variable else {}
            e0 = int(dev["edge_index"].shape[1])
            g = GraphedMDStep(model, dev, capacity=e0 // 2, **kw)  # too small: the first call re-captures
            cell = dev["cell"] * 1.01 if variable else None
            args = (pos1, cell) if variable else (pos1,)
            o1 = {k: v.clone() for k, v in g(*args).items()}
            assert g.recaptures == 1
            o2 = {k: v.clone() for k, v in g(dev["pos"], *((dev["cell"],) if variable else ())).items()}
            outs.append((o1, o2))
            del g
        monkeypatch.setattr(ops, "edge_pairs", real)
        for x, y in zip(outs[0], outs[1]):
            _same(x, y)
