"""Batches of frames with per-frame cells on the device: the batched neighbour list against frame-by-frame lists and
the brute-force list, the framed edge-embedding and ZBL kernels against per-frame calls, their write contracts,
whole models batched against frame by frame and against the float64 batched oracle, gradient isolation between
frames, a torch-sim-shaped input, and the unchanged single-cell paths."""
import math

import numpy as np
import pytest
import torch

import edge_type_oracle as eto
from batched_oracle import concat_frames, energy_forces_stress
from cell_frames import brute_list, cell_frame, named_cell
from kernel_contracts import guarded, is_poison
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.nn.model import NequIPEnergyModel
from nequip_b200.nn.pair import ZBL

pytestmark = pytest.mark.gpu

R_MAX = 5.0
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)  # water_1k family
TUTORIAL = dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2, radial_mlp_width=64)
LI3PO4_TABLE = {"Li": {"Li": 3.2, "O": 4.1}, "P": 3.6, "O": {"Li": 2.7, "O": 4.4}}


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) / float(b.abs().max())


def _strip(d):
    return {k: v for k, v in d.items() if k != "_meta"}


def _mixed_frames():
    """(frames, pbcs): the cubic, tilted, skewed, left and small cells, a slab (TTF), a molecule without a cell, a
    frame of one atom, a frame without edges and a frame without atoms."""
    fr, pbcs = [], []
    for s, name in enumerate(["cubic", "tilted", "skewed", "left"]):
        fr.append(_strip(cell_frame("li3po4", 3, name, seed=s, outside=True)))
        pbcs.append([True] * 3)
    fr.append(_strip(cell_frame("li3po4", 2, "small", seed=4, outside=True)))
    pbcs.append([True] * 3)
    fr.append(_strip(cell_frame("li3po4", 3, "tilted", seed=5, outside=True, pbc=(True, True, False))))
    pbcs.append([True, True, False])
    mol = _strip(cell_frame("li3po4", 3, "cubic", seed=6, pbc=False))
    mol.pop("cell")
    fr.append(mol)
    pbcs.append([False] * 3)
    one_cell = named_cell("small", 1)  # every width below r_max: the atom sees its own images
    ei, sh = brute_list(np.zeros((1, 3)), one_cell, True, R_MAX)
    fr.append({"pos": torch.zeros((1, 3), dtype=torch.float64), "cell": torch.from_numpy(one_cell.copy()),
               "atom_types": torch.tensor([1]), "edge_index": torch.from_numpy(ei), "edge_cell_shift": torch.from_numpy(sh)})
    pbcs.append([True] * 3)
    fr.append({"pos": torch.tensor([[0.0, 0.0, 0.0], [20.0, 1.0, -3.0]], dtype=torch.float64),
               "atom_types": torch.tensor([0, 2]), "edge_index": torch.zeros((2, 0), dtype=torch.int64),
               "edge_cell_shift": torch.zeros((0, 3), dtype=torch.float64)})
    pbcs.append([False] * 3)
    fr.append({"pos": torch.zeros((0, 3), dtype=torch.float64), "cell": torch.from_numpy(named_cell("cubic", 2)),
               "atom_types": torch.zeros(0, dtype=torch.int64), "edge_index": torch.zeros((2, 0), dtype=torch.int64),
               "edge_cell_shift": torch.zeros((0, 3), dtype=torch.float64)})
    pbcs.append([True] * 3)
    return fr, pbcs


def _concat_lists(outs, counts, with_perm):
    """The frame-by-frame lists as one: atom indices offset by each frame's first atom, edge positions by its first
    edge."""
    ei, sh, rp, perm = [], [], [], []
    a_off = e_off = 0
    for out, n in zip(outs, counts):
        if out is not None:
            ei.append(out["edge_index"] + a_off)
            sh.append(out["edge_cell_shift"])
            rp.append(out["row_ptr"][:-1] + e_off)
            if with_perm:
                perm.append(out["edge_transpose_perm"] + e_off)
            e_off += out["edge_index"].shape[1]
        a_off += n
    rp.append(torch.tensor([e_off], device="cuda"))
    res = {"edge_index": torch.cat(ei, 1), "edge_cell_shift": torch.cat(sh), "row_ptr": torch.cat(rp)}
    if with_perm:
        res["edge_transpose_perm"] = torch.cat(perm)
    return res


# ------------------------------------------------------------------------------------------------------------------
# batched neighbour list
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_perm", [False, True], ids=["no_perm", "perm"])
@pytest.mark.parametrize("T", [0, 3, 89], ids=["untyped", "T3", "T89"])
def test_batched_list_equals_frame_by_frame_lists(T, with_perm):
    frames, pbcs = _mixed_frames()
    b = concat_frames(frames, pbcs)
    counts = [d["pos"].shape[0] for d in frames]
    rng = np.random.default_rng(T)
    types = torch.from_numpy(rng.integers(0, max(T, 1), size=sum(counts)))
    typed = {}
    table = None
    if T:
        table = eto.random_table(T, R_MAX, seed=T)
        typed = dict(atom_types=types.cuda(), edge_type_cutoff=torch.from_numpy(table))
    pos = b["pos"].cuda()
    got = ops.neighbor_list(pos, b["cell"].cuda(), b["pbc"].cuda(), R_MAX, transpose_perm=with_perm,
                            batch=b["batch"].cuda(), **typed)
    outs, off = [], 0
    for d, p, n in zip(frames, pbcs, counts):
        if n == 0:
            outs.append(None)
            continue
        kw = {}
        if T:
            kw = dict(atom_types=types[off:off + n].cuda(), edge_type_cutoff=torch.from_numpy(table))
        outs.append(ops.neighbor_list(pos[off:off + n], d.get("cell"), p, R_MAX, transpose_perm=with_perm, **kw))
        off += n
    want = _concat_lists(outs, counts, with_perm)
    assert set(got) == set(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
    # the one-atom frame has edges to its own images, the frame of two distant atoms none
    assert got["edge_index"].shape[1] > 0
    # and against the brute-force list of each frame
    off = e_off = 0
    for d, p, n in zip(frames, pbcs, counts):
        if n == 0:
            continue
        x = d["pos"].numpy()
        cell = None if d.get("cell") is None else d["cell"].numpy()
        if T:
            ei, sh = eto.pruned_brute_list(x, cell, p, R_MAX, types[off:off + n].numpy(), table)
        else:
            ei, sh = brute_list(x, cell, p, R_MAX)
        E = ei.shape[1]
        assert np.array_equal(got["edge_index"][:, e_off:e_off + E].cpu().numpy(), ei + off)
        assert np.array_equal(got["edge_cell_shift"][e_off:e_off + E].cpu().numpy(), sh)
        off += n
        e_off += E
    assert e_off == got["edge_index"].shape[1]


def test_batched_list_write_contracts():
    """bin, count and fill of a batch write every element of their outputs and nothing outside them."""
    frames, pbcs = _mixed_frames()
    b = concat_frames(frames, pbcs)
    N = b["pos"].shape[0]
    ref = ops.neighbor_list(b["pos"].cuda(), b["cell"].cuda(), b["pbc"], R_MAX, batch=b["batch"])
    E = ref["edge_index"].shape[1]
    # the host arguments as neighbor_list builds them, then the three calls on guarded buffers
    F, pbc_np, cells = ops._nl_frame_args(b["cell"], b["pbc"], b["batch"], N)
    invs = np.linalg.inv(cells)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()  # noqa: E731
    pos, frame = b["pos"].cuda(), b["batch"].cuda()
    args = []
    for f in range(F):
        x = b["pos"][b["batch"] == f].numpy() @ invs[f]
        lo, width = np.zeros(3), np.ones(3)
        for d in range(3):
            if not pbc_np[f, d] and x.shape[0]:
                lo[d], width[d] = x[:, d].min(), max(x[:, d].max() - x[:, d].min(), 1e-9) * (1 + 1e-9)
        args.append(ops._NlArgs(x.shape[0], cells[f], invs[f], [bool(v) for v in pbc_np[f]], R_MAX, lo, width))
    cat = lambda k: [v for a in args for v in getattr(a, k)]  # noqa: E731
    I3, D9, D3 = ctypes_arrays(F)
    blocks = ctypes_buffer(F * int(L.nqb_nl_params_bytes()))
    _capi.check(L.nqb_nl_frames_pack(F, D9(*cells.reshape(-1)), D9(*invs.reshape(-1)), I3(*cat("pbc")), I3(*cat("nb")),
                                     I3(*cat("sr")), D3(*cat("lo")), D3(*cat("width")), R_MAX, blocks))
    blocks_dev = torch.frombuffer(bytearray(blocks.raw), dtype=torch.uint8).cuda()
    bin_base = torch.tensor(np.cumsum([0] + [a.nbins for a in args]), dtype=torch.int64).cuda()
    wpos, ck_w = guarded(N, 3, torch.float64)
    base, ck_b = guarded(N, 3, torch.int32)
    binid, ck_i = guarded(N, 1, torch.int64)
    cidx, ck_c = guarded(N, 3, torch.int32)
    fr = (p(blocks_dev), p(frame), p(bin_base))
    _capi.check(L.nqb_nl_bin_frames(p(pos), N, *fr, p(wpos), p(base), p(binid), p(cidx), st))
    torch.cuda.synchronize()
    for ck, t, what in ((ck_w, wpos, "wpos"), (ck_b, base, "base"), (ck_i, binid, "bin"), (ck_c, cidx, "cidx")):
        ck(what)
        assert not bool(is_poison(t).any()), what
    # every atom's bin lies in its frame's range
    lo, hi = bin_base[frame], bin_base[frame + 1]
    assert bool(((binid.view(-1) >= lo) & (binid.view(-1) < hi)).all())
    sorted_bin, order = torch.sort(binid.reshape(-1).clone(), stable=True)
    bin_start = torch.searchsorted(sorted_bin, torch.arange(int(bin_base[-1]) + 1, device="cuda"))
    counts, ck_n = guarded(N, 1, torch.int64)
    _capi.check(L.nqb_nl_count_frames(N, *fr, p(wpos), p(cidx), p(order), p(bin_start), 0, 0, 0, p(counts), st))
    torch.cuda.synchronize()
    ck_n("counts")
    assert torch.equal(counts.reshape(-1), ref["row_ptr"][1:] - ref["row_ptr"][:-1])
    ei, ck_e = guarded(2, E, torch.int64)
    sh, ck_s = guarded(E, 3, torch.float64)
    _capi.check(L.nqb_nl_fill_frames(N, E, *fr, p(wpos), p(cidx), p(base), p(order), p(bin_start),
                                     p(ref["row_ptr"]), 0, 0, 0, p(ei), p(sh), st))
    torch.cuda.synchronize()
    ck_e("edge_index")
    ck_s("shifts")
    assert torch.equal(ei, ref["edge_index"]) and torch.equal(sh, ref["edge_cell_shift"])


def ctypes_arrays(F):
    import ctypes as C

    return C.c_int * (3 * F), C.c_double * (9 * F), C.c_double * (3 * F)


def ctypes_buffer(n):
    import ctypes as C

    return C.create_string_buffer(n)


# ------------------------------------------------------------------------------------------------------------------
# framed edge-embedding and ZBL kernels
# ------------------------------------------------------------------------------------------------------------------
def _device_batch(seed=0):
    frames, pbcs = _mixed_frames()
    b = concat_frames(frames, pbcs)
    return frames, {k: v.cuda() for k, v in b.items()}


def _segments(frames):
    a = e = 0
    for d in frames:
        n, m = d["pos"].shape[0], d["edge_index"].shape[1]
        yield (a, a + n), (e, e + m)
        a, e = a + n, e + m


@pytest.mark.parametrize("typed", [False, True], ids=["untyped", "typed"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("lmax", [0, 1, 2, 3, 4])
def test_framed_embedding_is_bitwise_per_frame(lmax, dtype, typed):
    frames, b = _device_batch()
    E = b["edge_index"].shape[1]
    kw = dict(lmax=lmax, num_bessel=8, r_max=R_MAX, prefactor=2 * math.pi / R_MAX ** 2, out_dtype=dtype)
    table = torch.as_tensor(eto.random_table(3, R_MAX, seed=lmax), dtype=torch.float64)
    g = torch.Generator().manual_seed(lmax)
    gy = torch.randn(E, (lmax + 1) ** 2, generator=g, dtype=torch.float64).cuda()
    ge = torch.randn(E, 8, generator=g, dtype=torch.float64).cuda()

    def run(pos, ei, sh, cell, types, **extra):
        pos = pos.clone().requires_grad_(True)
        tk = dict(types=types, edge_type_recip=table.reciprocal().reshape(-1).cuda()) if typed else {}
        sink = {}
        v, y, emb = ops.edge_embed(pos, ei, sh, cell, edge_grad_sink=sink, **kw, **tk, **extra)
        return v, y, emb, sink, pos

    v, y, emb, sink, pos = run(b["pos"], b["edge_index"], b["edge_cell_shift"], b["cell"], b["atom_types"],
                               batch=b["batch"])
    ((y.double() * gy).sum() + (emb.double() * ge).sum()).backward()
    for f, ((a0, a1), (e0, e1)) in enumerate(_segments(frames)):
        if e1 == e0:
            continue
        vf, yf, ef, sf, pf = run(b["pos"][a0:a1], b["edge_index"][:, e0:e1] - a0, b["edge_cell_shift"][e0:e1],
                                 b["cell"][f], b["atom_types"][a0:a1])
        ((yf.double() * gy[e0:e1]).sum() + (ef.double() * ge[e0:e1]).sum()).backward()
        assert torch.equal(v[e0:e1], vf) and torch.equal(y[e0:e1], yf) and torch.equal(emb[e0:e1], ef), f
        assert torch.equal(sink["edge_vector_grad"][e0:e1], sf["edge_vector_grad"]), f
        # fp64 atomics: to rounding of the per-edge terms (the one-atom frame's images cancel to ~0)
        scale = max(float(pf.grad.abs().max()), float(sf["edge_vector_grad"].abs().max()))
        assert float((pos.grad[a0:a1] - pf.grad).abs().max()) <= 1e-12 * scale, f
    # E = 0
    _v0, y0, e0_ = ops.edge_embed(b["pos"], b["edge_index"][:, :0], b["edge_cell_shift"][:0], b["cell"],
                                  batch=b["batch"], **kw)
    assert y0.shape == (0, (lmax + 1) ** 2) and e0_.shape == (0, 8)


@pytest.mark.parametrize("typed", [False, True], ids=["untyped", "typed"])
def test_framed_zbl_matches_per_frame(typed):
    frames, b = _device_batch()
    zt = ZBL(["Li", "P", "O"], ["Li", "P", "O"], "metal", model_dtype=torch.float64).table("cuda")
    table = torch.as_tensor(eto.random_table(3, R_MAX, seed=7), dtype=torch.float64)
    tk = dict(edge_type_recip=table.reciprocal().reshape(-1).cuda()) if typed else {}

    def run(pos, ei, sh, cell, types, **extra):
        pos = pos.clone().requires_grad_(True)
        sink = {}
        e = ops.zbl_energy(pos, ei, types, zt, shift=sh, cell=cell, r_max=R_MAX, edge_grad_sink=sink, **tk, **extra)
        e.sum().backward()
        return e, sink, pos.grad

    e, sink, gpos = run(b["pos"], b["edge_index"], b["edge_cell_shift"], b["cell"], b["atom_types"], batch=b["batch"])
    assert float(e.detach().abs().max()) > 0
    for f, ((a0, a1), (e0, e1)) in enumerate(_segments(frames)):
        if a1 == a0:
            continue
        ef, sf, gf = run(b["pos"][a0:a1], b["edge_index"][:, e0:e1] - a0, b["edge_cell_shift"][e0:e1], b["cell"][f],
                         b["atom_types"][a0:a1])
        assert torch.equal(e[a0:a1], ef), f  # one warp per row, CSR order: bitwise
        if e1 > e0:
            want = sf["pair_edge_vector_grad"]
            assert float((sink["pair_edge_vector_grad"][e0:e1] - want).abs().max()) <= 1e-12 * float(want.abs().max())
            scale = max(float(gf.abs().max()), float(want.abs().max()))
            assert float((gpos[a0:a1] - gf).abs().max()) <= 1e-12 * scale, f
    # E = 0
    e_empty = ops.zbl_energy(b["pos"], b["edge_index"][:, :0], b["atom_types"], zt, shift=b["edge_cell_shift"][:0],
                             cell=b["cell"], batch=b["batch"], r_max=R_MAX)
    assert torch.equal(e_empty, torch.zeros_like(e_empty))


def test_framed_write_contracts():
    """Every output of nqb_edge_embed_fwd_frames, nqb_zbl_fwd_frames and nqb_zbl_bwd_frames fully written, nothing
    outside it; grad_pos accumulated into."""
    frames, b = _device_batch()
    N, E = b["pos"].shape[0], b["edge_index"].shape[1]
    recip = torch.as_tensor(eto.random_table(3, R_MAX, seed=2), dtype=torch.float64).reciprocal().reshape(-1).cuda()
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()  # noqa: E731
    geo = (p(b["pos"]), p(b["edge_index"]), p(b["edge_cell_shift"]), p(b["cell"]), p(b["batch"]))
    for typed in (False, True):
        ty = (p(b["atom_types"]), p(b["edge_index"]), p(recip), 3) if typed else (0, 0, 0, 0)
        for dt, code in ((torch.float32, 0), (torch.float64, 1)):
            vec, ck_v = guarded(E, 3, torch.float64)
            y, ck_y = guarded(E, 9, dt)
            emb, ck_e = guarded(E, 8, dt)
            _capi.check(L.nqb_edge_embed_fwd_frames(2, 8, R_MAX, 6.0, 1.0, *geo, N, E, *ty, code, p(vec), p(y),
                                                    p(emb), st))
            torch.cuda.synchronize()
            for ck, t, what in ((ck_v, vec, "vec"), (ck_y, y, "y"), (ck_e, emb, "emb")):
                ck(what)
                assert not bool(is_poison(t).any()), what
        zt = ZBL(["Li", "P", "O"], ["Li", "P", "O"], "metal", model_dtype=torch.float64).table("cuda")
        csr = ops.build_csr(b["edge_index"][0].contiguous(), N)
        zr = p(recip) if typed else 0
        e_atom, ck_a = guarded(N, 1, torch.float64)
        _capi.check(L.nqb_zbl_fwd_frames(*geo, p(b["atom_types"]), p(zt), 3, p(csr.row_ptr), 0, N, E, R_MAX, 6.0, 0,
                                         zr, p(e_atom), st))
        ga = torch.randn(N, device="cuda", dtype=torch.float64)
        gpos, ck_p = guarded(N, 3, torch.float64, body="random", generator=torch.Generator().manual_seed(3))
        base = gpos.detach().cpu().clone()
        gvec, ck_g = guarded(E, 3, torch.float64)
        _capi.check(L.nqb_zbl_bwd_frames(*geo, p(b["atom_types"]), p(zt), 3, N, E, R_MAX, 6.0, 0, zr, p(ga), p(gpos),
                                         p(gvec), st))
        torch.cuda.synchronize()
        for ck, what in ((ck_a, "e_atom"), (ck_p, "grad_pos"), (ck_g, "grad_vec")):
            ck(what)
        assert not bool(is_poison(e_atom).any()) and not bool(is_poison(gvec).any())
        ei = b["edge_index"].cpu()
        want = base.clone().index_add_(0, ei[1], gvec.cpu()).index_add_(0, ei[0], -gvec.cpu())
        assert float((gpos.cpu() - want).abs().max()) <= 1e-12 * float(want.abs().max())


# ------------------------------------------------------------------------------------------------------------------
# whole models
# ------------------------------------------------------------------------------------------------------------------
def _model(arch, names, dtype, ann, species=None, table=None):
    pp = None if species is None else {"units": "metal", "chemical_species": species}
    m = NequIPEnergyModel(parity=True, r_max=R_MAX, type_names=names, avg_num_neighbors=ann, model_dtype=dtype,
                          pair_potential=pp, per_edge_type_cutoff=table, strict_fast_path=(dtype == torch.float32),
                          **arch).cuda()
    for q in m.parameters():
        q.requires_grad_(False)
    return m


def _model_frames(kind):
    names = ["cubic", "tilted", "skewed", "left"]
    n_side = 4 if kind == "water" else 3
    fr = [cell_frame(kind, n_side, name, seed=10 + s, outside=True) for s, name in enumerate(names)]
    fr.append(cell_frame(kind, n_side, "tilted", seed=20, outside=True, pbc=(True, True, False)))
    meta = fr[0]["_meta"]
    pbcs = [[True] * 3] * 4 + [[True, True, False]]
    return [_strip(d) for d in fr], pbcs, meta


CASES = {
    "water_1k_l2_f32": ("water", WATER_L2, torch.float32, None, None, 2e-5),
    "water_l2_f64": ("water", WATER_L2, torch.float64, None, None, 1e-10),
    "tutorial_zbl_f32": ("li3po4", TUTORIAL, torch.float32, ["Li", "P", "O"], None, 2e-5),
    "tutorial_zbl_cutoffs_f64": ("li3po4", TUTORIAL, torch.float64, ["Li", "P", "O"], LI3PO4_TABLE, 1e-10),
    "tutorial_cutoffs_f32": ("li3po4", TUTORIAL, torch.float32, None, LI3PO4_TABLE, 2e-5),
}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("which", list(CASES))
def test_batched_model_matches_frame_by_frame(which):
    kind, arch, dtype, species, table, tol = CASES[which]
    frames, pbcs, meta = _model_frames(kind)
    model = _model(arch, meta["type_names"], dtype, meta["avg_num_neighbors"], species, table)
    b = {k: v.cuda() for k, v in concat_frames(frames, pbcs).items()}
    out = model(b, compute_stress=True)
    F = len(frames)
    assert out["total_energy"].shape == (F, 1)
    assert out["stress"].shape == out["virial"].shape == (F, 3, 3)
    a0 = 0
    for f, d in enumerate(frames):
        n = d["pos"].shape[0]
        ref = model(D.to_device(d, "cuda"), compute_stress=True)
        escale = max(1.0, float(ref["total_energy"].abs().max()))
        assert abs(float(out["total_energy"][f, 0]) - float(ref["total_energy"])) <= tol * escale, f
        assert _rel(out["atomic_energy"][a0:a0 + n], ref["atomic_energy"]) <= tol, f
        assert _rel(out["forces"][a0:a0 + n], ref["forces"]) <= tol, f
        for k in ("stress", "virial"):
            assert _rel(out[k][f], ref[k][0]) <= tol, (f, k)
        a0 += n
    if dtype == torch.float64 and table is None:
        # the float64 oracle on the whole batch
        e, ea, fo, so, vo = energy_forces_stress({k: v.cpu() for k, v in model.state_dict().items()}, model.config,
                                                 concat_frames(frames, pbcs), torch.float64)
        assert _rel(out["total_energy"], e) <= 1e-9 and _rel(out["atomic_energy"], ea) <= 1e-9
        assert _rel(out["forces"], fo) <= 1e-9
        assert _rel(out["stress"], so) <= 1e-9 and _rel(out["virial"], vo) <= 1e-9


@pytest.mark.parametrize("species", [None, ["Li", "P", "O"]], ids=["plain", "zbl"])
def test_gradient_of_one_frame_stays_in_that_frame(species):
    frames, pbcs, meta = _model_frames("li3po4")
    model = _model(TUTORIAL, meta["type_names"], torch.float32, meta["avg_num_neighbors"], species)
    b = {k: v.cuda() for k, v in concat_frames(frames, pbcs).items()}
    pos = b["pos"].clone().requires_grad_(True)
    out = model.energy(dict(b, pos=pos))
    (g,) = torch.autograd.grad([out["total_energy"][0, 0]], [pos])
    n0 = frames[0]["pos"].shape[0]
    assert float(g[:n0].abs().max()) > 0
    assert bool((g[n0:] == 0).all())


def test_torch_sim_input_runs_and_single_cell_paths_make_no_frames_call(monkeypatch):
    frames, pbcs, meta = _model_frames("li3po4")
    model = _model(TUTORIAL, meta["type_names"], torch.float32, meta["avg_num_neighbors"], ["Li", "P", "O"])
    cpu = concat_frames(frames, pbcs)
    # torch-sim's dict: cell [F, 3, 3], pbc [F, 3], batch, num_atoms; the list from the batched device list
    ts = {k: cpu[k].cuda().contiguous() for k in ("pos", "cell", "pbc", "batch", "num_atoms", "atom_types")}
    nl = ops.neighbor_list(ts["pos"], ts["cell"], ts["pbc"], R_MAX, batch=ts["batch"])
    out = model(dict(ts, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]), compute_stress=True)
    F = len(frames)
    assert out["total_energy"].shape == (F, 1) and out["forces"].shape == ts["pos"].shape
    assert out["stress"].shape == (F, 3, 3) and bool(torch.isfinite(out["stress"]).all())
    # a single frame, and a batch of frames that share one cell, never reach a _frames entry point
    L = _capi.lib()
    calls = []
    for name in [n for n in _capi.SIGNATURES if n.endswith("_frames") or n == "nqb_nl_frames_pack"]:
        def boom(*a, _n=name, **k):
            calls.append(_n)
            raise AssertionError(f"{_n} called")
        monkeypatch.setattr(L, name, boom)
    single = D.to_device(frames[1], "cuda")
    model(single, compute_stress=True)
    shared = concat_frames([frames[1], dict(frames[1], pos=frames[1]["pos"] + 0.05)])
    for cell in (shared["cell"][0], shared["cell"][:1]):
        d = {k: v.cuda() for k, v in shared.items()}
        d["cell"] = cell.cuda()
        r = model(d, compute_stress=True)
        assert r["stress"].shape == (2, 3, 3)
    assert calls == []
