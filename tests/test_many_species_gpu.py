"""Models with many atom types on the device, against float64 references.

Foundation-style models carry up to 89 species.  The self-connection of each interaction layer is one grouped-GEMM
launch of T x (instructions x irrep components) problems, row-masked by a one-hot [T, M] row scale and added onto
linear_2's output (``SelfConnectionGemm``).  From 8 types on, the bench family's layer-2 launch has more N-tiles than
an H100 has SMs, and at 89 types so has layer 1's (tests/test_many_species.py counts them): the grouped GEMM then
drops the cost-weighted split, and each CTA owns N-tiles b, b + G, ... and sweeps every M-tile of each.  Every test
that relies on that branch reads the launch it ran and checks it (``_assert_sweeping``).

* the launch pattern of the self-connection at the kernel level, element by element against float64;
* the bench family at 8 and 89 types and an l_max 3 model at 5 types against the float64 oracle, with per-type
  ``avg_num_neighbors``, energy scales and shifts (float32 fast path and float64 model);
* ZBL and an asymmetric 89 x 89 per-edge-type cutoff table;
* relabelling the types (with every per-type table) leaves energies and forces unchanged;
* the 10 648-atom bench frame with 89 types, float32 fast path against the float64 kernels;
* a batch of two frames with disjoint species, and a captured MD step.

The tests print each comparison's largest relative error next to its bound.
"""
import math

import pytest
import torch

import edge_type_oracle as eto
import kernel_contracts as kc
from batched_oracle import concat_frames, energy_forces_stress
from kernel_contracts import Guarded, assert_elementwise
from nequip_b200 import data as D
from nequip_b200 import ops
from nequip_b200.graph import GraphedMDStep
from nequip_b200.nn.model import NequIPEnergyModel
from test_many_species import (BENCH, L3, R_MAX, SPECIES_89, many_species_frame, per_type_tables, relabel_kwargs,
                               relabel_state, species_types, table_spec)

pytestmark = pytest.mark.gpu

F32, F64 = torch.float32, torch.float64


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max()) / float(b.detach().abs().max())


def _within(what, err, bound):
    print(f"{what}: {err:.2e} (bound {bound:.0e})")
    assert err <= bound, (what, err, bound)


def _assert_sweeping(model, layers):
    """The self-connection launches of ``layers``, forward and backward, have more N-tiles than the device has SMs
    and no cost-weighted split: each CTA owns several N-tiles and sweeps every M-tile of each."""
    for li in layers:
        blocks = model.layers[li].conv._tc_cache[1]
        assert blocks is not None and blocks["sc"] is not None, li
        for d, gg in (("fwd", blocks["sc"].fwd), ("bwd", blocks["sc"].bwd)):
            assert gg.ntiles_total > _sms() and gg.tile_ctas is None, (li, d, gg.ntiles_total, _sms())


# ---------------------------------------------------------------------------------------------------------------
# the launch pattern of the self-connection, element by element
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
def test_self_connection_launch_pattern_many_types():
    """One grouped launch per direction built as ``SelfConnectionGemm`` builds it: T = 89 types x instructions x irrep
    components, one-hot [T, M] row scale, ``skip_zero_rows``, out chunk 0 fed by two in chunks (``atomic``) and the
    others by one (``accumulate``), the backward with transposed weights.  K = 32, 64 and 132 / 160 mix resident and
    streamed weights, and the 132- and 160-wide chunks end in ragged N-tiles.  M = 5000 (40 M-tiles per N-tile, about
    five N-tiles per CTA).  Rows of no type (a zero one-hot column) hold NaN inputs and must stay bitwise equal to
    their base; every other element within ``kc.gemm_bound`` of float64, and no guard word touched."""
    T, M, n_none = 89, 5000, 37
    g = torch.Generator().manual_seed(89)
    fin = [(64, 1), (32, 3), (160, 1)]  # (multiplicity, irrep dimension) of each chunk
    fout = [(132, 1), (32, 3), (64, 1)]
    instr = [(0, 0, 0.5), (2, 0, -0.25), (1, 1, 0.7), (0, 2, 1.3)]  # (in chunk, out chunk, path weight)

    def offsets(ch):
        o = [0]
        for m, d in ch:
            o.append(o[-1] + m * d)
        return o

    in_off, out_off = offsets(fin), offsets(fout)
    d_in, d_out = in_off[-1], out_off[-1]
    ldi, ldo = d_in + 4, d_out + 8  # x and gx / out and gout: strided, sentinels in the gaps
    W = [torch.randn(T, fin[i][0], fout[o][0], generator=g) for (i, o, _s) in instr]
    fwd, bwd = [], []
    for n, (i, o, s) in enumerate(instr):
        mi, dim = fin[i]
        mo = fout[o][0]
        multi_o = sum(1 for (_i, o2, _s) in instr if o2 == o) > 1
        multi_i = sum(1 for (i2, _o, _s) in instr if i2 == i) > 1
        for t in range(T):
            for c in range(dim):
                a_off, c_off = in_off[i] + c * mi, out_off[o] + c * mo
                fwd.append(ops.GemmProblem(a_off, ldi, c_off, ldo, W[n][t], scale=s, accumulate=not multi_o,
                                           atomic=multi_o, rs_off=t, skip_zero_rows=True))
                bwd.append(ops.GemmProblem(c_off, ldo, a_off, ldi, W[n][t], scale=s, transposed=True,
                                           accumulate=not multi_i, atomic=multi_i, rs_off=t, skip_zero_rows=True))
    gf, gb = ops.GroupedGemm(fwd, "cuda"), ops.GroupedGemm(bwd, "cuda")
    for gg in (gf, gb):
        assert gg.ntiles_total >= 4 * _sms() and gg.tile_ctas is None, (gg.ntiles_total, _sms())

    typed = species_types(M - n_none, range(T), seed=5, n_absent=9, n_single=6)
    types = torch.cat([typed, torch.full((n_none,), -1)])[torch.randperm(M, generator=g)]
    none = types < 0
    onehot = torch.zeros(T, M)
    onehot[types[~none], torch.nonzero(~none).flatten()] = 1.0
    grs = Guarded(T, M, F32, body=onehot)

    def launch(gg, inp, lda, n_out, ldc, pairs):
        """Run ``gg`` on ``inp`` (row stride ``lda``) into a random base [M, n_out] (row stride ``ldc``) and check it
        against float64; the worst error / bound.  ``pairs``: (type, its rows, A's columns, C's columns, B [K, N],
        scale) of every problem whose type holds atoms."""
        ga = Guarded(M, inp.shape[1], F32, ld=lda, body=inp)
        gc = Guarded(M, n_out, F32, ld=ldc, body="random", generator=g)
        base = gc.initial.double()
        gg.run(ga.view, gc.view, M, rowscale=grs.view)
        torch.cuda.synchronize()
        ga.check_guards("A")
        grs.check_guards("rowscale")
        gc.check_guards("C")
        C = gc.view.cpu()
        assert torch.equal(C[none].view(torch.int32), gc.initial[none].view(torch.int32)), "a row of no type was written"
        ref, mag, bound = base.clone(), torch.zeros_like(base), torch.zeros_like(base)
        for t, rows, acols, ccols, B, s in pairs:
            A = inp[rows][:, acols]
            prod = A.double() @ B.double() * s
            ref[rows[:, None], ccols] += prod
            mag[rows[:, None], ccols] += prod.abs()
            bound[rows[:, None], ccols] += kc.gemm_bound(A, B, s)
        # the store / the adds onto the base (one or two red.global.add per element): fp32 rounding of each partial sum
        bound += 2.0 ** -22 * (base.abs() + mag)
        assert_elementwise(C[~none], ref[~none], bound[~none], "self-connection launch")
        return float(((C.double() - ref).abs()[~none] / bound[~none]).max())

    x = torch.randn(M, d_in, generator=g)
    x[none] = float("nan")
    gout = torch.randn(M, d_out, generator=g)
    gout[none] = float("nan")
    pf, pb = [], []
    for t in range(T):
        rows = torch.nonzero(types == t).flatten()
        if rows.numel() == 0:
            continue
        for n, (i, o, s) in enumerate(instr):
            mi, dim = fin[i]
            mo = fout[o][0]
            for c in range(dim):
                acols = torch.arange(in_off[i] + c * mi, in_off[i] + (c + 1) * mi)
                ccols = torch.arange(out_off[o] + c * mo, out_off[o] + (c + 1) * mo)
                pf.append((t, rows, acols, ccols, W[n][t], s))
                pb.append((t, rows, ccols, acols, W[n][t].t(), s))
    wf = launch(gf, x, ldi, d_out, ldo, pf)
    wb = launch(gb, gout, ldo, d_in, ldi, pb)
    print(f"self-connection launch, 89 types: worst err / bound forward {wf:.2f}, backward {wb:.2f} "
          f"({gf.ntiles_total} / {gb.ntiles_total} N-tiles on {_sms()} SMs, {math.ceil(M / 128)} M-tiles)")


# ---------------------------------------------------------------------------------------------------------------
# models against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
#: (architecture, T, absent types, types held by one atom, layers whose self-connection launches sweep)
CASES = {
    "bench_T8": (BENCH, 8, 2, 2, (2,)),
    "bench_T89": (BENCH, 89, 12, 8, (1, 2)),
    "l3_T5": (L3, 5, 1, 1, (2,)),
}


def _model(arch, T, dtype, ann, seed=0, table=None, zbl=False):
    names = SPECIES_89[:T]
    kw = dict(r_max=R_MAX, type_names=names, parity=True, model_dtype=dtype, strict_fast_path=(dtype == F32),
              per_edge_type_cutoff=None if table is None else table_spec(names, table),
              pair_potential=dict(units="metal", chemical_species=names) if zbl else None,
              **arch, **per_type_tables(T, ann, seed))
    return _frozen(NequIPEnergyModel(**kw)), kw


def _frozen(m):
    m = m.cuda()
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def _oracle(model, frames, dtype, pbcs=None):
    """Per-frame energies, per-atom energies, forces, stress and virial of the float64 batched oracle (the frame-by-
    frame oracle on the batch's edge vectors), under the model's per-edge-type cutoffs when it has a table."""
    b = concat_frames(frames, pbcs)
    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    if model.per_edge_type_cutoff is None:
        return energy_forces_stress(sd, model.config, b, dtype)
    with eto.per_edge_cutoffs(eto.edge_recip(b["atom_types"], b["edge_index"], model.per_edge_type_cutoff)):
        return energy_forces_stress(sd, model.config, b, dtype)


def _compare(what, out, ref, tol, a0=0, f=0):
    """Frame f of a model output against the oracle's frame f, whose atoms start at a0 of the oracle's batch.
    ``out``: the frame's per-atom energies and forces, the model's per-frame energies, stress and virial.  The energy
    is relative to sum |E_i|, the rest relative to their largest magnitude."""
    e, ea, fo, so, vo = ref
    sl = slice(a0, a0 + out["atomic_energy"].shape[0])
    _within(f"{what} energy", abs(float(out["total_energy"].view(-1)[f]) - float(e.view(-1)[f]))
            / float(ea[sl].abs().sum()), tol)
    _within(f"{what} atomic energies", _rel(out["atomic_energy"], ea[sl]), tol)
    _within(f"{what} forces", _rel(out["forces"], fo[sl]), tol)
    _within(f"{what} stress", _rel(out["stress"].view(-1, 3, 3)[f], so[f]), tol)
    _within(f"{what} virial", _rel(out["virial"].view(-1, 3, 3)[f], vo[f]), tol)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("dtype,tol", [(F32, 1e-5), (F64, 1e-9)], ids=["f32", "f64"])
@pytest.mark.parametrize("case", list(CASES))
def test_models_match_oracle(case, dtype, tol):
    """Energy, per-atom energies, forces, stress and virial against the oracle, with T distinct per-type
    ``avg_num_neighbors`` (linear_1's row scale), energy scales and energy shifts.  The float32 model runs the fast
    path, whose self-connection launches sweep; the float64 model runs the torch dense blocks, so it pins the per-type
    tables rather than the GEMM."""
    arch, T, n_absent, n_single, layers = CASES[case]
    fr = many_species_frame(T, 6, seed=T, n_absent=n_absent, n_single=n_single)
    meta = fr.pop("_meta")
    model, _kw = _model(arch, T, dtype, meta["avg_num_neighbors"], seed=T)
    out = model(D.to_device(fr, "cuda"), compute_stress=True)
    if dtype == F32:
        _assert_sweeping(model, layers)
    _compare(f"{case} {dtype}", out, _oracle(model, [fr], dtype), tol)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("which", ["zbl_f64", "network_f32"])
def test_zbl_and_cutoff_table_with_89_species(which):
    """An asymmetric 89 x 89 per-edge-type cutoff table.  ZBL between high-Z pairs dominates the forces and would hide
    a network error under a max |F| bound, so the ZBL model is checked in float64 and the float32 fast path on the
    network alone."""
    T = 89
    fr = many_species_frame(T, 6, seed=21, n_absent=12, n_single=8)
    meta = fr.pop("_meta")
    zbl = which == "zbl_f64"
    dtype, tol = (F64, 1e-9) if zbl else (F32, 1e-5)
    table = eto.random_table(T, R_MAX, seed=8)
    model, _kw = _model(BENCH, T, dtype, meta["avg_num_neighbors"], seed=3, table=table, zbl=zbl)
    assert torch.equal(model.per_edge_type_cutoff, torch.as_tensor(table))
    out = model(D.to_device(fr, "cuda"), compute_stress=True)
    if not zbl:
        _assert_sweeping(model, (1, 2))
    ref = _oracle(model, [fr], dtype)
    _compare(which, out, ref, tol)
    # the table prunes: a fifth of the r_max list lies at or beyond its pair's cutoff
    vec = fr["pos"][fr["edge_index"][1]] - fr["pos"][fr["edge_index"][0]] + fr["edge_cell_shift"] @ fr["cell"]
    x = vec.norm(dim=1) * eto.edge_recip(fr["atom_types"], fr["edge_index"], table).view(-1)
    assert float((x >= 1.0).double().mean()) > 0.2


@pytest.mark.timeout(900)
@pytest.mark.parametrize("which", ["network_f32", "zbl_f64"])
def test_relabelling_types_changes_nothing(which):
    """Type t becomes type p[t], and with it the type-embedding row, ``avg_num_neighbors``, the energy scale and
    shift, the cutoff table's rows and columns and ZBL's species: energies and forces agree to rounding.  A swapped
    ``T * t_i + t_j`` or a one-hot row of the wrong type would not."""
    T = 89
    fr = many_species_frame(T, 6, seed=33, n_absent=12, n_single=8)
    meta = fr.pop("_meta")
    zbl = which == "zbl_f64"
    dtype, tol = (F64, 1e-12) if zbl else (F32, 2e-6)
    model, kw = _model(BENCH, T, dtype, meta["avg_num_neighbors"], seed=5, table=eto.random_table(T, R_MAX, seed=9),
                       zbl=zbl)
    p = torch.randperm(T, generator=torch.Generator().manual_seed(2))
    m2 = _frozen(NequIPEnergyModel(**relabel_kwargs(kw, p)))
    sd2 = relabel_state(model.state_dict(), p)
    for k in ("scales", "shifts", "rmax_recip") + (("pair_potential.atomic_numbers",) if zbl else ()):
        assert torch.equal(m2.state_dict()[k], sd2[k]), k
    for l1, l2 in zip(model.layers, m2.layers):
        assert torch.equal(l2.conv.norm_const[p.cuda()], l1.conv.norm_const)
    m2.load_state_dict(sd2)
    dev = D.to_device(fr, "cuda")
    out = model(dev)
    out2 = m2(dict(dev, atom_types=p.cuda()[dev["atom_types"]]))
    if not zbl:
        _assert_sweeping(model, (1, 2))
        _assert_sweeping(m2, (1, 2))
    _within(f"relabelled {which} energy", abs(float(out["total_energy"]) - float(out2["total_energy"]))
            / float(out["atomic_energy"].abs().sum()), tol)
    _within(f"relabelled {which} atomic energies", _rel(out2["atomic_energy"], out["atomic_energy"]), tol)
    _within(f"relabelled {which} forces", _rel(out2["forces"], out["forces"]), tol)


# ---------------------------------------------------------------------------------------------------------------
# at scale, batched, captured
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_bench_frame_with_89_types_fp32_vs_fp64_kernels():
    """The 10 648-atom bench frame with its types redrawn over 89 species (about 120 atoms per type, 84 M-tiles per
    N-tile): the float32 fast path against the float64 kernels of the same weights at 1e-5, as
    test_model_gpu.py::test_bench_size_fp32_kernels_vs_fp64_kernels does for three types."""
    T = 89
    sysd = D.make_system("li3po4", 22, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    sysd["atom_types"] = species_types(sysd["pos"].shape[0], range(T), seed=7, n_absent=4, n_single=4)
    m32, kw = _model(BENCH, T, F32, meta["avg_num_neighbors"], seed=7)
    m64 = _frozen(NequIPEnergyModel(**dict(kw, model_dtype=F64, strict_fast_path=False)))
    m64.load_state_dict({k: v.double() if v.is_floating_point() else v for k, v in m32.state_dict().items()})
    dev = D.to_device(sysd, "cuda")
    out32 = m32(dev, compute_stress=True)
    _assert_sweeping(m32, (1, 2))
    out32 = {k: out32[k].clone() for k in ("total_energy", "atomic_energy", "forces", "stress", "virial")}
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out64 = m64(dev, compute_stress=True)
    ea = out64["atomic_energy"]
    _within("bench frame 89 types energy", abs(float(out32["total_energy"]) - float(out64["total_energy"]))
            / float(ea.abs().sum()), 1e-5)
    for k in ("atomic_energy", "forces", "stress", "virial"):
        _within(f"bench frame 89 types {k}", _rel(out32[k], out64[k]), 1e-5)


@pytest.mark.timeout(900)
def test_batch_of_frames_with_disjoint_species():
    """One batched call of two frames, types 0-44 and 45-88, against frame-by-frame calls and the float32 batched
    oracle."""
    T = 89
    frames, pbcs = [], [[True] * 3, [True] * 3]
    for s, (cell, pool) in enumerate((("tilted", range(0, 45)), ("cubic", range(45, 89)))):
        fr = many_species_frame(T, 5, seed=40 + s, cell=cell, n_absent=6, n_single=4, pool=pool)
        meta = fr.pop("_meta")
        frames.append(fr)
    assert set(frames[0]["atom_types"].tolist()).isdisjoint(frames[1]["atom_types"].tolist())
    model, _kw = _model(BENCH, T, F32, meta["avg_num_neighbors"], seed=11)
    b = {k: v.cuda() for k, v in concat_frames(frames, pbcs).items()}
    out = model(b, compute_stress=True)
    _assert_sweeping(model, (1, 2))
    assert out["total_energy"].shape == (2, 1) and out["stress"].shape == (2, 3, 3)
    ref = _oracle(model, frames, F32, pbcs)
    a0 = 0
    for f, d in enumerate(frames):
        n = d["pos"].shape[0]
        one = model(D.to_device(d, "cuda"), compute_stress=True)
        _within(f"batch frame {f} vs alone: energy", abs(float(out["total_energy"][f, 0]) - float(one["total_energy"]))
                / float(one["atomic_energy"].abs().sum()), 2e-5)
        for k in ("atomic_energy", "forces"):
            _within(f"batch frame {f} vs alone: {k}", _rel(out[k][a0:a0 + n], one[k]), 2e-5)
        for k in ("stress", "virial"):
            _within(f"batch frame {f} vs alone: {k}", _rel(out[k][f], one[k][0]), 2e-5)
        sub = {k: out[k][a0:a0 + n] for k in ("atomic_energy", "forces")}
        sub.update(total_energy=out["total_energy"], stress=out["stress"], virial=out["virial"])
        _compare(f"batch frame {f} vs oracle", sub, ref, 1e-5, a0=a0, f=f)
        a0 += n


@pytest.mark.timeout(900)
def test_graphed_md_step_with_89_types():
    """A captured MD step of the 89-type float32 model: replay against eager calls on the exact list, with the
    tolerances of test_md_step_gpu.py."""
    T = 89
    sysd = D.make_system("li3po4", 6, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    sysd["atom_types"] = species_types(sysd["pos"].shape[0], range(T), seed=13, n_absent=12, n_single=8)
    dev = D.to_device(sysd, "cuda")
    model, _kw = _model(BENCH, T, F32, meta["avg_num_neighbors"], seed=13)
    g = GraphedMDStep(model, dev)
    _assert_sweeping(model, (1, 2))
    pos0 = dev["pos"].clone()
    for t in range(4):
        pos = D.oscillating_positions(pos0, t, period=50, seed=7)
        out = {k: v.clone() for k, v in g(pos).items()}
        nl = ops.neighbor_list(pos, dev["cell"], True, R_MAX)
        ref = model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
        assert int(out["num_edges"]) == nl["edge_index"].shape[1]
        e_ref = float(ref["total_energy"])
        torch.testing.assert_close(out["total_energy"], ref["total_energy"], rtol=1e-12, atol=1e-9 * abs(e_ref))
        _within(f"captured step {t} forces", _rel(out["forces"], ref["forces"]), 2e-6)
