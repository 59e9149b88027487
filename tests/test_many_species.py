"""Models with many atom types, on the host: the frames and per-type tables of the many-species tests
(tests/test_many_species_gpu.py), the relabelling of a model's types, and the number of N-tiles of each
self-connection launch.

The self-connection of an interaction layer is one grouped-GEMM launch of T x (instructions x irrep components)
problems (``SelfConnectionGemm``), so its N-tile count grows with the number of types T.  Once it exceeds the SM
count the grouped GEMM drops the cost-weighted split and each CTA owns N-tiles b, b + G, ... and sweeps every M-tile
of each (``Sched`` in nqb_gemm.cu).  The counts pinned below say which launches take that branch on a 132-SM H100.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

import edge_type_oracle as eto
from batched_oracle import concat_frames, energy_forces_stress
from cell_frames import cell_frame
from nequip_b200.nn.model import NequIPEnergyModel
from nequip_b200.nn.pair import ATOMIC_NUMBERS

R_MAX = 5.0
#: hydrogen to actinium: the 89 species of foundation-style models, so that ZBL has an atomic number for each
SPECIES_89 = list(ATOMIC_NUMBERS)[:89]
#: the bench model family (bench.py) and the l_max 3 model of test_model_gpu.py
BENCH = dict(l_max=2, num_layers=4, num_features=64, radial_mlp_depth=1, radial_mlp_width=128)
L3 = dict(l_max=3, num_layers=5, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)


def species_types(n: int, pool, seed: int, n_absent: int, n_single: int) -> torch.Tensor:
    """[n] int64 types drawn from ``pool`` (a list of type indices): ``n_absent`` types of the pool that no atom has,
    ``n_single`` types held by exactly one atom, and the smallest and the largest type of the pool present.  The
    other atoms draw uniformly from the remaining types, and the order is shuffled."""
    rng = np.random.default_rng(seed)
    pool = sorted(int(t) for t in pool)
    ends = [pool[0], pool[-1]]
    inner = [t for t in pool if t not in ends]
    pick = rng.permutation(inner)
    absent, single = pick[:n_absent], pick[n_absent:n_absent + n_single]
    common = np.array(sorted(set(pool) - set(absent.tolist()) - set(single.tolist())))
    rest = n - len(single) - len(ends)
    assert rest >= 0 and len(common) >= 2
    types = np.concatenate([single, ends, rng.choice(common, size=rest)])
    return torch.from_numpy(rng.permutation(types).astype(np.int64))


def many_species_frame(T: int, n_side: int, seed: int, cell: str = "tilted", n_absent: int = 0, n_single: int = 0,
                       pool=None):
    """The Li3PO4-density frame of ``cell_frame`` (atoms outside the cell) with its types redrawn over T species by
    ``species_types`` (from ``pool``, default all T); ``_meta`` names the types H, He, ... (``SPECIES_89[:T]``)."""
    fr = cell_frame("li3po4", n_side, cell, seed=seed, outside=True)
    n = fr["pos"].shape[0]
    fr["atom_types"] = species_types(n, range(T) if pool is None else pool, seed + 100, n_absent, n_single)
    fr["_meta"]["type_names"] = SPECIES_89[:T]
    return fr


def per_type_tables(T: int, ann: float, seed: int) -> dict:
    """T distinct values each of ``avg_num_neighbors`` (keyed by name), energy scales and energy shifts."""
    rng = np.random.default_rng(seed)
    names = SPECIES_89[:T]
    u = rng.permutation(T) / max(1, T - 1)
    return dict(avg_num_neighbors={nm: float(ann * (0.6 + 0.8 * u[t])) for t, nm in enumerate(names)},
                per_type_energy_scales=(0.5 + rng.permutation(T) / T).tolist(),
                per_type_energy_shifts=(0.1 * (rng.permutation(T) / T - 0.5)).tolist())


def table_spec(names, table) -> dict:
    """A [T, T] cutoff table as the model's ``per_edge_type_cutoff`` dict, every ordered pair keyed by name."""
    table = np.asarray(table, dtype=np.float64)
    return {a: {b: float(table[i, j]) for j, b in enumerate(names)} for i, a in enumerate(names)}


# ---------------------------------------------------------------------------------------------------------------
# relabelling: type t becomes type p[t]
# ---------------------------------------------------------------------------------------------------------------
def relabel_kwargs(kw: dict, p) -> dict:
    """Model keyword arguments for the relabelled types: every per-type list moved to its new index.  Tables keyed by
    name (``avg_num_neighbors``, ``per_edge_type_cutoff``) follow the names."""
    p = [int(v) for v in p]

    def move(seq):
        out = [None] * len(seq)
        for t, v in enumerate(seq):
            out[p[t]] = v
        return out

    kw = dict(kw)
    kw["type_names"] = move(kw["type_names"])
    for k in ("per_type_energy_scales", "per_type_energy_shifts"):
        if kw.get(k) is not None and not isinstance(kw[k], (int, float)):
            kw[k] = move(list(kw[k]))
    if kw.get("pair_potential") is not None:
        kw["pair_potential"] = dict(kw["pair_potential"], chemical_species=move(kw["pair_potential"]["chemical_species"]))
    return kw


def relabel_state(sd: dict, p) -> dict:
    """The state dict with every per-type entry moved to the new type indices: the type-embedding rows, the energy
    scales and shifts, the [T * T] reciprocal cutoff table and ZBL's atomic numbers."""
    p = torch.as_tensor(p, dtype=torch.int64)
    T = p.numel()
    out = dict(sd)

    def rows(t):
        r = torch.empty_like(t)
        r[p.to(t.device)] = t
        return r

    for k in ("type_embed.weight", "scales", "shifts", "pair_potential.atomic_numbers"):
        if k in sd and sd[k].numel():
            out[k] = rows(sd[k])
    if "rmax_recip" in sd:
        out["rmax_recip"] = rows(rows(sd["rmax_recip"].view(T, T)).t()).t().reshape(-1).contiguous()
    return out


def sc_ntiles(model, T: int):
    """[(layer index, forward N-tiles, backward N-tiles)] of every self-connection launch of ``model`` with T types,
    counted as ``SelfConnectionGemm`` lays out its problems (one per type, instruction and irrep component, each
    ceil(N / 128) tiles; N is the output width forward and the input width backward)."""
    out = []
    for li, layer in enumerate(model.layers):
        sc = layer.conv.sc
        if sc is None:
            continue
        fwd = bwd = 0
        for (i, o, _off, _pw) in sc.instr:
            mi, ir = sc.irreps_in[i]
            mo = sc.irreps_out[o][0]
            fwd += T * ir.dim * math.ceil(mo / 128)
            bwd += T * ir.dim * math.ceil(mi / 128)
        out.append((li, fwd, bwd))
    return out


# ---------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------
def test_species_are_hydrogen_to_actinium():
    assert len(SPECIES_89) == 89 and SPECIES_89[0] == "H" and SPECIES_89[-1] == "Ac"
    assert [ATOMIC_NUMBERS[s] for s in SPECIES_89] == list(range(1, 90))


@pytest.mark.parametrize("T,n_side,n_absent,n_single", [(8, 6, 2, 2), (89, 6, 12, 8), (5, 6, 1, 1), (89, 22, 4, 4)])
def test_frame_types_cover_the_edges_of_the_type_range(T, n_side, n_absent, n_single):
    """Absent types, types held by one atom, and types 0 and T - 1 present; the same seed gives the same frame."""
    t = species_types(n_side ** 3, range(T), seed=T + n_side, n_absent=n_absent, n_single=n_single)
    counts = torch.bincount(t, minlength=T)
    assert counts.numel() == T and int(t.min()) == 0 and int(t.max()) == T - 1
    assert int((counts == 0).sum()) >= n_absent and int((counts == 1).sum()) >= n_single
    assert counts[0] > 0 and counts[T - 1] > 0
    assert torch.equal(t, species_types(n_side ** 3, range(T), seed=T + n_side, n_absent=n_absent, n_single=n_single))


def test_disjoint_pools():
    a = species_types(125, range(0, 45), seed=1, n_absent=5, n_single=3)
    b = species_types(125, range(45, 89), seed=2, n_absent=5, n_single=3)
    assert set(a.tolist()).isdisjoint(b.tolist())
    assert 0 in a.tolist() and 88 in b.tolist()


def test_per_type_tables_are_distinct():
    tab = per_type_tables(89, 40.0, seed=0)
    for v in (list(tab["avg_num_neighbors"].values()), tab["per_type_energy_scales"], tab["per_type_energy_shifts"]):
        assert len(v) == 89 and len(set(v)) == 89


def _model(arch, T, **kw):
    return NequIPEnergyModel(r_max=R_MAX, type_names=SPECIES_89[:T], parity=True, **arch, **kw)


def test_self_connection_n_tiles():
    """N-tiles (forward / backward) of the self-connection launches of layers 1-3.  An H100 SXM has 132 SMs: the
    bench family takes the more-tiles-than-SMs branch in layer 2 from 8 types on, and in layers 1 and 2 at 89."""
    want = {3: [(1, 33, 27), (2, 57, 54), (3, 3, 3)],
            8: [(1, 88, 72), (2, 152, 144), (3, 8, 8)],
            89: [(1, 979, 801), (2, 1691, 1602), (3, 89, 89)]}
    for T, rows in want.items():
        assert sc_ntiles(_model(BENCH, T), T) == rows, T
    l3 = sc_ntiles(_model(L3, 5), 5)
    assert l3[1] == (2, 165, 160)


def test_relabelled_model_matches_in_float64_oracle():
    """The relabelling helpers are a symmetry of the float64 oracle (network, per-type tables, ZBL and per-edge-type
    cutoffs): what the device tests rely on when they compare a model with its relabelled copy."""
    T = 89
    fr = many_species_frame(T, 3, seed=4, n_absent=20, n_single=3)
    meta = fr.pop("_meta")
    table = eto.random_table(T, R_MAX, seed=3)
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], parity=True, l_max=1, num_layers=2, num_features=8,
              model_dtype=torch.float64, per_edge_type_cutoff=table_spec(meta["type_names"], table),
              pair_potential=dict(units="metal", chemical_species=list(meta["type_names"])),
              **per_type_tables(T, meta["avg_num_neighbors"], seed=1))
    m = NequIPEnergyModel(**kw)
    p = torch.from_numpy(np.random.default_rng(0).permutation(T))
    m2 = NequIPEnergyModel(**relabel_kwargs(kw, p))
    sd2 = relabel_state(m.state_dict(), p)
    for k in ("scales", "shifts", "rmax_recip", "pair_potential.atomic_numbers"):
        assert torch.equal(m2.state_dict()[k], sd2[k]), k  # the relabelled constructor builds the moved tables
    m2.load_state_dict(sd2)
    fr2 = dict(fr, atom_types=p[fr["atom_types"]])
    res = []
    for model, f, tab in ((m, fr, table), (m2, fr2, m2.per_edge_type_cutoff)):
        with eto.per_edge_cutoffs(eto.edge_recip(f["atom_types"], f["edge_index"], tab)):
            res.append(energy_forces_stress(model.state_dict(), model.config, concat_frames([f]), torch.float64))
    for a, b in zip(res[0], res[1]):
        assert float((a - b).abs().max()) <= 1e-12 * float(a.abs().max())
    # the relabelling moves something: the same types under the relabelled model give another energy
    with eto.per_edge_cutoffs(eto.edge_recip(fr["atom_types"], fr["edge_index"], m2.per_edge_type_cutoff)):
        e_wrong = energy_forces_stress(m2.state_dict(), m2.config, concat_frames([fr]), torch.float64)[0]
    assert float((e_wrong - res[0][0]).abs().max()) > 1e-3 * float(res[0][1].abs().sum())
