#!/usr/bin/env python
"""Cost of the ZBL pair potential (``nqb_zbl_fwd`` / ``nqb_zbl_bwd``), in one process:

* ``kernel`` lines: the two kernels alone on the bench frame (Li3PO4-like, 10 648 atoms, 588 616 edges), CUDA events
  around ``--launches`` launches after warm-up; bytes counted from the shapes (every input read once, every output
  written once; grad_pos read and written) and the fraction of the H100 SXM data-sheet 3.35 TB/s;
* ``torch`` lines: the same term in torch on the device (``oracle.pair.zbl_atom_energy`` on CUDA tensors, forward and
  forward + autograd backward), timed the same way;
* ``md`` lines: ``GraphedMDStep`` without (A) and with (B) ZBL, same weights, on the bounded trajectory of
  ``tools/bench_md.py``, timed A, B, A, B; every 10th step B's energy and forces are compared with the eager model
  with ZBL at the same positions.

The first line names the GPU, its power limit and its maximum SM clock.

    python tools/bench_zbl.py [--steps 100] [--warmup 10] [--launches 200] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import bench_md  # noqa: E402  (gpu_info, timed, arm_graph, arm_eager: the MD step harness)

HBM_BYTES_PER_S = 3.35e12
R_MAX = bench_md.R_MAX
SPECIES = {"water": ["H", "O"], "li3po4": ["Li", "P", "O"]}
# name: (structure kind, n_side, model kwargs or a preset name)
WORKLOADS = {
    "water_1k_l2_f32": bench_md.WORKLOADS["water_1k_l2_f32"],
    "S_li3po4_10k": bench_md.WORKLOADS["S_li3po4_10k"],
    "tutorial_water_1k": ("water", 10, dict(l_max=1, num_layers=4, num_features=32, radial_mlp_depth=2,
                                            radial_mlp_width=64)),
}


def event_ms(fn, launches, warmup=10):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def run_kernels(launches, sink):
    import torch

    from nequip_b200 import _capi, ops
    from nequip_b200 import data as D
    from nequip_b200.nn.pair import ZBL
    from oracle import pair as opair

    sysd = D.make_system("li3po4", 22, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    dev = D.to_device(sysd, "cuda")
    N, E = dev["atom_types"].numel(), dev["edge_index"].shape[1]
    m = ZBL(meta["type_names"], SPECIES["li3po4"], "metal", model_dtype=torch.float32).cuda()
    table = m.table(dev["pos"].device)
    csr = ops.build_csr(dev["edge_index"][0].contiguous(), N)
    L, st = _capi.lib(), torch.cuda.current_stream().cuda_stream
    geom = (dev["pos"].data_ptr(), dev["edge_index"].data_ptr(), dev["edge_cell_shift"].data_ptr(),
            dev["cell"].data_ptr(), 0, dev["atom_types"].data_ptr(), table.data_ptr(), table.shape[0])
    e_atom = torch.empty(N, dtype=torch.float64, device="cuda")
    ge = torch.ones(N, dtype=torch.float64, device="cuda")
    gpos = torch.zeros(N, 3, dtype=torch.float64, device="cuda")
    gvec = torch.empty(E, 3, dtype=torch.float64, device="cuda")

    def fwd():
        _capi.check(L.nqb_zbl_fwd(*geom, csr.row_ptr.data_ptr(), 0, N, E, R_MAX, 6.0, 1, e_atom.data_ptr(), st))

    def bwd(with_vec):
        _capi.check(L.nqb_zbl_bwd(*geom, N, E, R_MAX, 6.0, 1, ge.data_ptr(), gpos.data_ptr(),
                                  gvec.data_ptr() if with_vec else 0, st))

    # bytes from shapes: pos [N,3] f64, edge_index [2,E] i64, shifts [E,3] f64, types [N] i64, row_ptr [N+1] i64
    geom_bytes = N * 24 + E * 16 + E * 24 + N * 8
    rows = [("nqb_zbl_fwd", fwd, geom_bytes + (N + 1) * 8 + N * 8),
            ("nqb_zbl_bwd", lambda: bwd(False), geom_bytes + N * 8 + 2 * N * 24),
            ("nqb_zbl_bwd+grad_vec", lambda: bwd(True), geom_bytes + N * 8 + 2 * N * 24 + E * 24)]
    for name, fn, nbytes in rows:
        ms = event_ms(fn, launches)
        bench_md.emit({"kind": "kernel", "kernel": name, "atoms": N, "edges": E, "launches": launches,
                       "us": round(ms * 1e3, 2), "bytes": nbytes, "bytes_per_edge": round(nbytes / E, 1),
                       "hbm_fraction": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 4)}, sink)
    # the same term in torch on the device (the oracle's op sequence, float32 model dtype)
    pos = dev["pos"].clone().requires_grad_(True)
    Z, qq, ei, types = m.atomic_numbers, m._qqr2exesquare, dev["edge_index"], dev["atom_types"]
    from oracle import model as omodel

    def torch_fwd():
        with torch.no_grad():
            vec = omodel.edge_vectors(pos, ei, dev["cell"], dev["edge_cell_shift"])
            opair.zbl_atom_energy(Z, qq, 6.0, R_MAX, vec, types, ei, N, torch.float32)

    def torch_fwd_bwd():
        vec = omodel.edge_vectors(pos, ei, dev["cell"], dev["edge_cell_shift"])
        e = opair.zbl_atom_energy(Z, qq, 6.0, R_MAX, vec, types, ei, N, torch.float32)
        torch.autograd.grad(e.sum(), pos)

    t_fwd = event_ms(torch_fwd, max(20, launches // 4))
    t_both = event_ms(torch_fwd_bwd, max(20, launches // 4))
    k_fwd = event_ms(fwd, launches)
    k_both = k_fwd + event_ms(lambda: bwd(False), launches)
    # agreement of the kernels with the torch term on this frame
    fwd()
    ref = opair.zbl_atom_energy(Z, qq, 6.0, R_MAX, omodel.edge_vectors(dev["pos"], ei, dev["cell"],
                                                                       dev["edge_cell_shift"]),
                                types, ei, N, torch.float32).view(-1)
    dev_rel = float((e_atom - ref).abs().max() / ref.abs().max())
    bench_md.emit({"kind": "torch", "atoms": N, "edges": E, "torch_fwd_us": round(t_fwd * 1e3, 1),
                   "torch_fwd_bwd_us": round(t_both * 1e3, 1), "kernels_fwd_us": round(k_fwd * 1e3, 2),
                   "kernels_fwd_bwd_us": round(k_both * 1e3, 2),
                   "speedup_fwd_bwd": round(t_both / k_both, 2), "max_rel_dev_e_atom_vs_torch": dev_rel}, sink)


def build_pair(workload):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.nn.model import NequIPEnergyModel

    kind, n_side, mk = WORKLOADS[workload]
    sysd = D.make_system(kind, n_side, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    zbl = {"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": SPECIES[kind]}
    models = []
    for pp in (None, zbl):  # same seed: the same network weights
        m = (NequIPEnergyModel.from_preset(mk, pair_potential=pp, **kw) if isinstance(mk, str)
             else NequIPEnergyModel(parity=True, pair_potential=pp, **mk, **kw)).cuda()
        for p in m.parameters():
            p.requires_grad_(False)
        models.append(m)
    dev = D.to_device({k: sysd[k] for k in ("pos", "atom_types", "cell")}, "cuda")
    return models, dev, int(sysd["edge_index"].shape[1])


def run_md(workload, steps, warmup, sink):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.graph import GraphedMDStep

    (m_a, m_b), dev, E0 = build_pair(workload)
    pos0 = dev["pos"].clone()
    positions = [D.oscillating_positions(pos0, t, bench_md.PERIOD, bench_md.AMPLITUDE, seed=1) for t in range(steps)]
    warm = [D.oscillating_positions(pos0, -1 - t, bench_md.PERIOD, bench_md.AMPLITUDE, seed=1) for t in range(warmup)]
    g_a, g_b = GraphedMDStep(m_a, dev), GraphedMDStep(m_b, dev)
    ms = {"A": [], "B": []}
    got = None
    for rep in range(2):
        t_a, _, _ = bench_md.timed(lambda p, k: bench_md.arm_graph(g_a, p, k), warm, positions)
        t_b, got, _ = bench_md.timed(lambda p, k: bench_md.arm_graph(g_b, p, k), warm, positions)
        ms["A"].append(t_a)
        ms["B"].append(t_b)
    ref, _ = bench_md.arm_eager(m_b, dev, positions, True)
    de, df = 0.0, 0.0
    for t, (e_r, f_r) in ref.items():
        e_g, f_g = got[t]
        de = max(de, abs(e_g - e_r) / abs(e_r))
        df = max(df, float((f_g - f_r).abs().max()) / float(f_r.abs().max()))
    bench_md.emit({"kind": "md", "workload": workload, "atoms": int(pos0.shape[0]), "E0": E0, "steps": steps,
                   "A_graph_ms_per_step": [round(x, 4) for x in ms["A"]],
                   "B_graph_zbl_ms_per_step": [round(x, 4) for x in ms["B"]],
                   "zbl_overhead": round(min(ms["B"]) / min(ms["A"]) - 1.0, 4),
                   "launches_per_replay_A": g_a.launches_per_replay, "launches_per_replay_B": g_b.launches_per_replay,
                   "checked_steps": len(ref), "max_rel_energy_dev_B_graph_vs_eager": de,
                   "max_force_dev_B_graph_vs_eager_over_max_F": df}, sink)
    del g_a, g_b
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_zbl.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    sink = []
    bench_md.emit(bench_md.gpu_info(), sink)
    run_kernels(a.launches, sink)
    for w in a.workloads.split(","):
        run_md(w, a.steps, a.warmup, sink)
    if a.out:
        with open(a.out, "w") as f:
            for line in sink:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
