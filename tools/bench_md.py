#!/usr/bin/env python
"""MD step: eager neighbour list + model against the graphed step (``graph.GraphedMDStep``) on a moving frame.

Each workload follows the bounded trajectory ``data.oscillating_positions`` (0.2 A amplitude, period 50 steps), whose
edge count changes at most steps.  Positions start on the device; each step ends with the forces on the host, as in
a host-driven MD loop.
  A: ``ops.neighbor_list`` + ``model(d)`` (eager launches, one host synchronisation for the edge count), forces D2H;
  B: ``GraphedMDStep`` (one graph replay, 12-byte read-back of the edge count / overflow flag), forces D2H.
Arms are timed A, B, A, B in one process; every 10th step B's energy and forces are compared with A's at the same
positions.  ``pad`` lines time B on the frozen first frame with capacity E, 1.02 E and 1.05 E (the cost of the null
edges).  The first line names the GPU, its power limit and its maximum SM clock.

``--cell npt`` runs the same workloads with a cell that changes every step: ``cell(t) = cell0 @ S(t)`` and positions
``oscillating_positions(pos0, t) @ S(t)`` with ``S = data.oscillating_strain`` (I + eps, eps symmetric, 2 % diagonal and
3 % shear amplitude, period 50).  Positions and cells start on the device; each step ends with forces and stress on
the host.
  A: ``ops.neighbor_list`` + ``model(d, compute_stress=True)``;
  B: ``GraphedMDStep(variable_cell=True)``, ``g(pos, cell)``.
Timed A, B, A, B; every 10th step B's energy, forces and stress are compared with A's.  ``npt_overhead`` lines time the
fixed-cell graph against the variable-cell graph on the frozen first frame, alternated (the cost of the device
parameter block plus the stress).

``--cell open`` runs the open workloads (``OPEN_WORKLOADS``): the water_1k cube without a cell, a 21-atom cluster
cut from it (the launch-bound size of an aspirin molecule), and the 10 648-atom Li3PO4 frame on a tilted cell as a
slab (periodic along a and b, open along c), with the l_max 2 model and with preset S.  The trajectory is the bounded
one above plus a slow drift (``DRIFT`` A per step), so the bounding box moves.  Forces end on the host each step.
  A: ``ops.neighbor_list`` + ``model(d)`` without a cell (with the slab's cell and periodicity);
  B: ``GraphedMDStep`` with open directions (device bounding box, ``plan.cell`` in the captured call);
  C: ``GraphedMDStep`` in a periodic box with ``VACUUM`` A more than the frame's extent along each open direction
     (the cell the frame had to be put in before open directions were supported).
Timed A, B, C twice in one process; every 10th step B's (and C's) energy and forces are compared with A's.  An
``nl_open`` line times ``plan.run`` of B and C and ``nqb_nl_bbox`` alone with CUDA events.

    python tools/bench_md.py [--workloads water_1k_l2_f32,li3po4_10k_l2_f64,S_li3po4_10k] [--steps 100]
                             [--warmup 10] [--cell fixed|npt|open] [--out FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R_MAX = 5.0
PERIOD, AMPLITUDE = 50, 0.2
# name: (structure kind, n_side, model kwargs or a preset name) -- the first two are bench.py's workloads
WORKLOADS = {
    "water_1k_l2_f32": ("water", 10, dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1,
                                          radial_mlp_width=128)),
    "li3po4_10k_l2_f64": ("li3po4", 22, dict(l_max=2, num_layers=4, num_features=64, radial_mlp_depth=1,
                                             radial_mlp_width=128)),
    "S_li3po4_10k": ("li3po4", 22, "S"),
}
# name: (frame, model kwargs or a preset name) -- the frames of --cell open
OPEN_WORKLOADS = {
    "water_1k_open": ("water_cube", WORKLOADS["water_1k_l2_f32"][2]),
    "water_cluster_21_open": ("water_cluster", WORKLOADS["water_1k_l2_f32"][2]),
    "li3po4_10k_slab": ("li3po4_slab", WORKLOADS["li3po4_10k_l2_f64"][2]),
    "S_li3po4_10k_slab": ("li3po4_slab", "S"),
}
DRIFT = (0.011, -0.006, 0.017)  # A per step
VACUUM = R_MAX + 2.0
TILT = [[1.0, 0.0, 0.0], [0.3, 1.0, 0.0], [-0.2, 0.15, 1.0]]


def emit(line, sink):
    print(json.dumps(line), flush=True)
    sink.append(line)


def gpu_info():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    dev = torch.cuda.current_device()
    rows = [r.split(", ") for r in q.stdout.strip().splitlines()] if q.returncode == 0 else []
    row = next((r for r in rows if r and r[0] == str(dev)), None)
    return {"kind": "gpu", "name": torch.cuda.get_device_name(dev),
            "power_limit": row[2] if row else "not read", "max_sm_clock": row[3] if row else "not read"}


def build(workload):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.nn.model import NequIPEnergyModel

    kind, n_side, mk = WORKLOADS[workload]
    sysd = D.make_system(kind, n_side, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    model = (NequIPEnergyModel.from_preset(mk, **kw) if isinstance(mk, str)
             else NequIPEnergyModel(parity=True, **mk, **kw)).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    dev = D.to_device({k: sysd[k] for k in ("pos", "atom_types", "cell")}, "cuda")
    return model, dev, int(sysd["edge_index"].shape[1])


def arm_eager(model, dev, positions, keep):
    from nequip_b200 import ops

    kept, counts = {}, []
    for t, pos in enumerate(positions):
        nl = ops.neighbor_list(pos, dev["cell"], True, R_MAX)
        out = model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))
        f = out["forces"].cpu()
        counts.append(int(nl["edge_index"].shape[1]))
        if keep and t % 10 == 0:
            kept[t] = (float(out["total_energy"]), f)
    return kept, counts


def arm_graph(g, positions, keep):
    kept, counts = {}, []
    for t, pos in enumerate(positions):
        out = g(pos)
        f = out["forces"].cpu()
        counts.append(int(g._num_edges_host[0]))  # read back by the call itself
        if keep and t % 10 == 0:
            kept[t] = (float(out["total_energy"]), f)
    return kept, counts


def timed(fn, warm_positions, positions):
    import torch

    fn(warm_positions, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    kept, counts = fn(positions, True)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / len(positions), kept, counts


def run_workload(workload, steps, warmup, sink):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.graph import GraphedMDStep

    model, dev, E0 = build(workload)
    N = dev["pos"].shape[0]
    pos0 = dev["pos"].clone()
    positions = [D.oscillating_positions(pos0, t, PERIOD, AMPLITUDE, seed=1) for t in range(steps)]
    warm = [D.oscillating_positions(pos0, -1 - t, PERIOD, AMPLITUDE, seed=1) for t in range(warmup)]
    g = GraphedMDStep(model, dev)
    cap0 = g.capacity
    ms = {"A": [], "B": []}
    ref, got, counts = None, None, None
    for rep in range(2):
        t_a, ref, counts = timed(lambda p, k: arm_eager(model, dev, p, k), warm, positions)
        t_b, got, counts_b = timed(lambda p, k: arm_graph(g, p, k), warm, positions)
        if counts_b != counts:
            raise RuntimeError(f"{workload}: graphed edge counts differ from the eager list's")
        ms["A"].append(t_a)
        ms["B"].append(t_b)
        emit({"kind": "md_rep", "workload": workload, "rep": rep, "A_eager_ms_per_step": round(t_a, 4),
              "B_graph_ms_per_step": round(t_b, 4)}, sink)
    de, df = 0.0, 0.0
    for t, (e_a, f_a) in ref.items():
        e_b, f_b = got[t]
        de = max(de, abs(e_b - e_a) / abs(e_a))
        df = max(df, float((f_b - f_a).abs().max()) / float(f_a.abs().max()))
    changed = sum(a != b for a, b in zip(counts, counts[1:]))
    emit({"kind": "md", "workload": workload, "atoms": N, "E0": E0, "steps": steps, "period": PERIOD,
          "amplitude_A": AMPLITUDE, "A_eager_ms_per_step": [round(x, 4) for x in ms["A"]],
          "B_graph_ms_per_step": [round(x, 4) for x in ms["B"]],
          "speedup_B_over_A": round(min(ms["A"]) / min(ms["B"]), 3),
          "edge_count_changed_fraction": round(changed / (steps - 1), 4),
          "E_over_E0_min": round(min(counts) / E0, 5), "E_over_E0_max": round(max(counts) / E0, 5),
          "capacity_initial": cap0, "capacity_final": g.capacity, "recaptures": g.recaptures,
          "launches_per_replay": g.launches_per_replay, "checked_steps": len(ref),
          "max_rel_energy_dev_B_vs_A": de, "max_force_dev_B_vs_A_over_max_F": df}, sink)
    del g
    torch.cuda.empty_cache()
    # cost of the padding: B on the frozen first frame
    frozen = [pos0] * steps
    for slack in (0.0, 0.02, 0.05):
        cap = E0 + math.ceil(slack * E0)
        g = GraphedMDStep(model, dev, capacity=cap)
        t_pad, _, _ = timed(lambda p, k: arm_graph(g, p, False), [pos0] * warmup, frozen)
        emit({"kind": "pad", "workload": workload, "E": E0, "capacity": cap, "slack": slack,
              "B_graph_ms_per_step": round(t_pad, 4), "recaptures": g.recaptures}, sink)
        del g
        torch.cuda.empty_cache()


def arm_eager_npt(model, dev, frames, keep):
    from nequip_b200 import ops

    kept, counts = {}, []
    for t, (pos, cell) in enumerate(frames):
        nl = ops.neighbor_list(pos, cell, True, R_MAX)
        out = model(dict(dev, pos=pos, cell=cell, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]),
                    compute_stress=True)
        f, s = out["forces"].cpu(), out["stress"].cpu()
        counts.append(int(nl["edge_index"].shape[1]))
        if keep and t % 10 == 0:
            kept[t] = (float(out["total_energy"]), f, s)
    return kept, counts


def arm_graph_npt(g, frames, keep):
    kept, counts = {}, []
    for t, (pos, cell) in enumerate(frames):
        out = g(pos, cell)
        f, s = out["forces"].cpu(), out["stress"].cpu()
        counts.append(int(g._num_edges_host[0]))  # read back by the call itself
        if keep and t % 10 == 0:
            kept[t] = (float(out["total_energy"]), f, s)
    return kept, counts


def run_workload_npt(workload, steps, warmup, sink):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.graph import GraphedMDStep

    model, dev, E0 = build(workload)
    N = dev["pos"].shape[0]
    pos0, cell0 = dev["pos"].clone(), dev["cell"].clone()

    def frame(t):
        S = D.oscillating_strain(t, PERIOD).cuda()
        return D.oscillating_positions(pos0, t, PERIOD, AMPLITUDE, seed=1) @ S, cell0 @ S

    frames = [frame(t) for t in range(steps)]
    warm = [frame(-1 - t) for t in range(warmup)]
    g = GraphedMDStep(model, dev, variable_cell=True)
    cap0 = g.capacity
    ms = {"A": [], "B": []}
    ref, got, counts = None, None, None
    for rep in range(2):
        t_a, ref, counts = timed(lambda p, k: arm_eager_npt(model, dev, p, k), warm, frames)
        t_b, got, counts_b = timed(lambda p, k: arm_graph_npt(g, p, k), warm, frames)
        if counts_b != counts:
            raise RuntimeError(f"{workload}: graphed edge counts differ from the eager list's")
        ms["A"].append(t_a)
        ms["B"].append(t_b)
        emit({"kind": "npt_rep", "workload": workload, "rep": rep, "A_eager_ms_per_step": round(t_a, 4),
              "B_graph_ms_per_step": round(t_b, 4)}, sink)
    de, df, ds = 0.0, 0.0, 0.0
    for t, (e_a, f_a, s_a) in ref.items():
        e_b, f_b, s_b = got[t]
        de = max(de, abs(e_b - e_a) / abs(e_a))
        df = max(df, float((f_b - f_a).abs().max()) / float(f_a.abs().max()))
        ds = max(ds, float((s_b - s_a).abs().max()) / float(s_a.abs().max()))
    vols = [abs(float(torch.linalg.det(c))) for _p, c in frames]
    emit({"kind": "npt", "workload": workload, "atoms": N, "E0": E0, "steps": steps, "period": PERIOD,
          "amplitude_A": AMPLITUDE, "strain_diagonal": 0.02, "strain_shear": 0.03,
          "volume_over_V0_min": round(min(vols) / vols[0], 5), "volume_over_V0_max": round(max(vols) / vols[0], 5),
          "A_eager_ms_per_step": [round(x, 4) for x in ms["A"]],
          "B_graph_ms_per_step": [round(x, 4) for x in ms["B"]],
          "speedup_B_over_A": round(min(ms["A"]) / min(ms["B"]), 3),
          "E_over_E0_min": round(min(counts) / E0, 5), "E_over_E0_max": round(max(counts) / E0, 5),
          "capacity_initial": cap0, "capacity_final": g.capacity, "recaptures": g.recaptures,
          "launches_per_replay": g.launches_per_replay, "checked_steps": len(ref),
          "max_rel_energy_dev_B_vs_A": de, "max_force_dev_B_vs_A_over_max_F": df,
          "max_stress_dev_B_vs_A_over_max_stress": ds}, sink)
    del g
    torch.cuda.empty_cache()
    # cost of the variable cell: fixed-cell graph against variable-cell graph on the frozen first frame, alternated
    g_fixed = GraphedMDStep(model, dev)
    g_var = GraphedMDStep(model, dev, variable_cell=True)
    frozen = [(pos0, cell0)] * steps
    fixed_ms, var_ms = [], []
    for _rep in range(2):
        t_f, _, _ = timed(lambda p, k: arm_graph(g_fixed, [q for q, _c in p], False), frozen[:warmup], frozen)
        t_v, _, _ = timed(lambda p, k: arm_graph_npt(g_var, p, False), frozen[:warmup], frozen)
        fixed_ms.append(round(t_f, 4))
        var_ms.append(round(t_v, 4))
    emit({"kind": "npt_overhead", "workload": workload, "capacity_fixed": g_fixed.capacity,
          "capacity_variable": g_var.capacity, "fixed_cell_graph_ms_per_step": fixed_ms,
          "variable_cell_graph_ms_per_step": var_ms,
          "variable_over_fixed": round(min(var_ms) / min(fixed_ms), 3)}, sink)
    del g_fixed, g_var
    torch.cuda.empty_cache()


def build_open(workload):
    """Model, frame (``pos``, ``atom_types``, ``cell`` or None, ``pbc``) and the periodic-box frame of arm C."""
    import numpy as np
    import torch

    from nequip_b200 import data as D
    from nequip_b200.nn.model import NequIPEnergyModel

    kind, mk = OPEN_WORKLOADS[workload]
    sysd = D.make_system("water" if kind.startswith("water") else "li3po4", 10 if kind.startswith("water") else 22,
                         r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    pos, types = sysd["pos"].numpy(), sysd["atom_types"]
    if kind == "water_cluster":
        keep = np.sort(np.argsort(np.linalg.norm(pos - pos.mean(0), axis=1), kind="stable")[:21])
        pos, types = pos[keep], types[torch.from_numpy(keep)]
    if kind == "li3po4_slab":
        cell = np.asarray(TILT) @ sysd["cell"].numpy()
        pos = (pos @ np.linalg.inv(sysd["cell"].numpy())) @ cell
        pbc = (True, True, False)
        box = cell.copy()
        perp_c = 1.0 / np.linalg.norm(np.linalg.inv(cell)[:, 2])
        box[2] *= 1.0 + VACUUM / perp_c  # the slab spans at most perp_c along c
    else:
        cell, pbc = None, (False, False, False)
        box = np.diag(pos.max(0) - pos.min(0) + VACUUM)
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    model = (NequIPEnergyModel.from_preset(mk, **kw) if isinstance(mk, str)
             else NequIPEnergyModel(parity=True, **mk, **kw)).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    frame = {"pos": torch.from_numpy(pos.copy()).cuda(), "atom_types": types.cuda(),
             "cell": None if cell is None else torch.from_numpy(cell).cuda(), "pbc": pbc}
    boxed = {"pos": frame["pos"], "atom_types": frame["atom_types"], "cell": torch.from_numpy(box).cuda()}
    return model, frame, boxed


def arm_eager_open(model, frame, positions, keep):
    from nequip_b200 import ops

    kept, counts = {}, []
    for t, pos in enumerate(positions):
        nl = ops.neighbor_list(pos, frame["cell"], frame["pbc"], R_MAX)
        d = {"pos": pos, "atom_types": frame["atom_types"], "edge_index": nl["edge_index"]}
        if frame["cell"] is not None:
            d.update(cell=frame["cell"], edge_cell_shift=nl["edge_cell_shift"])
        out = model(d)
        f = out["forces"].cpu()
        counts.append(int(nl["edge_index"].shape[1]))
        if keep and t % 10 == 0:
            kept[t] = (float(out["total_energy"]), f)
    return kept, counts


def _event_ms(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def run_workload_open(workload, steps, warmup, sink):
    import torch

    from nequip_b200 import _capi
    from nequip_b200 import data as D
    from nequip_b200.graph import GraphedMDStep
    from nequip_b200.ops import _ptr

    model, frame, boxed = build_open(workload)
    N = frame["pos"].shape[0]
    pos0 = frame["pos"].clone()
    drift = torch.tensor(DRIFT, dtype=torch.float64, device="cuda")

    def at(t):
        return D.oscillating_positions(pos0, t, PERIOD, AMPLITUDE, seed=1) + t * drift

    positions = [at(t) for t in range(steps)]
    warm = [at(-1 - t) for t in range(warmup)]
    example = {"pos": frame["pos"], "atom_types": frame["atom_types"], "pbc": torch.tensor(frame["pbc"])}
    if frame["cell"] is not None:
        example["cell"] = frame["cell"]
    g_open = GraphedMDStep(model, example)
    g_box = GraphedMDStep(model, boxed)
    caps = (g_open.capacity, g_box.capacity)
    ms = {"A": [], "B": [], "C": []}
    for rep in range(2):
        t_a, ref, counts = timed(lambda p, k: arm_eager_open(model, frame, p, k), warm, positions)
        t_b, got, counts_b = timed(lambda p, k: arm_graph(g_open, p, k), warm, positions)
        t_c, got_c, counts_c = timed(lambda p, k: arm_graph(g_box, p, k), warm, positions)
        if counts_b != counts:
            raise RuntimeError(f"{workload}: graphed edge counts differ from the eager list's")
        for k, v in zip("ABC", (t_a, t_b, t_c)):
            ms[k].append(v)
        emit({"kind": "md_open_rep", "workload": workload, "rep": rep, "A_eager_ms_per_step": round(t_a, 4),
              "B_graph_open_ms_per_step": round(t_b, 4), "C_graph_box_ms_per_step": round(t_c, 4)}, sink)

    def devs(other):
        de, df = 0.0, 0.0
        for t, (e_a, f_a) in ref.items():
            e_b, f_b = other[t]
            de = max(de, abs(e_b - e_a) / abs(e_a))
            df = max(df, float((f_b - f_a).abs().max()) / float(f_a.abs().max()))
        return de, df

    (de_b, df_b), (de_c, df_c) = devs(got), devs(got_c)
    changed = sum(a != b for a, b in zip(counts, counts[1:]))
    emit({"kind": "md_open", "workload": workload, "atoms": N, "pbc": list(frame["pbc"]), "steps": steps,
          "period": PERIOD, "amplitude_A": AMPLITUDE, "drift_A_per_step": list(DRIFT), "vacuum_A": VACUUM,
          "A_eager_ms_per_step": [round(x, 4) for x in ms["A"]],
          "B_graph_open_ms_per_step": [round(x, 4) for x in ms["B"]],
          "C_graph_box_ms_per_step": [round(x, 4) for x in ms["C"]],
          "speedup_B_over_A": round(min(ms["A"]) / min(ms["B"]), 3),
          "speedup_B_over_C": round(min(ms["C"]) / min(ms["B"]), 3),
          "edge_count_changed_fraction": round(changed / (steps - 1), 4),
          "E_min": min(counts), "E_max": max(counts), "C_counts_equal_A": counts_c == counts,
          "capacity_initial_B_C": list(caps), "capacity_final_B_C": [g_open.capacity, g_box.capacity],
          "recaptures_B_C": [g_open.recaptures, g_box.recaptures],
          "launches_per_replay_B_C": [g_open.launches_per_replay, g_box.launches_per_replay],
          # the plans' host grids; along B's open directions that is the scratch grid (cap), of which the device
          # picks at most that many bins per step
          "bins_B": list(g_open.plan._a.nb), "bins_C": list(g_box.plan._a.nb), "checked_steps": len(ref),
          "max_rel_energy_dev_B_vs_A": de_b, "max_force_dev_B_vs_A_over_max_F": df_b,
          "max_rel_energy_dev_C_vs_A": de_c, "max_force_dev_C_vs_A_over_max_F": df_c}, sink)
    # the list alone: plan.run of both graphs' plans and the bounding box kernel, CUDA events
    p = positions[-1]
    L = _capi.lib()
    plan = g_open.plan
    bbox = lambda: _capi.check(L.nqb_nl_bbox(_ptr(p), N, _ptr(plan._params_dev), _ptr(plan._bbox_work),
                                             torch.cuda.current_stream().cuda_stream), "nqb_nl_bbox")
    emit({"kind": "nl_open", "workload": workload, "atoms": N,
          "B_plan_run_ms": [round(_event_ms(lambda: plan.run(p), 50), 4) for _ in range(2)],
          "C_plan_run_ms": [round(_event_ms(lambda: g_box.plan.run(p), 50), 4) for _ in range(2)],
          "bbox_ms": [round(_event_ms(bbox, 200), 5) for _ in range(2)]}, sink)
    del g_open, g_box
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=None, help="default: every workload of the chosen --cell")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--cell", choices=("fixed", "npt", "open"), default="fixed",
                    help="fixed: the cell of the first frame throughout; npt: a cell that changes every step; "
                         "open: molecules without a cell and slabs")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch

    torch.backends.cuda.matmul.allow_tf32 = False
    sink = []
    emit(gpu_info(), sink)
    runner = {"fixed": run_workload, "npt": run_workload_npt, "open": run_workload_open}[args.cell]
    names = args.workloads or ",".join(OPEN_WORKLOADS if args.cell == "open" else WORKLOADS)
    for w in names.split(","):
        runner(w, args.steps, args.warmup, sink)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            for line in sink:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
