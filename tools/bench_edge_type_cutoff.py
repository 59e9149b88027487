"""Per-edge-type cutoffs on bench.py's default frame and model (Li3PO4, 10 648 atoms, l_max 2, 4 layers, 64 features).

The table (TABLE below, rc[source, target] in A, r_max 5) keeps r_max for O-O and cuts every pair with Li or P to 4 A.
Reported, one JSON line each, with the card's name, power limit and max SM clock read in the same process:
  * E of the r_max list and of the pruned list;
  * the device list (NeighborListPlan.run: bins, sort, count, scan, pad, fill) without and with the table, alternated
    over ROUNDS rounds of LAUNCHES runs;
  * the graphed MD step (GraphedMDStep, STEPS steps of data.oscillating_positions) of the model without the table and
    of the same weights with it, on their own lists, alternated over ROUNDS rounds.

    python tools/bench_edge_type_cutoff.py [--out FILE.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nequip_b200 import data as D  # noqa: E402
from nequip_b200 import ops  # noqa: E402
from nequip_b200.graph import GraphedMDStep  # noqa: E402
from nequip_b200.nn.model import NequIPEnergyModel  # noqa: E402

ROUNDS, LAUNCHES, STEPS = 5, 20, 100
R_MAX = 5.0
TABLE = {"Li": 4.0, "P": 4.0, "O": {"Li": 4.0, "P": 4.0}}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    dev = torch.device("cuda")
    gpu = card()
    sysd = D.make_system("li3po4", 22, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    d = D.to_device(sysd, dev)
    N = d["pos"].shape[0]
    models = {}
    for arm, table in (("global", None), ("table", TABLE)):
        m = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=2, num_layers=4, num_features=64,
                              parity=True, radial_mlp_depth=1, radial_mlp_width=128,
                              avg_num_neighbors=meta["avg_num_neighbors"], strict_fast_path=True,
                              per_edge_type_cutoff=table).to(dev)
        for p in m.parameters():
            p.requires_grad_(False)
        models[arm] = m
    tab = models["table"].per_edge_type_cutoff
    lines = []

    def emit(rec):
        rec.update(gpu=gpu, table=TABLE, r_max=R_MAX, N=N)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    kw = {"global": {}, "table": dict(atom_types=d["atom_types"], edge_type_cutoff=tab)}
    E = {arm: int(ops.neighbor_list(d["pos"], d["cell"], True, R_MAX, **kw[arm])["edge_index"].shape[1])
         for arm in kw}
    emit({"what": "edges", "E_global": E["global"], "E_pruned": E["table"], "ratio": E["table"] / E["global"]})

    plans = {arm: ops.NeighborListPlan(N, d["cell"], True, R_MAX, E[arm] + E[arm] // 50, **kw[arm]) for arm in kw}
    for arm in plans:
        timed(lambda: plans[arm].run(d["pos"]), 3)
    for r in range(ROUNDS):
        for arm in ("global", "table"):
            ms = timed(lambda: plans[arm].run(d["pos"]), LAUNCHES)
            emit({"what": "neighbor_list_plan_run", "arm": arm, "round": r, "ms": ms, "E": E[arm]})

    steps = {arm: GraphedMDStep(models[arm], d) for arm in models}
    pos0 = d["pos"].clone()
    traj = [D.oscillating_positions(pos0, t, period=50, seed=7) for t in range(STEPS)]
    for arm in steps:
        for t in range(5):
            steps[arm](traj[t])
    torch.cuda.synchronize()
    for r in range(ROUNDS):
        for arm in ("global", "table"):
            g = steps[arm]

            def run():
                for t in range(STEPS):
                    g(traj[t])

            ms = timed(run, 1) / STEPS
            emit({"what": "graphed_md_step", "arm": arm, "round": r, "ms_per_step": ms, "steps": STEPS,
                  "capacity": g.capacity, "recaptures": g.recaptures, "E_last": int(g.num_edges)})
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
