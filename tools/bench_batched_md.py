"""MD steps of a batch of frames: the eager batched list + model (arm A), one batched ``GraphedMDStep`` (arm B) and F
single-frame ``GraphedMDStep``s replayed in turn (arm C), over the same bounded trajectory.

Workloads (frame k has its own seed, and its own phase in ``data.oscillating_positions``):
  * water_125_x128      128 frames of a 125-atom water box (periodic), l_max 2, 4 layers, 32 features;
  * cluster_21_x64      64 clusters of the 21 water atoms nearest a box's centre, no cell, each drifting;
  * S_water_1k_x16      16 frames of the 1 000-atom water box, preset S;
  * water_125_x128_npt  the first workload at constant pressure: frame k's cell follows
                        ``data.oscillating_strain(t + 7 k)``, and every arm also returns per-frame stress.
Many small frames are what torch-sim batches, and where launch overhead and host read-backs dominate an eager step.

The three arms alternate over ROUNDS rounds in one process, each round timing ``--steps`` steps with CUDA events after
``--warmup`` steps; the card's name, power limit and max SM clock are read in the same process.  One JSON line per
(workload, arm, round) with ms per step of the whole batch and atom-steps/s, and one per workload with how far B is
from A at every 10th step: the largest per-frame energy difference, the largest force difference over max|F| and, for
NPT, the largest stress difference.

    python tools/bench_batched_md.py [--workloads ...] [--steps 100] [--warmup 10] [--out FILE.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nequip_b200 import data as D  # noqa: E402
from nequip_b200 import ops  # noqa: E402
from nequip_b200.graph import GraphedMDStep  # noqa: E402
from nequip_b200.nn.model import NequIPEnergyModel  # noqa: E402

ROUNDS = 3
R_MAX = 5.0
PERIOD, AMPLITUDE = 50, 0.2
DRIFT = (0.013, -0.007, 0.021)
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)
WORKLOADS = {
    # name: (kind, frames, n_side, preset, npt)
    "water_125_x128": ("water", 128, 5, None, False),
    "cluster_21_x64": ("cluster", 64, 10, None, False),
    "S_water_1k_x16": ("water", 16, 10, "S", False),
    "water_125_x128_npt": ("water", 128, 5, None, True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def frames(kind, count, n_side, dev):
    """[(pos, cell or None, atom_types)] on ``dev``: water boxes strained by up to +-2 % (frame k from seed k), or the
    21 atoms nearest the centre of water box k without a cell."""
    out = []
    for k in range(count):
        s = D.make_system("water", n_side, r_max=R_MAX, seed=k)
        meta = s["_meta"]
        if kind == "cluster":
            pos = s["pos"].numpy()
            keep = np.sort(np.argsort(np.linalg.norm(pos - pos.mean(0), axis=1), kind="stable")[:21])
            out.append((torch.from_numpy(pos[keep].copy()), None, s["atom_types"].view(-1)[torch.from_numpy(keep)]))
        else:
            eps = np.random.default_rng(1000 + k).uniform(-0.02, 0.02, size=(3, 3))
            m = torch.from_numpy(np.eye(3) + 0.5 * (eps + eps.T))
            out.append((s["pos"].double() @ m, s["cell"].double().view(3, 3) @ m, s["atom_types"].view(-1)))
    return [tuple(None if t is None else t.to(dev) for t in f) for f in out], meta


def model_for(preset, meta, dev):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    m = (NequIPEnergyModel.from_preset(preset, **kw) if preset
         else NequIPEnergyModel(parity=True, **WATER_L2, **kw)).to(dev)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batched_md.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    gpu = card()
    lines = []

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for name in args.workloads.split(","):
        kind, count, n_side, preset, npt = WORKLOADS[name]
        fr, meta = frames(kind, count, n_side, dev)
        model = model_for(preset, meta, dev)
        counts = [f[0].shape[0] for f in fr]
        atoms = sum(counts)
        periodic = kind != "cluster"
        batch = torch.repeat_interleave(torch.arange(count, device=dev), torch.tensor(counts, device=dev))
        types = torch.cat([f[2] for f in fr])
        cells0 = torch.stack([f[1] for f in fr]) if periodic else torch.eye(3, dtype=torch.float64,
                                                                            device=dev).expand(count, 3, 3).clone()
        pbc = torch.tensor([[periodic] * 3] * count)
        drift = torch.tensor(DRIFT, dtype=torch.float64, device=dev)
        starts = np.cumsum([0] + counts)

        def at(t):
            """(pos [N, 3], cells [F, 3, 3]) of step t."""
            pos, cells = [], []
            for k, (p0, c0, _) in enumerate(fr):
                p = D.oscillating_positions(p0, t, PERIOD, AMPLITUDE, seed=k)
                c = cells0[k]
                if npt:
                    s = D.oscillating_strain(t + 7 * k, PERIOD).to(dev)
                    p, c = p @ s, c0 @ s
                elif not periodic:
                    p = p + t * drift * (1 + k % 3)
                pos.append(p)
                cells.append(c)
            return torch.cat(pos), torch.stack(cells)

        steps = [at(t) for t in range(args.steps)]
        warm = [at(-1 - t) for t in range(args.warmup)]
        example = {"pos": steps[0][0], "atom_types": types, "batch": batch, "num_atoms": torch.tensor(counts, device=dev),
                   "cell": cells0, "pbc": pbc}
        if not periodic:
            example.pop("cell")

        def arm_a(pos, cells):
            nl = ops.neighbor_list(pos, cells if periodic else None, pbc, R_MAX, batch=batch)
            d = {"pos": pos, "atom_types": types, "batch": batch, "num_atoms": example["num_atoms"], "cell": cells,
                 "edge_index": nl["edge_index"], "edge_cell_shift": nl["edge_cell_shift"]}
            return model(d, compute_stress=npt)

        g_b = GraphedMDStep(model, example, variable_cell=npt)

        def arm_b(pos, cells):
            return g_b(pos, cells) if npt else g_b(pos)

        g_c = []
        for k, (p0, c0, t0) in enumerate(fr):
            ex = {"pos": p0, "atom_types": t0}
            if periodic:
                ex["cell"] = c0
            g_c.append(GraphedMDStep(model, ex, variable_cell=npt, warmup=1))

        def arm_c(pos, cells):
            for k, g in enumerate(g_c):
                p = pos[starts[k]:starts[k + 1]]
                g(p, cells[k]) if npt else g(p)

        # B against A at every 10th step
        de = df = ds = 0.0
        for t in range(0, args.steps, 10):
            ra, rb = arm_a(*steps[t]), {k: v.clone() for k, v in arm_b(*steps[t]).items()}
            de = max(de, float((rb["total_energy"] - ra["total_energy"]).abs().max()))
            df = max(df, float((rb["forces"] - ra["forces"]).abs().max() / ra["forces"].abs().max()))
            if npt:
                ds = max(ds, float((rb["stress"] - ra["stress"]).abs().max()))
        rec = {"workload": name, "what": "b_vs_a", "frames": count, "atoms": atoms, "steps_checked": len(
            range(0, args.steps, 10)), "max_frame_energy_diff": de, "max_force_diff_over_max_f": df,
            "capacity_b": g_b.capacity, "recaptures_b": g_b.recaptures}
        if npt:
            rec["max_stress_diff"] = ds
        emit(rec)
        arms = (("A_eager_batched", arm_a), ("B_graphed_batched", arm_b), ("C_graphed_per_frame", arm_c))
        for r in range(ROUNDS):
            for arm, fn in arms:
                for s in warm:
                    fn(*s)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for s in steps:
                    fn(*s)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / len(steps)
                emit({"workload": name, "what": "npt_step" if npt else "md_step", "arm": arm, "round": r,
                      "frames": count, "atoms": atoms, "steps": len(steps), "ms_per_step": ms,
                      "atom_steps_per_s": atoms / (ms * 1e-3)})
        del model, fr, g_b, g_c, steps, warm
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
