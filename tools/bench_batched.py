"""Batched inference of independent frames: one batched neighbour list and one model call for all frames (arm B)
against a loop of per-frame lists and model calls (arm A), both eager, forces and stress included.

Workloads (every frame with its own seed and a cell strained by a random symmetric strain of up to +-2 %):
  * water_1k_l2_f32  32 frames of the 1 000-atom water box, l_max 2, 4 layers, 32 features (bench_md's model);
  * water_125_l2_f32 128 frames of a 125-atom water box, the same model;
  * S_water_1k       16 frames of the 1 000-atom water box, preset S.
Small frames are where launch overhead dominates a step, and batching is what amortises it; the 1 000-atom frames show
where that stops mattering.

A and B alternate over ROUNDS rounds in one process, each timed over REPS calls with CUDA events; the card's name, power
limit and max SM clock are read in the same process.  One JSON line per (workload, arm, round) with ms per batch and
atom-steps/s, and one per workload with how far B is from A: the largest per-frame energy difference, the largest
force difference over max|F| and the largest stress difference.

    python tools/bench_batched.py [--workloads water_1k_l2_f32,water_125_l2_f32,S_water_1k] [--out FILE.jsonl]
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
from nequip_b200.nn.model import NequIPEnergyModel  # noqa: E402

ROUNDS, REPS = 5, 3
R_MAX = 5.0
WATER_L2 = dict(l_max=2, num_layers=4, num_features=32, radial_mlp_depth=1, radial_mlp_width=128)
WORKLOADS = {
    "water_1k_l2_f32": (32, 10, None),
    "water_125_l2_f32": (128, 5, None),
    "S_water_1k": (16, 10, "S"),
}


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


def frames(count: int, n_side: int, dev):
    """``count`` water frames of n_side^3 atoms, frame k from seed k, strained by a symmetric strain with entries in
    [-0.02, 0.02]: (pos, cell, atom_types) on ``dev``."""
    out = []
    for k in range(count):
        s = D.make_system("water", n_side, r_max=R_MAX, seed=k)
        eps = np.random.default_rng(1000 + k).uniform(-0.02, 0.02, size=(3, 3))
        m = torch.from_numpy(np.eye(3) + 0.5 * (eps + eps.T))
        out.append((s["pos"].double() @ m, s["cell"].double().view(3, 3) @ m, s["atom_types"].view(-1)))
        meta = s["_meta"]
    return [tuple(t.to(dev) for t in f) for f in out], meta


def model_for(preset, meta, dev):
    kw = dict(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
              strict_fast_path=True)
    m = (NequIPEnergyModel.from_preset(preset, **kw) if preset
         else NequIPEnergyModel(parity=True, **WATER_L2, **kw)).to(dev)
    for p in m.parameters():
        p.requires_grad_(False)
    return m


def arm_a(model, fr):
    """One list and one model call per frame."""
    outs = []
    for pos, cell, types in fr:
        nl = ops.neighbor_list(pos, cell, True, R_MAX)
        outs.append(model({"pos": pos, "cell": cell, "atom_types": types, "edge_index": nl["edge_index"],
                           "edge_cell_shift": nl["edge_cell_shift"]}, compute_stress=True))
    return outs


def arm_b(model, batch):
    """One batched list and one model call for every frame."""
    nl = ops.neighbor_list(batch["pos"], batch["cell"], True, R_MAX, batch=batch["batch"])
    return model(dict(batch, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]), compute_stress=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_batched.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    gpu = card()
    lines = []

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for name in args.workloads.split(","):
        count, n_side, preset = WORKLOADS[name]
        fr, meta = frames(count, n_side, dev)
        model = model_for(preset, meta, dev)
        counts = [f[0].shape[0] for f in fr]
        batch = {"pos": torch.cat([f[0] for f in fr]), "cell": torch.stack([f[1] for f in fr]),
                 "atom_types": torch.cat([f[2] for f in fr]),
                 "batch": torch.repeat_interleave(torch.arange(count, device=dev), torch.tensor(counts, device=dev)),
                 "num_atoms": torch.tensor(counts, device=dev)}
        atoms = sum(counts)
        # warm-up (kernel libraries, allocator) and the accuracy check of B against A
        outs_a, out_b = arm_a(model, fr), arm_b(model, batch)
        arm_a(model, fr), arm_b(model, batch)
        e_a = torch.cat([o["total_energy"].view(1) for o in outs_a])
        f_a = torch.cat([o["forces"] for o in outs_a])
        s_a = torch.cat([o["stress"] for o in outs_a])
        emit({"workload": name, "what": "b_vs_a", "frames": count, "atoms": atoms,
              "max_frame_energy_diff": float((out_b["total_energy"].view(-1) - e_a).abs().max()),
              "max_force_diff_over_max_f": float((out_b["forces"] - f_a).abs().max() / f_a.abs().max()),
              "max_stress_diff": float((out_b["stress"] - s_a).abs().max()),
              "max_abs_stress": float(s_a.abs().max())})
        for r in range(ROUNDS):
            for arm, fn in (("A_per_frame", lambda: arm_a(model, fr)), ("B_batched", lambda: arm_b(model, batch))):
                ms = timed(fn, REPS)
                emit({"workload": name, "what": "eager_forces_stress", "arm": arm, "round": r, "frames": count,
                      "atoms": atoms, "ms_per_batch": ms, "atom_steps_per_s": atoms / (ms * 1e-3), "reps": REPS})
        del model, fr, batch, outs_a, out_b
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
