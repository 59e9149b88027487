"""Nose-Hoover MD trajectories: the update in torch on the host around ``GraphedMDStep`` (arm A, what a user writes
today) against ``GraphedMD``, which captures the update with the step and reads from the host once per block of
1, 10 or 100 steps (arms B, C, D).

Workloads:
  * water_1k_l2_f32   the 1 000-atom water box, l_max 2, 4 layers, 32 features (tools/bench_md.py);
  * S_li3po4_10k      preset S on the 10 k-atom Li3PO4 frame (tools/bench_md.py);
  * cluster_21_x64    64 clusters of 21 water atoms without a cell, one batch (tools/bench_batched_md.py).
Small systems and batches are where a per-step host read and a handful of eager torch ops could be a visible share
of the step; the 10 k frame is where they should not be.

Every arm integrates at 0.5 fs, 300 K, nvt_q 334 (the reference's docstring example) from the same initial state.
The arms alternate over ROUNDS rounds in one process; each round times ``--steps`` steps with CUDA events after
``--warmup`` steps, continuing the arm's own trajectory.  The card's name, power limit and max SM clock are read in
the same process.  One JSON line per (workload, arm, round) with ms per step, and one per workload comparing A and C
over ``--check-steps`` steps from one state: the largest position difference and the largest per-frame difference
of the potential energy and of the conserved quantity.

    python tools/bench_md_run.py [--workloads ...] [--steps 200] [--warmup 20] [--out FILE.jsonl]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_batched_md as BB  # noqa: E402
import bench_md as BM  # noqa: E402
from nequip_b200 import md  # noqa: E402
from nequip_b200.graph import GraphedMDStep  # noqa: E402

ROUNDS = 3
TIMESTEP_FS, TEMPERATURE, NVT_Q = 0.5, 300.0, 334.0
MASS = {"H": 1.008, "O": 15.999, "Li": 6.94, "P": 30.974}
WORKLOADS = ("water_1k_l2_f32", "S_li3po4_10k", "cluster_21_x64")
ARMS = (("A_host_update", None), ("B_block_1", 1), ("C_block_10", 10), ("D_block_100", 100))


def workload(name, dev):
    """(model, example, masses per type)."""
    if name == "cluster_21_x64":
        kind, count, n_side, preset, _ = BB.WORKLOADS[name]
        fr, meta = BB.frames(kind, count, n_side, dev)
        model = BB.model_for(preset, meta, dev)
        counts = [f[0].shape[0] for f in fr]
        ex = {"pos": torch.cat([f[0] for f in fr]).double(), "atom_types": torch.cat([f[2] for f in fr]),
              "batch": torch.repeat_interleave(torch.arange(count, device=dev), torch.tensor(counts, device=dev)),
              "num_atoms": torch.tensor(counts, device=dev), "pbc": torch.zeros(count, 3, dtype=torch.bool)}
    else:
        model, ex, _ = BM.build(name)
        ex = dict(ex, pos=ex["pos"].double())
        meta = {"type_names": model.config["type_names"]}
    return model, ex, [MASS[t] for t in meta["type_names"]]


class HostUpdate:
    """Arm A: ``GraphedMDStep`` for the forces and the reference's update (``NoseHoover.step``) in eager torch."""

    def __init__(self, model, ex, m):
        self.g = GraphedMDStep(model, ex)
        s = m.state
        self.pos, self.vel, self.f = s["pos"].clone(), s["vel"].clone(), s["forces"].clone()
        self.zeta, self.eta = s["zeta"].clone(), s["eta"].clone()
        self.mass, self.dt, self.gkT, self.Q = m._mass.unsqueeze(1), m.dt, m._gkT, m._Q
        counts = (m._atom_ptr[1:] - m._atom_ptr[:-1])
        self.frame = torch.repeat_interleave(torch.arange(m.num_frames, device=counts.device), counts)
        self.F = m.num_frames

    def _sum(self, v):
        return torch.zeros(self.F, dtype=torch.float64, device=v.device).index_add_(0, self.frame,
                                                                                     (self.mass * v * v).sum(1))

    def step(self):
        dt, z = self.dt, self.zeta[self.frame].unsqueeze(1)
        acc = self.f / self.mass - z * self.vel
        self.pos = self.pos + dt * self.vel + 0.5 * dt * dt * acc
        vh = self.vel + 0.5 * dt * acc
        zh = self.zeta + 0.5 * dt * (0.5 * (self._sum(self.vel) - self.gkT)) / self.Q
        zn = zh + 0.5 * dt * (0.5 * (self._sum(vh) - self.gkT)) / self.Q
        self.eta = self.eta + 0.5 * dt * (self.zeta + zn)
        self.zeta = zn
        out = self.g(self.pos)
        self.f = out["forces"].double().clone()
        self.vel = (vh + 0.5 * dt * self.f / self.mass) / (1 + 0.5 * dt * zn[self.frame].unsqueeze(1))
        e = out["total_energy"].double().view(-1).clone()
        return e + 0.5 * self._sum(self.vel) + self.Q * self.zeta ** 2 + self.gkT * self.eta, e

    def run(self, n):
        for _ in range(n):
            self.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--check-steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_md_run.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    gpu = BM.gpu_info()
    lines = []

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for name in args.workloads.split(","):
        model, ex, masses = workload(name, dev)
        kw = dict(thermostat="nose_hoover", temperature=TEMPERATURE, nvt_q=NVT_Q)
        atoms, frames = ex["pos"].shape[0], int(ex["num_atoms"].numel()) if "num_atoms" in ex else 1
        # A against C over the same steps from one state
        c = md.GraphedMD(model, ex, masses, TIMESTEP_FS, **kw)
        a = HostUpdate(model, ex, c)
        log = c.run(args.check_steps, block=10)
        h_a, e_a = zip(*[a.step() for _ in range(args.check_steps)])
        h_a, e_a = torch.stack(h_a).cpu(), torch.stack(e_a).cpu()
        emit({"workload": name, "what": "a_vs_c", "atoms": atoms, "frames": frames, "steps": args.check_steps,
              "max_pos_diff": float((a.pos - c.state["pos"]).abs().max()),
              "max_e_pot_diff": float((e_a - log["e_pot"]).abs().max()),
              "max_conserved_diff": float((h_a - log["conserved"]).abs().max()),
              "conserved_drift_c": float((log["conserved"] - log["conserved"][0]).abs().max()),
              "e_kin_0": float(log["e_kin"][0].max())})
        arms = {"A_host_update": a}
        for arm, block in ARMS[1:]:
            arms[arm] = md.GraphedMD(model, ex, masses, TIMESTEP_FS, **kw)
        for r in range(ROUNDS):
            for arm, block in ARMS:
                obj = arms[arm]
                go = (lambda n: obj.run(n)) if block is None else (lambda n: obj.run(n, block=block))
                go(args.warmup)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                go(args.steps)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                rec = {"workload": name, "what": "nvt_step", "arm": arm, "round": r, "atoms": atoms, "frames": frames,
                       "steps": args.steps, "ms_per_step": ms, "atom_steps_per_s": atoms / (ms * 1e-3)}
                if block is not None:
                    rec.update(block=block, host_reads=obj.host_reads, recaptures=obj.recaptures)
                emit(rec)
        del model, ex, arms, a, c
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
