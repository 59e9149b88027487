"""FIRE relaxations: ``GraphedMDStep`` plus the FIRE / Frechet-filter update in eager torch with a host ``set_cell``
every step (arm A, what a user writes today) against ``GraphedRelax`` with blocks of 1 and 50 steps (arms B, C).

Workloads:
  * S_water125_x64_frechet  64 rattled (0.05 Angstrom) water boxes of 125 atoms strained by up to +-2 %, preset S,
                            with the Frechet cell filter;
  * S_li3po4_10k_frechet    the rattled 10 k-atom Li3PO4 frame, preset S, with the filter;
  * S_water125_x64          the batch with the positions only.

Per workload and arm: ms per FIRE step over ``--steps`` steps after ``--warmup`` (at fmax = 1e-9, so no frame stops; a moving cell can
overflow the edge capacity, and the re-captures that follow are inside the timed window and counted in the line),
then a relaxation to fmax = 0.05 eV/Angstrom (at most ``--max-steps``) giving the steps each frame took and the
relaxed energies; one line compares the arms' relaxed energies.  The card's name and power limit are read in the same
process.

    python tools/bench_relax.py [--workloads ...] [--steps 50] [--warmup 5] [--max-steps 1500] [--out FILE.jsonl]
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
from nequip_b200.graph import GraphedMDStep  # noqa: E402
from nequip_b200.relax import FIRE_DEFAULTS, GraphedRelax  # noqa: E402

WORKLOADS = ("S_water125_x64_frechet", "S_li3po4_10k_frechet", "S_water125_x64")
ARMS = (("A_host_update", None), ("B_block_1", 1), ("C_block_50", 50))
FMAX = 0.05


def workload(name, dev):
    """(model, batched example, use the filter)."""
    g = torch.Generator().manual_seed(0)
    if name.startswith("S_water125_x64"):
        fr, meta = BB.frames("water", 64, 5, dev)
        model = BB.model_for("S", meta, dev)
        counts = [f[0].shape[0] for f in fr]
        pos = torch.cat([f[0] for f in fr]).double()
        ex = {"pos": pos, "atom_types": torch.cat([f[2] for f in fr]), "cell": torch.stack([f[1] for f in fr]),
              "batch": torch.repeat_interleave(torch.arange(64, device=dev), torch.tensor(counts, device=dev)),
              "num_atoms": torch.tensor(counts, device=dev)}
    else:
        model, d, _ = BM.build("S_li3po4_10k")
        N = d["pos"].shape[0]
        ex = {"pos": d["pos"].double(), "atom_types": d["atom_types"].view(-1), "cell": d["cell"].double().view(1, 3, 3),
              "batch": torch.zeros(N, dtype=torch.int64, device=dev), "num_atoms": torch.tensor([N], device=dev)}
    ex["pos"] = ex["pos"] + 0.05 * torch.randn(ex["pos"].shape, generator=g, dtype=torch.float64).to(dev)
    return model, ex, name.endswith("frechet")


class HostFire:
    """Arm A: the forces (and virial) of ``GraphedMDStep``, ASE's FIRE and FrechetCellFilter in eager torch on the
    device, a host ``set_cell`` inside every step with the filter, and one host read per step for the stop test."""

    def __init__(self, model, ex, filt, fmax):
        self.g = GraphedMDStep(model, ex, variable_cell=filt)
        self.filt, self.fmax = filt, fmax
        counts = ex["num_atoms"].long()
        self.frame = ex["batch"].long()
        F = counts.numel()
        dev = ex["pos"].device
        self.F, self.c = F, counts.double().clamp_min(1)
        self.s = ex["pos"].double().clone()
        self.C0 = ex["cell"].double().clone()
        self.Q = torch.zeros(F, 3, 3, dtype=torch.float64, device=dev)
        self.v = torch.zeros_like(self.s)
        self.vc = torch.zeros_like(self.Q)
        self.dt = torch.full((F,), FIRE_DEFAULTS["dt"], dtype=torch.float64, device=dev)
        self.a = torch.full((F,), FIRE_DEFAULTS["a"], dtype=torch.float64, device=dev)
        self.n = torch.zeros(F, dtype=torch.int64, device=dev)
        self.first = True
        self.done = torch.zeros(F, dtype=torch.bool, device=dev)
        self.steps = torch.zeros(F, dtype=torch.int64, device=dev)
        self.energy = None
        self._eval()

    def _fsum(self, x):
        return torch.zeros(self.F, dtype=torch.float64, device=x.device).index_add_(0, self.frame, x)

    def _eval(self):
        Fd = torch.matrix_exp(self.Q / self.c.view(-1, 1, 1)) if self.filt else None
        if self.filt:
            cell = self.C0 @ Fd.transpose(1, 2)
            pos = torch.einsum("ni,nji->nj", self.s, Fd[self.frame])
            out = self.g(pos, cell)
            f = out["forces"].double()
            self.ga = torch.einsum("ni,nij->nj", f, Fd[self.frame])
            W = out["virial"].double()  # p = 0
            M = W @ torch.linalg.inv(Fd).transpose(1, 2)
            L = (self.Q / self.c.view(-1, 1, 1)).transpose(1, 2)
            Z = torch.zeros(self.F, 6, 6, dtype=torch.float64, device=L.device)
            Z[:, :3, :3] = Z[:, 3:, 3:] = L
            Z[:, :3, 3:] = M
            self.gc = torch.matrix_exp(Z)[:, :3, 3:] / self.c.view(-1, 1, 1)
            m = torch.maximum(torch.zeros(self.F, dtype=torch.float64, device=L.device).index_reduce_(
                0, self.frame, (self.ga ** 2).sum(1), "amax"), (self.gc ** 2).sum(2).amax(1))
        else:
            out = self.g(self.s)
            self.ga = out["forces"].double()
            m = torch.zeros(self.F, dtype=torch.float64, device=self.s.device).index_reduce_(
                0, self.frame, (self.ga ** 2).sum(1), "amax")
        self.energy = out["total_energy"].double().view(-1)
        self.done |= m < self.fmax ** 2

    def step(self):
        act = ~self.done
        ga, gc = self.ga, (self.gc if self.filt else None)
        vg, vv, gg = (self._fsum((self.v * ga).sum(1)), self._fsum((self.v * self.v).sum(1)), self._fsum((ga * ga).sum(1)))
        if self.filt:
            vg, vv, gg = vg + (self.vc * gc).sum((1, 2)), vv + (self.vc ** 2).sum((1, 2)), gg + (gc ** 2).sum((1, 2))
        if self.first:
            cv = torch.zeros(self.F, dtype=torch.float64, device=vg.device)
            cg = cv.clone()
            self.first = False
        else:
            mix = vg > 0
            cv = torch.where(mix, 1 - self.a, 0.0)
            cg = torch.where(mix, self.a * vv.sqrt() / gg.sqrt(), 0.0)
            grow = mix & (self.n > FIRE_DEFAULTS["Nmin"])
            dt = torch.where(grow, torch.clamp(self.dt * FIRE_DEFAULTS["finc"], max=FIRE_DEFAULTS["dtmax"]),
                             torch.where(mix, self.dt, self.dt * FIRE_DEFAULTS["fdec"]))
            a = torch.where(grow, self.a * FIRE_DEFAULTS["fa"], torch.where(mix, self.a, FIRE_DEFAULTS["astart"]))
            n = torch.where(mix, self.n + 1, 0)
            self.dt, self.a, self.n = torch.where(act, dt, self.dt), torch.where(act, a, self.a), torch.where(act, n, self.n)
        cg = cg + self.dt
        vnew = cv[self.frame].unsqueeze(1) * self.v + cg[self.frame].unsqueeze(1) * ga
        nr2 = self._fsum((vnew * vnew).sum(1))
        if self.filt:
            vcn = cv.view(-1, 1, 1) * self.vc + cg.view(-1, 1, 1) * gc
            nr2 = nr2 + (vcn ** 2).sum((1, 2))
        ndr = self.dt * nr2.sqrt()
        sc = torch.where(ndr > FIRE_DEFAULTS["maxstep"], self.dt * FIRE_DEFAULTS["maxstep"] / ndr, self.dt)
        sc = torch.where(act, sc, 0.0)
        keep = act[self.frame].unsqueeze(1)
        self.v = torch.where(keep, vnew, self.v)
        self.s = self.s + sc[self.frame].unsqueeze(1) * self.v
        if self.filt:
            self.vc = torch.where(act.view(-1, 1, 1), vcn, self.vc)
            self.Q = self.Q + sc.view(-1, 1, 1) * self.vc
        self.steps += act.long()
        self._eval()
        return bool(self.done.all())  # the per-step host read

    def run(self, n):
        for _ in range(n):
            if self.step():
                break


def recaptures(obj):
    return (obj.g if isinstance(obj, HostFire) else obj).recaptures


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--max-steps", type=int, default=1500)
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_relax.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    gpu = BM.gpu_info()
    lines = []

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for name in args.workloads.split(","):
        model, ex, filt = workload(name, dev)
        kw = {"cell_filter": "frechet"} if filt else {}
        atoms, frames = ex["pos"].shape[0], int(ex["num_atoms"].numel())

        def make(block, fmax):
            return HostFire(model, ex, filt, fmax) if block is None else GraphedRelax(model, ex, fmax=fmax, **kw)

        # time per FIRE step, no frame stopping
        for arm, block in ARMS:
            obj = make(block, 1e-9)
            go = (lambda n: obj.run(n)) if block is None else (lambda n: obj.run(n, block=block))
            go(args.warmup)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            go(args.steps)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            emit({"workload": name, "what": "fire_step", "arm": arm, "atoms": atoms, "frames": frames,
                  "steps": args.steps, "ms_per_step": ms, "block": block, "recaptures": recaptures(obj)})
            del obj
        # relax to FMAX
        energies = {}
        for arm, block in ARMS:
            obj = make(block, FMAX)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if block is None:
                obj.run(args.max_steps)
                steps, conv, e = obj.steps.cpu(), obj.done.cpu(), obj.energy.cpu()
            else:
                res = obj.run(args.max_steps, block=block)
                steps, conv = res["steps"], res["converged"]
                e = res["log"]["e_pot"][-1] if res["log"]["e_pot"].shape[0] else torch.full((frames,), float("nan"))
            e1.record()
            torch.cuda.synchronize()
            energies[arm] = e.double()
            emit({"workload": name, "what": "relax", "arm": arm, "atoms": atoms, "frames": frames, "fmax": FMAX,
                  "converged": int(conv.sum()), "steps_max": int(steps.max()), "steps_mean": float(steps.double().mean()),
                  "wall_ms": e0.elapsed_time(e1), "block": block, "recaptures": recaptures(obj)})
            del obj
        ref = energies["A_host_update"]
        emit({"workload": name, "what": "agreement", "atoms": atoms, "frames": frames,
              "max_energy_diff_B_vs_A": float((energies["B_block_1"] - ref).abs().max()),
              "max_energy_diff_C_vs_A": float((energies["C_block_50"] - ref).abs().max()),
              "max_energy_diff_B_vs_C": float((energies["B_block_1"] - energies["C_block_50"]).abs().max()),
              "max_abs_energy": float(ref.abs().max())})
        del model, ex
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
