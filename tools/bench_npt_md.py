"""Constant-pressure MD: ``GraphedMDStep(variable_cell=True)`` plus the same isotropic MTK update in eager torch on the
device and ``g(pos, cell)`` (a host ``set_cell``) every step (arm A, what a user writes today) against ``GraphedNPT``
with blocks of 1 and 50 steps (arms B, C).  With ``--flexible`` the arms are C and F:
``GraphedNPT(barostat="flexible")`` with blocks of 50 steps, the fully flexible cell (DESIGN.md section 4.17),
alternated within each round.

Workloads:
  * water_1k_l2_f32   the 1 000-atom water box, l_max 2, 4 layers, 32 features (tools/bench_md.py);
  * S_li3po4_10k      preset S on the 10 648-atom Li3PO4 frame (tools/bench_md.py);
  * water_125_x128    128 water boxes of 125 atoms strained by up to +-2 %, one batch, the water_1k model
                      (tools/bench_batched_md.py).

Every arm runs at 300 K and 1 bar with tau_T = 100 fs, tau_P = 1 000 fs, chains of 3 and dt = 0.5 fs.  Per workload:
ms per step of each arm in ``--rounds`` rounds, the arms alternated within a round, each timed window of ``--steps``
steps after ``--warmup`` steps; arm A against arm C over 50 steps from one state (positions, E_pot, H); and with
``--long N`` an N-step run of arm C on water_1k_l2_f32 reporting <T>, <P>, <V> with errors from 10 block averages and
the drift of H.  The card's name, power limit and SM clock are read in the same process.

    python tools/bench_npt_md.py [--workloads ...] [--steps 100] [--warmup 20] [--rounds 3] [--long 40000]
                                 [--flexible] [--out FILE.jsonl]
"""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_batched_md as BB  # noqa: E402
import bench_md as BM  # noqa: E402
from nequip_b200.graph import GraphedMDStep  # noqa: E402
from nequip_b200.md import FS, KB  # noqa: E402
from nequip_b200.npt import GPA, GraphedNPT  # noqa: E402

WORKLOADS = ("water_1k_l2_f32", "S_li3po4_10k", "water_125_x128")
ARMS = (("A_host_update", None), ("B_block_1", 1), ("C_block_50", 50))
FLEX_ARMS = (("C_block_50", 50), ("F_flexible_block_50", 50))
MASS = {"H": 1.008, "O": 15.999, "Li": 6.94, "P": 30.974}
BAR = 1e-4 * GPA
BATH = dict(temperature=300.0, pressure=BAR, tdamp_fs=100.0, pdamp_fs=1000.0)
DT_FS, CHAIN = 0.5, 3


def workload(name, dev):
    """(model, batched example, per-type masses)."""
    if name == "water_125_x128":
        fr, meta = BB.frames("water", 128, 5, dev)
        model = BB.model_for(None, meta, dev)
        counts = [f[0].shape[0] for f in fr]
        ex = {"pos": torch.cat([f[0] for f in fr]).double(), "atom_types": torch.cat([f[2] for f in fr]),
              "cell": torch.stack([f[1] for f in fr]).double(),
              "batch": torch.repeat_interleave(torch.arange(128, device=dev), torch.tensor(counts, device=dev)),
              "num_atoms": torch.tensor(counts, device=dev)}
    else:
        model, d, _ = BM.build(name)
        N = d["pos"].shape[0]
        ex = {"pos": d["pos"].double(), "atom_types": d["atom_types"].view(-1),
              "cell": d["cell"].double().view(1, 3, 3), "batch": torch.zeros(N, dtype=torch.int64, device=dev),
              "num_atoms": torch.tensor([N], device=dev)}
    return model, ex, [MASS[t] for t in model.config["type_names"]]


class HostNPT:
    """Arm A: the forces and virial of ``GraphedMDStep(variable_cell=True)``, the MTK step of GraphedNPT (the same
    splitting, chains and masses) in eager torch over all frames at once, and ``g(pos, cell)`` every step, which packs
    the cells on the host and reads the edge count back."""

    def __init__(self, model, ex, masses, vel):
        self.g = GraphedMDStep(model, ex, variable_cell=True)
        dev = ex["pos"].device
        self.frame = ex["batch"].long()
        counts = ex["num_atoms"].double()
        F = counts.numel()
        self.F, self.dt = F, DT_FS * FS
        self.mass = torch.tensor(masses, dtype=torch.float64, device=dev)[ex["atom_types"].long()]
        self.kT = torch.full((F,), KB * BATH["temperature"], dtype=torch.float64, device=dev)
        self.P = BATH["pressure"]
        self.Nf = 3 * counts
        tt, tp = BATH["tdamp_fs"] * FS, BATH["pdamp_fs"] * FS
        self.W = (self.Nf + 3) * self.kT * tp ** 2
        self.Q = [(self.Nf if k == 0 else 1.0) * self.kT * tt ** 2 for k in range(CHAIN)]
        self.Qp = [self.kT * tp ** 2 for _ in range(CHAIN)]
        self.C0 = ex["cell"].double().clone()
        self.V0 = torch.linalg.det(self.C0).abs()
        z = lambda: torch.zeros(F, dtype=torch.float64, device=dev)  # noqa: E731
        self.eps, self.veps = z(), z()
        self.xi, self.vxi = [z() for _ in range(CHAIN)], [z() for _ in range(CHAIN)]
        self.eta, self.veta = [z() for _ in range(CHAIN)], [z() for _ in range(CHAIN)]
        self.pos, self.vel = ex["pos"].double().clone(), vel.clone()
        self.K2 = self._fsum(self.mass * (self.vel ** 2).sum(1))
        out = self.g(self.pos, self.C0)
        self.forces, self.vir = out["forces"].double().clone(), out["virial"].double().clone()
        self.e_pot = out["total_energy"].double().view(-1).clone()

    def _fsum(self, x):
        return torch.zeros(self.F, dtype=torch.float64, device=x.device).index_add_(0, self.frame, x)

    def _nhc(self, h, Nf, Q, x, v, K2):
        M = len(Q)
        d2, d4 = 0.5 * h, 0.25 * h

        def G(k):
            return (K2 - Nf * self.kT) / Q[0] if k == 0 else (Q[k - 1] * v[k - 1] ** 2 - self.kT) / Q[k]

        v[M - 1] = v[M - 1] + d2 * G(M - 1)
        for k in range(M - 2, -1, -1):
            e = torch.exp(-d4 * v[k + 1])
            v[k] = (v[k] * e + d2 * G(k)) * e
        sc = torch.exp(-h * v[0])
        K2 = K2 * sc * sc
        for k in range(M):
            x[k] = x[k] + h * v[k]
        for k in range(M - 1):
            e = torch.exp(-d4 * v[k + 1])
            v[k] = (v[k] * e + d2 * G(k)) * e
        v[M - 1] = v[M - 1] + d2 * G(M - 1)
        return sc, K2

    def _baro_kick(self, K2, vir):
        alpha = 1 + 3 / self.Nf
        V = self.V0 * torch.exp(3 * self.eps)
        self.veps = self.veps + 0.5 * self.dt * (alpha * K2 + vir.diagonal(dim1=1, dim2=2).sum(1) - 3 * self.P * V) / self.W

    def _coefs(self):
        def sinhc(x):  # the Taylor branch of nqb_npt.cu and tests/npt_oracle.py (NQB_NPT_SINHC_TAYLOR)
            x2 = x * x
            return torch.where(x.abs() < 0.1, 1 + x2 * (1 / 6 + x2 * (1 / 120 + x2 * (1 / 5040 + x2 / 362880))),
                               torch.sinh(x) / x)

        a, b = (1 + 3 / self.Nf) * self.veps * self.dt, self.veps * self.dt
        return (torch.exp(-0.5 * a)[self.frame, None], (0.5 * self.dt * torch.exp(-0.25 * a) * sinhc(0.25 * a))[self.frame, None],
                torch.exp(b)[self.frame, None], (self.dt * torch.exp(0.5 * b) * sinhc(0.5 * b))[self.frame, None])

    def step(self):
        h = 0.5 * self.dt
        sb, _ = self._nhc(h, 1.0, self.Qp, self.eta, self.veta, self.W * self.veps ** 2)
        self.veps = self.veps * sb
        s, self.K2 = self._nhc(h, self.Nf, self.Q, self.xi, self.vxi, self.K2)
        self._baro_kick(self.K2, self.vir)
        ev, kf, er, df = self._coefs()
        m = self.mass.unsqueeze(1)
        self.vel = (s[self.frame, None] * self.vel) * ev + kf * (self.forces / m)
        self.pos = self.pos * er + df * self.vel
        self.eps = self.eps + self.dt * self.veps
        out = self.g(self.pos, self.C0 * torch.exp(self.eps).view(-1, 1, 1))  # host set_cell and edge-count read
        self.forces, self.vir = out["forces"].double().clone(), out["virial"].double().clone()
        self.e_pot = out["total_energy"].double().view(-1).clone()
        self.vel = self.vel * ev + kf * (self.forces / m)
        K2 = self._fsum(self.mass * (self.vel ** 2).sum(1))
        self._baro_kick(K2, self.vir)
        s, self.K2 = self._nhc(h, self.Nf, self.Q, self.xi, self.vxi, K2)
        self.vel = s[self.frame, None] * self.vel
        sb, _ = self._nhc(h, 1.0, self.Qp, self.eta, self.veta, self.W * self.veps ** 2)
        self.veps = self.veps * sb

    def conserved(self):
        V = self.V0 * torch.exp(3 * self.eps)
        H = self.e_pot + 0.5 * self.K2 + 0.5 * self.W * self.veps ** 2 + self.P * V
        for k in range(CHAIN):
            H = H + 0.5 * self.Q[k] * self.vxi[k] ** 2 + (self.Nf if k == 0 else 1.0) * self.kT * self.xi[k]
            H = H + 0.5 * self.Qp[k] * self.veta[k] ** 2 + self.kT * self.eta[k]
        return H

    def run(self, n, block=None):
        for _ in range(n):
            self.step()

    @property
    def recaptures(self):
        return self.g.recaptures


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--long", type=int, default=0, help="steps of the long water_1k run (0: none)")
    ap.add_argument("--flexible", action="store_true",
                    help="time the flexible barostat against C_block_50 (and skip the A-vs-C agreement)")
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_npt_md.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    gpu = BM.gpu_info()

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(rec) + "\n")

    for name in args.workloads.split(","):
        model, ex, masses = workload(name, dev)
        atoms, frames = ex["pos"].shape[0], int(ex["num_atoms"].numel())

        def make(block, barostat="isotropic"):
            npt = GraphedNPT(model, ex, masses, DT_FS, tchain=CHAIN, pchain=CHAIN, seed=1, barostat=barostat, **BATH)
            if block is None:
                vel = npt.state["vel"].clone()
                del npt
                return HostNPT(model, ex, masses, vel)
            return npt

        arms = FLEX_ARMS if args.flexible else ARMS
        objs = {arm: make(block, "flexible" if arm.startswith("F_") else "isotropic") for arm, block in arms}
        for rnd in range(args.rounds):
            for arm, block in arms:
                obj = objs[arm]
                obj.run(args.warmup, block=block or 1)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                obj.run(args.steps, block=block or 1)
                e1.record()
                torch.cuda.synchronize()
                emit({"workload": name, "what": "npt_step", "arm": arm, "round": rnd, "atoms": atoms,
                      "frames": frames, "steps": args.steps, "ms_per_step": e0.elapsed_time(e1) / args.steps,
                      "block": block, "recaptures": obj.recaptures,
                      "barostat": getattr(obj, "barostat", "isotropic")})
        if args.flexible:
            cell = objs["F_flexible_block_50"].state["cell"]
            off = cell - torch.diag_embed(cell.diagonal(dim1=1, dim2=2))
            emit({"workload": name, "what": "flexible_cell", "atoms": atoms, "frames": frames,
                  "steps": objs["F_flexible_block_50"].replays, "max_abs_offdiag_cell": float(off.abs().max())})
        del objs
        if args.flexible:
            del model, ex
            torch.cuda.empty_cache()
            continue
        # A against C over 50 steps from one state
        a, c = make(None), make(50)
        a.run(50)
        logc = c.run(50, block=50)
        torch.cuda.synchronize()
        h_a = a.conserved()
        emit({"workload": name, "what": "agreement_A_vs_C", "atoms": atoms, "frames": frames, "steps": 50,
              "max_pos_diff": float((a.pos - c.state["pos"]).abs().max()),
              "max_epot_diff": float((a.e_pot - logc["e_pot"][-1].to(dev)).abs().max()),
              "max_H_diff": float((h_a - logc["conserved"][-1].to(dev)).abs().max()),
              "max_abs_epot": float(a.e_pot.abs().max()),
              "max_eps_diff": float((a.eps - c.state["eps"]).abs().max())})
        del a, c, model, ex
        torch.cuda.empty_cache()

    if args.long:
        model, ex, masses = workload("water_1k_l2_f32", dev)
        npt = GraphedNPT(model, ex, masses, DT_FS, tchain=CHAIN, pchain=CHAIN, seed=1, **BATH)
        t0 = time.time()
        log = npt.run(args.long, block=50)
        wall = time.time() - t0
        nb = 10
        rec = {"workload": "water_1k_l2_f32", "what": "long_run", "steps": args.long, "dt_fs": DT_FS,
               "ps": args.long * DT_FS / 1000, "wall_s": wall, "recaptures": npt.recaptures, **BATH}
        half = args.long // 2  # the first half is equilibration
        for k, unit in (("temperature", 1.0), ("pressure", 1.0 / GPA), ("volume", 1.0)):
            x = log[k][half:, 0].double() * unit
            blocks = x[: (x.numel() // nb) * nb].view(nb, -1).mean(1)
            rec[f"mean_{k}"] = float(x.mean())
            rec[f"err_{k}"] = float(blocks.std() / math.sqrt(nb))
        rec["pressure_unit"] = "GPa"
        H = log["conserved"][:, 0]
        rec["H_drift_eV"] = float(H[-1] - H[0])
        rec["H_max_dev_eV"] = float((H - H[0]).abs().max())
        rec["H_drift_meV_per_atom_per_ps"] = 1e3 * float(H[-1] - H[0]) / ex["pos"].shape[0] / rec["ps"]
        emit(rec)


if __name__ == "__main__":
    main()
