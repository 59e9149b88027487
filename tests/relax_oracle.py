"""Float64 restatement of the device relaxation (nequip_b200/relax.py, csrc/nqb_relax.cu) on the host: ASE's
FIRE.step per frame and ASE's FrechetCellFilter as DESIGN.md section 4.15 defines it, with scipy's ``expm``.

One frame's DOF are the atom rows (s, with r = s Fd^T) and, with the filter, 3 cell rows (Q = c log Fd, cell =
C0 Fd^T).  The generalised forces are g_i = f_i Fd and G_uv = (1/c) sum_ab (W Fd^-T)_ab [D exp(Q/c)[E_uv]]_ab with
W = virial - p V I; D exp(L)[E] is the upper-right block of exp([[L, E], [0, L]])."""
from __future__ import annotations

import numpy as np
from scipy.linalg import expm

FIRE_DEFAULTS = dict(dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)


def dexp(L: np.ndarray, E: np.ndarray) -> np.ndarray:
    """The Frechet derivative of the matrix exponential at L in the direction E: a block of a 6x6 exponential."""
    Z = np.zeros((6, 6))
    Z[:3, :3] = Z[3:, 3:] = L
    Z[:3, 3:] = E
    return expm(Z)[:3, 3:]


def generalized_forces(forces, virial, Q, c: float, cell, p: float):
    """(g [N, 3], G [3, 3]): the forces on s and on Q of one frame at deformation Q (cell = the current cell)."""
    Fd = expm(Q / c)
    V = abs(np.linalg.det(cell))
    W = virial - p * V * np.eye(3)
    M = W @ np.linalg.inv(Fd).T
    G = np.zeros((3, 3))
    for u in range(3):
        for v in range(3):
            E = np.zeros((3, 3))
            E[u, v] = 1.0
            G[u, v] = np.sum(M * dexp(Q / c, E)) / c
    return forces @ Fd, G


class Frame:
    """One frame's relaxation: ``positions()`` / ``cell()`` to evaluate, then ``evaluate(e, forces, virial)`` (the
    generalised forces and the convergence test), then ``step()`` (one FIRE update unless frozen)."""

    def __init__(self, pos, cell, cell_filter: bool, fmax=0.05, p=0.0, c=None, fail_force=1e6, **fire):
        self.fp = dict(FIRE_DEFAULTS, **fire)
        self.s = np.array(pos, dtype=np.float64)
        self.C0 = np.array(cell, dtype=np.float64) if cell is not None else np.eye(3)
        self.filt = cell_filter
        self.Q = np.zeros((3, 3))
        self.c = float(max(len(self.s), 1) if c is None else c)
        self.p, self.fmax, self.fail_force = p, fmax, fail_force
        self.dt, self.a, self.Nsteps, self.v = self.fp["dt"], self.fp["a"], 0, None
        self.converged = self.failed = False
        self.steps = 0
        self.g = None
        self.log = None

    def Fd(self):
        return expm(self.Q / self.c) if self.filt else np.eye(3)

    def positions(self):
        return self.s @ self.Fd().T

    def cell(self):
        return self.C0 @ self.Fd().T

    def evaluate(self, e: float, forces, virial=None) -> None:
        forces = np.asarray(forces, dtype=np.float64)
        if self.filt:
            g, G = generalized_forces(forces, np.asarray(virial, dtype=np.float64), self.Q, self.c, self.cell(),
                                      self.p)
            g = np.concatenate([g, G])
        else:
            g = forces.copy()
        self.g = g
        m = float((g ** 2).sum(axis=1).max()) if len(g) else 0.0
        V = abs(np.linalg.det(self.cell()))
        self.log = (e, e + self.p * V, np.sqrt(m), V)
        if not (self.converged or self.failed):
            if not m <= self.fail_force ** 2:
                self.failed = True
            elif m < self.fmax ** 2:
                self.converged = True

    def step(self) -> None:
        if self.converged or self.failed:
            return
        fp, f = self.fp, self.g
        if self.v is None:
            self.v = np.zeros_like(f)
        else:
            vf = np.vdot(f, self.v)
            if vf > 0.0:
                self.v = (1.0 - self.a) * self.v + self.a * f / np.sqrt(np.vdot(f, f)) * np.sqrt(np.vdot(self.v, self.v))
                if self.Nsteps > fp["Nmin"]:
                    self.dt = min(self.dt * fp["finc"], fp["dtmax"])
                    self.a *= fp["fa"]
                self.Nsteps += 1
            else:
                self.v[:] *= 0.0
                self.a = fp["astart"]
                self.dt *= fp["fdec"]
                self.Nsteps = 0
        self.v += self.dt * f
        dr = self.dt * self.v
        normdr = np.sqrt(np.vdot(dr, dr))
        if normdr > fp["maxstep"]:
            dr = fp["maxstep"] * dr / normdr
        n = len(self.s)
        self.s = self.s + dr[:n]
        if self.filt:
            self.Q = self.Q + dr[n:]
        self.steps += 1
