"""Molecular dynamics on the device: velocity Verlet, optionally with the reference's Nose-Hoover thermostat
(nequip/ase/nosehoover.py), inside the captured MD step.

``GraphedMDStep`` captures positions -> neighbour list -> energy -> forces; a caller that integrates on the host reads
the edge count back after every step and can never queue step t+1 while step t runs.  ``GraphedMD`` captures the whole
step -- the first half of the update, the bath, the device neighbour list, the model, the second half of the update
and one row of a thermo log -- as one graph, and ``run(n_steps, block=K)`` replays it K times back to back and reads
from the host once per block (DESIGN.md section 4.14).

Units are the reference's (ASE's): Angstrom, eV, amu, so time is in Angstrom sqrt(amu / eV) and velocities in
Angstrom per that unit; the constants are ASE's CODATA-2014 ``units.kB`` and ``units.fs``.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch

from . import _capi, ops
from .graph import GraphedMDStep

#: Boltzmann constant in eV/K (CODATA 2014, ASE ``units.kB``)
KB = 8.617330337217213e-05
#: one femtosecond in Angstrom sqrt(amu / eV) (CODATA 2014, ASE ``units.fs``)
FS = 0.09822694788464065
#: the per-frame fields of a log row, in the order of ``nqb_md_log``
LOG_FIELDS = ("e_pot", "e_kin", "temperature", "zeta", "eta", "conserved")
#: log rows held on the device; a larger ``block`` re-captures the step with a longer log
DEFAULT_LOG_ROWS = 100
_THREADS, _MAX_CTAS = 256, 64  # CTA size of the nqb_md kernels (nqb.h) and the most CTAs per frame


def _per_frame(value, F: int, what: str) -> torch.Tensor:
    t = torch.as_tensor(value, dtype=torch.float64).cpu().reshape(-1)
    if t.numel() == 1:
        t = t.expand(F)
    if t.numel() != F:
        raise ValueError(f"GraphedMD: {what} must be a scalar or hold one value per frame ({F}), got {t.numel()}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"GraphedMD: {what} must be finite")
    return t.clone()


def zero_rotation_and_momentum(pos: torch.Tensor, vel: torch.Tensor, mass: torch.Tensor,
                               atom_ptr) -> torch.Tensor:
    """ASE's ``ZeroRotation`` then ``Stationary`` on every frame [atom_ptr[f], atom_ptr[f+1]) of float64 ``vel``: subtract
    omega x (r - r_com) with omega = I^-1 L about the centre of mass (a zero principal moment, as for one atom or a line
    of atoms, contributes no rotation), then the centre-of-mass velocity.  Temperatures are not rescaled."""
    vel = vel.clone()
    for f in range(len(atom_ptr) - 1):
        a, b = int(atom_ptr[f]), int(atom_ptr[f + 1])
        if b <= a:
            continue
        m, r, v = mass[a:b].unsqueeze(1), pos[a:b], vel[a:b]
        r = r - (m * r).sum(0) / m.sum()
        L = torch.cross(r, m * v, dim=1).sum(0)
        inertia = (m.squeeze(1) * (r * r).sum(1)).sum() * torch.eye(3, dtype=r.dtype) - (m * r).T @ r
        lam, basis = torch.linalg.eigh(inertia)
        inv = torch.where(lam > 1e-12 * lam.abs().max().clamp_min(1e-300), 1.0 / lam, torch.zeros_like(lam))
        omega = basis @ (inv * (basis.T @ L))
        v = v - torch.cross(omega.expand_as(r), r, dim=1)
        vel[a:b] = v - (m * v).sum(0) / m.sum()
    return vel


def maxwell_boltzmann(mass: torch.Tensor, temperature: torch.Tensor, seed: int = 0) -> torch.Tensor:
    """Float64 velocities [N, 3] drawn from the Maxwell-Boltzmann distribution at ``temperature`` [N] K (plain torch on
    the CPU, seeded): each component is normal with variance k_B T / m."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(mass.shape[0], 3, generator=g, dtype=torch.float64)
    return z * torch.sqrt(KB * temperature / mass).unsqueeze(1)


class BlockDriver(GraphedMDStep):
    """The block machinery that ``GraphedMD`` and ``relax.GraphedRelax`` share: a captured step that writes one row
    of a device log ring per replay (row ``step % rows``) and keeps sticky flags [4] i64 {overflow, unsorted, first
    overflowing step, largest edge count} (reset to {0, 0, -1, 0}), and ``_run_block(k)``, which replays the step k
    times from a device-side snapshot of the state, reads the block's log rows, the flags and ``_block_reads()`` with
    one host synchronisation, and rolls the block back and re-captures with ``capacity = ceil(1.02 * needed)`` when the
    neighbour list overflowed.  A subclass sets ``LOG_FIELDS`` and ``num_frames``, lists its device state in
    ``_state_list()``, calls ``_init_blocks`` before ``GraphedMDStep.__init__`` and writes the log from its captured
    step."""

    LOG_FIELDS: tuple = ()

    def _init_blocks(self, dev) -> None:
        self.host_reads = 0
        self._step = torch.zeros(1, dtype=torch.int64, device=dev)
        self._step_host = 0
        self._sticky0 = torch.tensor([0, 0, -1, 0], dtype=torch.int64, device=dev)
        self._sticky = self._sticky0.clone()
        self._sticky_host = torch.zeros(4, dtype=torch.int64).pin_memory()
        self._one = torch.ones(1, dtype=torch.int32, device=dev)
        self._alloc_log(DEFAULT_LOG_ROWS)

    def _state_list(self) -> list:
        raise NotImplementedError

    def _block_reads(self) -> list:
        """(device tensor, pinned host tensor) pairs copied with every block's host read."""
        return []

    def _alloc_log(self, rows: int) -> None:
        shape = (rows, self.num_frames, len(self.LOG_FIELDS))
        self._log = torch.zeros(shape, dtype=torch.float64, device=self._step.device)
        self._log_host = torch.zeros(shape, dtype=torch.float64).pin_memory()

    def _sorted_flag(self) -> torch.Tensor:
        """The captured step's "edges grouped by destination" flag (the capture's deferred flags)."""
        flags = getattr(ops._sorted_tls, "flags", None)
        return torch.stack([f.view(()) for f in flags]).min().view(1) if flags else self._one

    def _capture(self, model, example: Dict[str, torch.Tensor], capacity: int) -> None:
        # the warm-up before the capture executes the step: keep the state as it was
        saved = [t.clone() for t in self._state_list()]
        super()._capture(model, example, capacity)
        for t, s in zip(self._state_list(), saved):
            t.copy_(s)
        self._sticky.copy_(self._sticky0)

    def _read_block(self, k: int) -> torch.Tensor:
        """The block's k log rows, the sticky flags and ``_block_reads()``, with one host synchronisation."""
        R = self._log.shape[0]
        a = self._step_host % R
        n1 = min(k, R - a)
        self._log_host[:n1].copy_(self._log[a:a + n1], non_blocking=True)
        if n1 < k:
            self._log_host[n1:k].copy_(self._log[:k - n1], non_blocking=True)
        self._sticky_host.copy_(self._sticky, non_blocking=True)
        for dev_t, host_t in self._block_reads():
            host_t.copy_(dev_t, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        self.host_reads += 1
        return self._log_host[:k].clone()

    def _fit_log(self, block: int) -> None:
        """A log of at least ``block`` rows; the captured step holds the log's pointer and length, so a longer log
        is a re-capture (not counted in ``recaptures``)."""
        if block > self._log.shape[0]:
            self._alloc_log(block)
            n = self.recaptures
            self._recapture(self.capacity)
            self.recaptures = n

    def _check_block(self) -> None:
        """Raise for a block that must not be kept (after the overflow test)."""
        if int(self._sticky_host[1]) != 0:
            raise RuntimeError(f"{type(self).__name__}: a step's edge list was not grouped by destination; its "
                               "forces are invalid")

    def _run_block(self, k: int) -> torch.Tensor:
        """Replay the step k times; returns the block's log rows [k, F, len(LOG_FIELDS)]."""
        for s, t in zip(self._snap, self._state_list()):
            s.copy_(t)
        self._sticky.copy_(self._sticky0)
        while True:
            for _ in range(k):
                self.graph.replay()
            self.replays += k
            got = self._read_block(k)
            if int(self._sticky_host[0]) == 0:
                break
            for s, t in zip(self._snap, self._state_list()):
                t.copy_(s)
            self._sticky.copy_(self._sticky0)
            self._recapture(max(self.capacity + 1, math.ceil(1.02 * int(self._sticky_host[3]))))
        self._check_block()
        self._step_host += k
        return got


class GraphedMD(BlockDriver):
    """A device-resident MD driver: ``md = GraphedMD(model, example, masses, timestep_fs); log = md.run(n_steps)``.

    ``example`` holds what ``GraphedMDStep`` takes: ``pos`` [N, 3], ``atom_types`` [N], ``cell`` or none, ``pbc``, and
    ``batch`` / ``num_atoms`` for a batch of F frames, which are integrated side by side, each with its own bath.
    ``masses`` (amu) is per atom [N] or per type [T] (T = the model's type count; [N] wins when N == T).
    ``thermostat=None`` integrates NVE (velocity Verlet); ``"nose_hoover"`` the reference's ``NoseHoover.step`` with
    target ``temperature`` (K) and ``nvt_q`` (the reference's Q in its units, e.g. 334), each a scalar or [F].
    ``velocities`` [N, 3] (Angstrom per Angstrom sqrt(amu / eV), ASE's unit); when None they are drawn from the
    Maxwell-Boltzmann distribution at ``temperature`` (``seed``), or are zero without a temperature.  As the reference
    does, the initial velocities lose their rotation and then their centre-of-mass momentum, frame by frame.  The forces
    F(0) at the initial positions come from one eager neighbour list and model call.  ``variable_cell=True`` raises:
    this driver has no barostat (constant-pressure MD is ``npt.GraphedNPT``).  Invalid arguments raise ``ValueError`` before any CUDA work.

    ``run(n_steps, block=50, on_block=None)`` advances the state by ``n_steps`` and returns the log, a dict of host
    float64 tensors [n_steps, F] named by ``LOG_FIELDS``: the potential energy (the model's ``total_energy``), the
    kinetic energy, the kinetic temperature 2 E_kin / (3 N_f k_B), the bath variable zeta, its integral eta and the
    conserved quantity H = E_pot + E_kin + Q zeta^2 + g k_B T eta (g = 3 N_f + 1; H = E_pot + E_kin for NVE).  Row s
    describes the state after step s + 1 of the call.  ``on_block(log_block)`` sees each block's rows as it completes.

    Each block starts with a device-side copy of the state; the K replays then run without the host, and one read
    (``host_reads`` counts them) fetches the block's log rows and sticky flags.  A block in which the neighbour list
    overflowed its ``capacity`` is discarded: the state is restored, the step re-captured with
    ``capacity = ceil(1.02 * needed)`` (``recaptures`` counts them) and the block run again, so discarded steps never
    reach the log.  A block whose edges were not grouped by destination raises ``RuntimeError``.

    ``state`` holds the device buffers ``pos`` [N, 3], ``vel`` [N, 3], ``forces`` [N, 3] (all float64), ``zeta``
    and ``eta`` [F] and ``step`` [1] (int64); ``pos`` is the buffer the captured neighbour list reads."""

    LOG_FIELDS = LOG_FIELDS

    def __init__(self, model, example: Dict[str, torch.Tensor], masses, timestep_fs: float,
                 thermostat: Optional[str] = None, temperature=None, nvt_q=None, velocities=None,
                 capacity: Optional[int] = None, *, variable_cell: bool = False, seed: int = 0, warmup: int = 3):
        if variable_cell:
            raise ValueError("GraphedMD: variable_cell is not supported (there is no barostat)")
        if thermostat not in (None, "nose_hoover"):
            raise ValueError(f"GraphedMD: thermostat must be None or 'nose_hoover', got {thermostat!r}")
        if thermostat is not None and (temperature is None or nvt_q is None):
            raise ValueError("GraphedMD: the Nose-Hoover thermostat needs a temperature and nvt_q")
        if not (math.isfinite(float(timestep_fs)) and float(timestep_fs) > 0):
            raise ValueError(f"GraphedMD: timestep_fs must be finite and positive, got {timestep_fs}")
        pos = example["pos"]
        N = int(pos.shape[0])
        if example.get("batch") is not None:
            counts = torch.as_tensor(example["num_atoms"]).cpu().reshape(-1).long()
        else:
            counts = torch.tensor([N])
        F = int(counts.numel())
        if int(counts.sum()) != N:
            raise ValueError(f"GraphedMD: num_atoms sums to {int(counts.sum())}, pos has {N} atoms")
        types = example["atom_types"].reshape(-1).cpu().long()
        m = torch.as_tensor(masses, dtype=torch.float64).cpu().reshape(-1)
        T_types = len(model.config["type_names"])
        if m.numel() == N:
            mass = m.clone()
        elif m.numel() == T_types:
            mass = m[types]
        else:
            raise ValueError(f"GraphedMD: masses must hold one value per atom ({N}) or per type ({T_types}), "
                             f"got {m.numel()}")
        if not bool((torch.isfinite(mass) & (mass > 0)).all()):
            raise ValueError("GraphedMD: masses must be finite and positive")
        temp = None if temperature is None else _per_frame(temperature, F, "temperature")
        if temp is not None and bool((temp < 0).any()):
            raise ValueError("GraphedMD: temperature must not be negative")
        q = None if nvt_q is None else _per_frame(nvt_q, F, "nvt_q")
        if q is not None and bool((q <= 0).any()):
            raise ValueError("GraphedMD: nvt_q must be positive")
        if velocities is not None and tuple(velocities.shape) != (N, 3):
            raise ValueError(f"GraphedMD: velocities must be [{N}, 3], got {tuple(velocities.shape)}")

        atom_ptr = torch.zeros(F + 1, dtype=torch.int64)
        atom_ptr[1:] = torch.cumsum(counts, 0)
        pos_host = pos.detach().cpu().double()
        if velocities is not None:
            vel = velocities.detach().cpu().double()
        elif temp is not None:
            vel = maxwell_boltzmann(mass, torch.repeat_interleave(temp, counts), seed)
        else:
            vel = torch.zeros(N, 3, dtype=torch.float64)
        vel = zero_rotation_and_momentum(pos_host, vel, mass, atom_ptr.tolist())
        if pos.device.type != "cuda":
            raise RuntimeError("GraphedMD needs CUDA tensors (there is no CPU path)")

        dev = pos.device
        self.thermostat = thermostat
        self.dt = float(timestep_fs) * FS
        self.num_frames = F
        self._init_blocks(dev)
        self._nblk = max(1, min(_MAX_CTAS, -(-int(counts.max()) // _THREADS)))
        self._atom_ptr = atom_ptr.to(dev)
        self._mass = mass.to(dev)
        if thermostat is None:
            gkT, Q = torch.zeros(F, dtype=torch.float64), torch.zeros(F, dtype=torch.float64)
        else:
            gkT, Q = (3 * counts + 1).double() * KB * temp, q
        self._gkT, self._Q = gkT.to(dev), Q.to(dev)
        self._dof_kB = (3 * counts.double() * KB).clamp_min(1e-300).to(dev)
        self._pos = pos.detach().double().clone().to(dev)
        self._vel = vel.to(dev)
        self._forces = torch.zeros(N, 3, dtype=torch.float64, device=dev)
        self._zeta = torch.zeros(F, dtype=torch.float64, device=dev)
        self._eta = torch.zeros(F, dtype=torch.float64, device=dev)
        self._part = torch.zeros(F, self._nblk, 2, dtype=torch.float64, device=dev)
        self._ke_part = torch.zeros(F, self._nblk, dtype=torch.float64, device=dev)
        self._snap = [t.clone() for t in self._state_list()]
        self._forces.copy_(self._eager_forces(model, example))
        super().__init__(model, dict(example, pos=self._pos), capacity=capacity, warmup=warmup)

    # ---- state --------------------------------------------------------------------------------------------------
    def _state_list(self):
        return [self._pos, self._vel, self._forces, self._zeta, self._eta, self._step]

    @property
    def state(self) -> Dict[str, torch.Tensor]:
        return {"pos": self._pos, "vel": self._vel, "forces": self._forces, "zeta": self._zeta, "eta": self._eta,
                "step": self._step}

    def _eager_forces(self, model, example) -> torch.Tensor:
        """F(0): one eager neighbour list and model call at the initial positions (any edge count)."""
        dev = self._pos.device
        cell = example.get("cell")
        batch = {} if example.get("batch") is None else {"batch": example["batch"].to(dev).view(-1)}
        pbc = self._periodicity(example)
        if batch and isinstance(pbc[0], tuple):
            pbc = torch.tensor(pbc)
        nl = ops.neighbor_list(self._pos, cell, pbc, model.r_max, **self._edge_type_args(model, example), **batch)
        d = {"pos": self._pos, "atom_types": example["atom_types"].to(dev), "edge_index": nl["edge_index"],
             "edge_cell_shift": nl["edge_cell_shift"]}
        if cell is not None:
            d["cell"] = cell
        if batch:
            d.update(batch, num_atoms=torch.as_tensor(example["num_atoms"]).to(dev).view(-1))
        return model(d)["forces"].detach().double()

    # ---- the captured step --------------------------------------------------------------------------------------
    def _run(self):
        L, st = _capi.lib(), ops._stream()
        P = ops._ptr
        F, nb, dt = self.num_frames, self._nblk, self.dt
        # the neighbour list and the model read the state's position buffer itself, which the integrator moves
        self.static["pos"] = self._pos
        _capi.check(L.nqb_md_kick_drift(F, nb, P(self._atom_ptr), P(self._mass), P(self._forces), P(self._zeta), dt,
                                        P(self._pos), P(self._vel), P(self._part), st), "nqb_md_kick_drift")
        if self.thermostat is not None:
            _capi.check(L.nqb_md_bath(F, nb, P(self._part), P(self._gkT), P(self._Q), dt, P(self._zeta), P(self._eta),
                                      st), "nqb_md_bath")
        out = super()._run()
        f_new = out["forces"].detach().double().contiguous()
        _capi.check(L.nqb_md_kick(F, nb, P(self._atom_ptr), P(self._mass), P(f_new), P(self._zeta), dt, P(self._vel),
                                  P(self._forces), P(self._ke_part), st), "nqb_md_kick")
        sorted_flag = self._sorted_flag()
        e_pot = out["total_energy"].detach().double().reshape(-1).contiguous()
        _capi.check(L.nqb_md_log(F, nb, P(e_pot), P(self._ke_part), P(self._zeta), P(self._eta), P(self._Q),
                                 P(self._gkT), P(self._dof_kB), P(self._out["num_edges"]), P(self._out["overflow"]),
                                 P(sorted_flag), self._log.shape[0], P(self._step), P(self._log), P(self._sticky), st),
                    "nqb_md_log")
        return out

    def run(self, n_steps: int, block: int = 50,
            on_block: Optional[Callable[[Dict[str, torch.Tensor]], None]] = None) -> Dict[str, torch.Tensor]:
        if n_steps < 0 or block < 1:
            raise ValueError(f"GraphedMD.run: needs n_steps >= 0 and block >= 1, got {n_steps}, {block}")
        self._fit_log(block)
        rows = []
        done = 0
        while done < n_steps:
            k = min(block, n_steps - done)
            got = self._run_block(k)
            done += k
            rows.append(got)
            if on_block is not None:
                on_block({name: got[:, :, j] for j, name in enumerate(LOG_FIELDS)})
        log = torch.cat(rows) if rows else torch.zeros(0, self.num_frames, len(LOG_FIELDS), dtype=torch.float64)
        return {name: log[:, :, j].clone() for j, name in enumerate(LOG_FIELDS)}
