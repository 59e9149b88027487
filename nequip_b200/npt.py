"""Constant-pressure (NPT) molecular dynamics on the device: isotropic or fully flexible MTK with Nose-Hoover chains
inside one captured step.

The equations are Martyna, Tobias & Klein, J. Chem. Phys. 101, 4177 (1994) for an isotropic cell, integrated with the
measure-preserving splitting of Tuckerman, Alejandre, Lopez-Rendon, Jochim & Martyna, J. Phys. A 39, 5629 (2006); the
particles and the barostat each carry a Nose-Hoover chain (Martyna, Tuckerman, Tobias & Klein, Mol. Phys. 87, 1117
(1996)).  This is the scheme of ASE's ``IsotropicMTKNPT``.  ``GraphedNPT`` captures the whole step -- the first half
of the update, the drift of positions and cell, the cell packed into the device neighbour list
(``NeighborListPlan.set_cell_device``), the list, the model with stress, the second half of the update and one row of
a log -- as one CUDA graph for a batch of frames, and ``run(n_steps, block=K)`` replays it K times per host read
(DESIGN.md section 4.16).  ``barostat="flexible"`` lets the cell's shape move too: the fully flexible MTK equations
(Martyna, Tobias & Klein 1994; Martyna, Tuckerman, Tobias & Klein 1996) with a symmetric 3x3 cell velocity, in the
same splitting (DESIGN.md section 4.17).  Units are those of ``md``: Angstrom, eV, amu, ASE's CODATA-2014 ``KB``
and ``FS``.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import torch

from . import _capi, ops
from .md import _MAX_CTAS, _THREADS, FS, KB, BlockDriver, maxwell_boltzmann

#: one gigapascal in eV / Angstrom^3 (CODATA 2014, ASE ``units.GPa``)
GPA = 1.0 / 160.21766208
#: the per-frame fields of a log row, in the order of ``nqb_npt_log``
LOG_FIELDS = ("e_pot", "e_kin", "temperature", "volume", "pressure", "conserved")
#: the longest Nose-Hoover chain (NQB_NPT_MAX_CHAIN)
MAX_CHAIN = 8
_NS, _NP, _NC = 35, 22, 7  # NQB_NPT_STATE, NQB_NPT_PARAMS, NQB_NPT_COEF
_XI, _VXI, _ETA, _VETA = 3, 3 + MAX_CHAIN, 3 + 2 * MAX_CHAIN, 3 + 3 * MAX_CHAIN  # offsets in a state row
#: the barostats ``GraphedNPT`` runs
BAROSTATS = ("isotropic", "flexible")
# the flexible cell: NQB_NPTF_STATE, NQB_NPTF_COEF, NQB_NPTF_LOG_FIELDS and the offsets in its state row
_NFS, _NFC, _NFL = 50, 39, 24
_FKT, _FXI, _FVXI, _FETA, _FVETA = 9, 18, 18 + MAX_CHAIN, 18 + 2 * MAX_CHAIN, 18 + 3 * MAX_CHAIN
#: the barostat chain's degrees of freedom under the flexible barostat: the components of a symmetric v_g
FLEX_DOF = 6


def _per_frame(value, F: int, what: str) -> torch.Tensor:
    t = torch.as_tensor(value, dtype=torch.float64).cpu().reshape(-1)
    if t.numel() == 1:
        t = t.expand(F)
    if t.numel() != F:
        raise ValueError(f"GraphedNPT: {what} must be a scalar or hold one value per frame ({F}), got {t.numel()}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"GraphedNPT: {what} must be finite")
    return t.clone()


def _positive(value, F: int, what: str) -> torch.Tensor:
    t = _per_frame(value, F, what)
    if bool((t <= 0).any()):
        raise ValueError(f"GraphedNPT: {what} must be positive")
    return t


class GraphedNPT(BlockDriver):
    """Isotropic NPT on the device: ``npt = GraphedNPT(model, example, masses, timestep_fs, temperature, pressure,
    tdamp_fs=100, pdamp_fs=1000); log = npt.run(n_steps)``.

    ``example`` holds what ``GraphedMDStep`` takes: ``pos`` [N, 3], ``atom_types`` [N], ``cell``, and ``batch`` /
    ``num_atoms`` for a batch of F frames, which are integrated side by side, each with its own barostat and chains (a
    single frame is a batch of one).  Every frame must be periodic in all three directions and hold at least one atom.
    ``masses`` (amu) is per atom [N] or per type [T] as in ``md.GraphedMD``.  ``temperature`` (K), ``pressure``
    (eV / Angstrom^3; ``GPA`` converts), ``tdamp_fs`` and ``pdamp_fs`` (the thermostat's and barostat's time scales
    tau_T and tau_P) are each a scalar or [F].  The chain masses follow Martyna et al. (1996):
    Q_1 = N_f k_B T tau_T^2, Q_k = k_B T tau_T^2 (k >= 2), W = (N_f + 3) k_B T tau_P^2 and Q'_k = k_B T tau_P^2, with
    N_f = 3 N.  ``tchain`` and ``pchain`` (0 .. ``MAX_CHAIN``) are the chain lengths (0 removes that chain; both 0 is
    NPH), ``tloop`` and ``ploop`` (>= 1) their sub-steps per half step.  Only the cell's scale moves: the cell is
    C0 e^eps (C0 the initial cell), so its shape is kept exactly.

    ``velocities`` [N, 3] (ASE's unit); when None they are drawn from the Maxwell-Boltzmann distribution at each
    frame's temperature (``seed``).  Each frame's centre-of-mass momentum is removed; its rotation is not, since
    every frame is periodic.  The barostat velocity and the chains start at 0.  F(0) and the virial come from one eager
    neighbour list and model call with stress.  Invalid arguments raise ``ValueError`` before any CUDA work.

    ``run(n_steps, block=50, on_block=None)`` advances the state by ``n_steps`` and returns a dict of host float64
    tensors [n_steps, F] named by ``LOG_FIELDS``: the model's energy, the kinetic energy, the kinetic temperature,
    the volume, the instantaneous pressure (sum m v^2 + tr virial) / (3 V) and the conserved quantity
    H = E_pot + E_kin + W v_eps^2 / 2 + P V + sum Q_k v_xi_k^2 / 2 + N_f k_B T xi_1 + k_B T sum_{k>=2} xi_k
    + sum Q'_k v_eta_k^2 / 2 + k_B T sum eta_k.  Row s describes the state after step s + 1 of the call.  Blocks,
    ``host_reads``, rollback and re-capture on an overflowing neighbour list are ``md.BlockDriver``'s.  A block in
    which a frame's update became non-finite (the frame is then frozen: its positions and cell never take a
    non-finite value) or its cell was rejected by the neighbour list is discarded: the state is restored and
    ``RuntimeError`` names the frames.

    ``state`` holds the device buffers ``pos``, ``vel``, ``forces`` [N, 3], ``virial`` and ``cell`` [F, 3, 3], ``eps``,
    ``v_eps`` and ``K2`` (sum m v^2) [F], the chains ``xi``, ``v_xi`` [F, tchain] and ``eta``, ``v_eta`` [F, pchain],
    ``error`` [F] int32 and ``step`` [1] (views of the buffers the captured step reads and writes).

    ``barostat="flexible"`` runs the fully flexible MTK barostat instead (DESIGN.md section 4.17): a symmetric cell
    velocity v_g [3, 3] (so the cell does not rotate) driven by sym(Kt + virial) - P V I + (tr Kt / N_f) I, with
    Kt = sum m v (x) v, V = |det cell| and the cell's rows moving as da/dt = v_g a.  Its mass is
    W_g = (N_f + 3) k_B T tau_P^2 / 3 and its chain couples to W_g tr(v_g^2) with 6 degrees of freedom
    (Q'_1 = 6 k_B T tau_P^2, Q'_k = k_B T tau_P^2).  Every other argument, the blocks, rollback and freezing are as
    above.  ``state`` then holds ``pos``, ``vel``, ``forces``, ``virial``, ``cell``, ``v_g`` and ``kinetic`` (Kt)
    [F, 3, 3], the chains, ``error`` and ``step`` (no ``eps``: the cell itself is the state), and ``run`` also returns
    ``cell`` and ``pressure_tensor`` (Kt + virial) / V [n_steps, F, 3, 3]; ``volume`` is |det cell| and ``pressure``
    tr(pressure_tensor) / 3, and ``conserved`` carries W_g tr(v_g^2) / 2 and 6 k_B T eta_1.  A liquid has no shear
    resistance, so its cell drifts in shape under this barostat: use ``"isotropic"`` for liquids."""

    LOG_FIELDS = LOG_FIELDS

    def __init__(self, model, example: Dict[str, torch.Tensor], masses, timestep_fs: float, temperature, pressure, *,
                 tdamp_fs, pdamp_fs, tchain: int = 3, pchain: int = 3, tloop: int = 1, ploop: int = 1,
                 velocities=None, capacity: Optional[int] = None, seed: int = 0, warmup: int = 3,
                 barostat: str = "isotropic"):
        if barostat not in BAROSTATS:
            raise ValueError(f"GraphedNPT: barostat must be one of {BAROSTATS}, got {barostat!r}")
        self.barostat = barostat
        flex = barostat == "flexible"
        if not (math.isfinite(float(timestep_fs)) and float(timestep_fs) > 0):
            raise ValueError(f"GraphedNPT: timestep_fs must be finite and positive, got {timestep_fs}")
        for name, v, lo, hi in (("tchain", tchain, 0, MAX_CHAIN), ("pchain", pchain, 0, MAX_CHAIN),
                                ("tloop", tloop, 1, None), ("ploop", ploop, 1, None)):
            if int(v) != v or v < lo or (hi is not None and v > hi):
                raise ValueError(f"GraphedNPT: {name} must be an integer in [{lo}, {hi if hi is not None else 'inf'}]"
                                 f", got {v}")
        pos = example["pos"]
        N = int(pos.shape[0])
        if example.get("batch") is not None:
            counts = torch.as_tensor(example["num_atoms"]).cpu().reshape(-1).long()
            batch = torch.as_tensor(example["batch"]).reshape(-1)
        else:
            counts = torch.tensor([N])
            batch = torch.zeros(N, dtype=torch.int64)
        F = int(counts.numel())
        if int(counts.sum()) != N:
            raise ValueError(f"GraphedNPT: num_atoms sums to {int(counts.sum())}, pos has {N} atoms")
        if bool((counts < 1).any()):
            raise ValueError("GraphedNPT: every frame needs at least one atom (NPT of an empty box is undefined)")
        cell = example.get("cell")
        if cell is None:
            raise ValueError("GraphedNPT: every frame must be periodic in all three directions (no cell given)")
        cell = torch.as_tensor(cell)
        if cell.numel() != 9 * F:
            raise ValueError(f"GraphedNPT: cell must be [3, 3] or [{F}, 3, 3], got {tuple(cell.shape)}")
        pbc = example.get("pbc")
        pbc = torch.as_tensor(True if pbc is None else pbc).cpu()
        _, pbc_np, cells0 = ops._nl_frame_args(cell.reshape(F, 3, 3), pbc, batch.cpu(), N)
        if not pbc_np.all():
            raise ValueError("GraphedNPT: every frame must be periodic in all three directions")
        for f in range(F):
            ops._nl_check_cell(cells0[f], "GraphedNPT")
        types = example["atom_types"].reshape(-1).cpu().long()
        m = torch.as_tensor(masses, dtype=torch.float64).cpu().reshape(-1)
        T_types = len(model.config["type_names"]) if model is not None else -1
        if m.numel() == N:
            mass = m.clone()
        elif m.numel() == T_types:
            mass = m[types]
        else:
            raise ValueError(f"GraphedNPT: masses must hold one value per atom ({N}) or per type ({T_types}), "
                             f"got {m.numel()}")
        if not bool((torch.isfinite(mass) & (mass > 0)).all()):
            raise ValueError("GraphedNPT: masses must be finite and positive")
        temp = _positive(temperature, F, "temperature")
        pres = _per_frame(pressure, F, "pressure")
        tau_t = _positive(tdamp_fs, F, "tdamp_fs") * FS
        tau_p = _positive(pdamp_fs, F, "pdamp_fs") * FS
        if velocities is not None and tuple(velocities.shape) != (N, 3):
            raise ValueError(f"GraphedNPT: velocities must be [{N}, 3], got {tuple(velocities.shape)}")
        if pos.device.type != "cuda":
            raise RuntimeError("GraphedNPT needs CUDA tensors (there is no CPU path)")

        atom_ptr = torch.zeros(F + 1, dtype=torch.int64)
        atom_ptr[1:] = torch.cumsum(counts, 0)
        if velocities is not None:
            vel = velocities.detach().cpu().double().clone()
        else:
            vel = maxwell_boltzmann(mass, torch.repeat_interleave(temp, counts), seed)
        for f in range(F):
            a, b = int(atom_ptr[f]), int(atom_ptr[f + 1])
            mf = mass[a:b].unsqueeze(1)
            vel[a:b] -= (mf * vel[a:b]).sum(0) / mf.sum()
        # K2 = sum m v^2 per frame, correctly rounded (math.fsum), so the starting state depends only on the inputs
        k2 = [math.fsum((mass[int(atom_ptr[f]):int(atom_ptr[f + 1])] * (vel[int(atom_ptr[f]):int(atom_ptr[f + 1])] ** 2)
                         .sum(1)).tolist()) for f in range(F)]
        if flex:  # Kt = sum m v (x) v per frame and component, correctly rounded too
            kt = torch.zeros(F, 3, 3, dtype=torch.float64)
            for f in range(F):
                a, b = int(atom_ptr[f]), int(atom_ptr[f + 1])
                for i in range(3):
                    for j in range(i, 3):
                        kt[f, i, j] = kt[f, j, i] = math.fsum((mass[a:b] * vel[a:b, i] * vel[a:b, j]).tolist())

        dev = pos.device
        self.dt = float(timestep_fs) * FS
        self.num_frames = F
        self.chains = (int(tchain), int(pchain), int(tloop), int(ploop))
        self._init_blocks(dev)
        self._nblk = max(1, min(_MAX_CTAS, -(-int(counts.max()) // _THREADS)))
        self._atom_ptr = atom_ptr.to(dev)
        self._mass = mass.to(dev)
        # per-frame constants (nqb.h layout): kT, P, W, N_f, V0, N_f k_B, Q[8], Q'[8] (unused members 1)
        kT = KB * temp
        Nf = 3.0 * counts.double()
        prm = torch.ones(F, _NP, dtype=torch.float64)
        prm[:, 0], prm[:, 1], prm[:, 3], prm[:, 5] = kT, pres, Nf, Nf * KB
        prm[:, 2] = (Nf + 3.0) * kT * tau_p ** 2
        if flex:
            prm[:, 2] /= 3.0  # W_g
        prm[:, 4] = torch.from_numpy(cells0).double().det().abs()
        for k in range(int(tchain)):
            prm[:, 6 + k] = (Nf if k == 0 else 1.0) * kT * tau_t ** 2
        for k in range(int(pchain)):
            prm[:, 6 + MAX_CHAIN + k] = (FLEX_DOF if flex and k == 0 else 1.0) * kT * tau_p ** 2
        self._prm = prm.to(dev)
        f64 = dict(dtype=torch.float64, device=dev)
        self._pos = pos.detach().double().clone().to(dev)
        self._vel = vel.to(dev)
        self._forces = torch.zeros(N, 3, **f64)
        self._vir = torch.zeros(F, 3, 3, **f64)
        self._cell = torch.from_numpy(cells0.copy()).to(dev)
        self._err = torch.zeros(F, dtype=torch.int32, device=dev)
        if flex:
            self._st = torch.zeros(F, _NFS, **f64)
            self._st[:, _FKT:_FKT + 9] = kt.reshape(F, 9)
            self._coef = torch.zeros(F, _NFC, **f64)
            self._work = torch.zeros(F, _NFS, **f64)
            self._part = torch.zeros(F, self._nblk, 6, **f64)
        else:
            self._C0 = self._cell.clone()
            self._st = torch.zeros(F, _NS, **f64)
            self._st[:, 2] = torch.tensor(k2, dtype=torch.float64)
            self._coef = torch.zeros(F, _NC, **f64)
            self._work = torch.zeros(F, _NS, **f64)
            self._part = torch.zeros(F, self._nblk, **f64)
        self._err_host = torch.zeros(F, dtype=torch.int32).pin_memory()
        self._cerr_host = torch.zeros(F, dtype=torch.int32).pin_memory()
        self._snap = [t.clone() for t in self._state_list()]

        ex = {"pos": self._pos, "atom_types": example["atom_types"].to(dev).reshape(-1),
              "batch": batch.to(dev).long(), "num_atoms": counts.to(dev), "pbc": torch.as_tensor(pbc_np),
              "cell": self._cell}
        self._initial(model, ex)
        super().__init__(model, ex, capacity=capacity, warmup=warmup, variable_cell=True)
        self.plan.cell_error.zero_()

    # ---- state --------------------------------------------------------------------------------------------------
    def _state_list(self):
        return [self._pos, self._vel, self._forces, self._vir, self._cell, self._st, self._err, self._step]

    def _alloc_log(self, rows: int) -> None:
        if self.barostat != "flexible":
            return super()._alloc_log(rows)
        shape = (rows, self.num_frames, _NFL)  # LOG_FIELDS, the cell [9] and the pressure tensor [9]
        self._log = torch.zeros(shape, dtype=torch.float64, device=self._step.device)
        self._log_host = torch.zeros(shape, dtype=torch.float64).pin_memory()

    @property
    def state(self) -> Dict[str, torch.Tensor]:
        M, Mp = self.chains[:2]
        if self.barostat == "flexible":
            F = self.num_frames
            return {"pos": self._pos, "vel": self._vel, "forces": self._forces, "virial": self._vir,
                    "cell": self._cell, "v_g": self._st[:, 0:9].view(F, 3, 3),
                    "kinetic": self._st[:, _FKT:_FKT + 9].view(F, 3, 3),
                    "xi": self._st[:, _FXI:_FXI + M], "v_xi": self._st[:, _FVXI:_FVXI + M],
                    "eta": self._st[:, _FETA:_FETA + Mp], "v_eta": self._st[:, _FVETA:_FVETA + Mp],
                    "error": self._err, "step": self._step}
        return {"pos": self._pos, "vel": self._vel, "forces": self._forces, "virial": self._vir, "cell": self._cell,
                "eps": self._st[:, 0], "v_eps": self._st[:, 1], "K2": self._st[:, 2],
                "xi": self._st[:, _XI:_XI + M], "v_xi": self._st[:, _VXI:_VXI + M],
                "eta": self._st[:, _ETA:_ETA + Mp], "v_eta": self._st[:, _VETA:_VETA + Mp],
                "error": self._err, "step": self._step}

    def _block_reads(self) -> list:
        reads = [(self._err, self._err_host)]
        if self.plan is not None:
            reads.append((self.plan.cell_error, self._cerr_host))
        return reads

    def _initial(self, model, ex) -> None:
        """F(0) and the virial at the initial state: one eager list and model call with stress."""
        nl = ops.neighbor_list(self._pos, ex["cell"], ex["pbc"], model.r_max, **self._edge_type_args(model, ex),
                               batch=ex["batch"])
        d = {"pos": self._pos, "atom_types": ex["atom_types"], "edge_index": nl["edge_index"],
             "edge_cell_shift": nl["edge_cell_shift"], "batch": ex["batch"], "num_atoms": ex["num_atoms"],
             "cell": ex["cell"]}
        out = model(d, compute_stress=True)
        self._forces.copy_(out["forces"].detach().double())
        self._vir.copy_(out["virial"].detach().double().reshape(-1, 3, 3))
        if not (bool(torch.isfinite(self._forces).all()) and bool(torch.isfinite(self._vir).all())):
            raise RuntimeError("GraphedNPT: the model's forces or virial at the initial state are not finite")

    # ---- the captured step --------------------------------------------------------------------------------------
    def _capture(self, model, example: Dict[str, torch.Tensor], capacity: int) -> None:
        super()._capture(model, example, capacity)
        self.plan.cell_error.zero_()  # the warm-up moved the cell from the state it was restored to

    def _run(self):
        L, st, P = _capi.lib(), ops._stream(), ops._ptr
        F, nb, dt = self.num_frames, self._nblk, self.dt
        M, Mp, tl, pl = self.chains
        # the list and the model read the state's position and cell buffers themselves, which the integrator moves
        self.static["pos"] = self._pos
        self.static["cell"] = self._cell
        if self.barostat == "flexible":
            return self._run_flexible()
        _capi.check(L.nqb_npt_pre(F, M, Mp, tl, pl, dt, P(self._prm), P(self._C0), P(self._vir), P(self._st),
                                  P(self._cell), P(self._coef), P(self._err), P(self._work), st), "nqb_npt_pre")
        _capi.check(L.nqb_npt_move(F, nb, P(self._atom_ptr), P(self._mass), P(self._forces), P(self._coef),
                                   P(self._pos), P(self._vel), st), "nqb_npt_move")
        self.plan.set_cell_device(self._cell)
        out = super()._run()
        f_new = out["forces"].detach().double().contiguous()
        _capi.check(L.nqb_npt_kick(F, nb, P(self._atom_ptr), P(self._mass), P(f_new), P(self._coef), P(self._vel),
                                   P(self._forces), P(self._part), st), "nqb_npt_kick")
        vir_new = out["virial"].detach().double().contiguous()
        _capi.check(L.nqb_npt_post(F, nb, M, Mp, tl, pl, dt, P(self._prm), P(self._part), P(vir_new), P(self._st),
                                   P(self._vir), P(self._coef), P(self._err), P(self._work), st), "nqb_npt_post")
        _capi.check(L.nqb_npt_scale(F, nb, P(self._atom_ptr), P(self._coef), P(self._vel), st), "nqb_npt_scale")
        e_pot = out["total_energy"].detach().double().reshape(-1).contiguous()
        _capi.check(L.nqb_npt_log(F, M, Mp, P(e_pot), P(self._prm), P(self._st), P(self._vir),
                                  P(self._out["num_edges"]), P(self._out["overflow"]), P(self._sorted_flag()),
                                  self._log.shape[0], P(self._step), P(self._log), P(self._sticky), st), "nqb_npt_log")
        return out

    def _run_flexible(self):
        L, st, P = _capi.lib(), ops._stream(), ops._ptr
        F, nb, dt = self.num_frames, self._nblk, self.dt
        M, Mp, tl, pl = self.chains
        _capi.check(L.nqb_nptf_pre(F, M, Mp, tl, pl, dt, P(self._prm), P(self._vir), P(self._st), P(self._cell),
                                   P(self._coef), P(self._err), P(self._work), st), "nqb_nptf_pre")
        _capi.check(L.nqb_nptf_move(F, nb, P(self._atom_ptr), P(self._mass), P(self._forces), P(self._coef),
                                    P(self._pos), P(self._vel), st), "nqb_nptf_move")
        self.plan.set_cell_device(self._cell)
        out = super()._run()
        f_new = out["forces"].detach().double().contiguous()
        _capi.check(L.nqb_nptf_kick(F, nb, P(self._atom_ptr), P(self._mass), P(f_new), P(self._coef), P(self._vel),
                                    P(self._forces), P(self._part), st), "nqb_nptf_kick")
        vir_new = out["virial"].detach().double().contiguous()
        _capi.check(L.nqb_nptf_post(F, nb, M, Mp, tl, pl, dt, P(self._prm), P(self._part), P(vir_new), P(self._cell),
                                    P(self._st), P(self._vir), P(self._coef), P(self._err), P(self._work), st),
                    "nqb_nptf_post")
        _capi.check(L.nqb_nptf_scale(F, nb, P(self._atom_ptr), P(self._coef), P(self._vel), st), "nqb_nptf_scale")
        e_pot = out["total_energy"].detach().double().reshape(-1).contiguous()
        _capi.check(L.nqb_nptf_log(F, M, Mp, P(e_pot), P(self._prm), P(self._st), P(self._vir), P(self._cell),
                                   P(self._out["num_edges"]), P(self._out["overflow"]), P(self._sorted_flag()),
                                   self._log.shape[0], P(self._step), P(self._log), P(self._sticky), st),
                    "nqb_nptf_log")
        return out

    def _fields(self, rows: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Log rows [k, F, width] as the dict ``run`` returns."""
        out = {name: rows[:, :, j] for j, name in enumerate(LOG_FIELDS)}
        if self.barostat == "flexible":
            k, F = rows.shape[:2]
            out["cell"] = rows[:, :, 6:15].reshape(k, F, 3, 3)
            out["pressure_tensor"] = rows[:, :, 15:24].reshape(k, F, 3, 3)
        return out

    def _check_block(self) -> None:
        super()._check_block()
        bad = torch.nonzero((self._err_host != 0) | (self._cerr_host != 0)).flatten().tolist()
        if bad:
            for s, t in zip(self._snap, self._state_list()):
                t.copy_(s)
            self.plan.cell_error.zero_()
            raise RuntimeError(f"GraphedNPT: the update of frame(s) {bad} became non-finite or their cell was "
                               "rejected; the block was discarded and the state restored")

    def run(self, n_steps: int, block: int = 50,
            on_block: Optional[Callable[[Dict[str, torch.Tensor]], None]] = None) -> Dict[str, torch.Tensor]:
        if n_steps < 0 or block < 1:
            raise ValueError(f"GraphedNPT.run: needs n_steps >= 0 and block >= 1, got {n_steps}, {block}")
        self._fit_log(block)
        rows = []
        done = 0
        while done < n_steps:
            k = min(block, n_steps - done)
            got = self._run_block(k)
            done += k
            rows.append(got)
            if on_block is not None:
                on_block(self._fields(got))
        log = torch.cat(rows) if rows else torch.zeros(0, self.num_frames, self._log.shape[2], dtype=torch.float64)
        return {name: v.clone() for name, v in self._fields(log).items()}
