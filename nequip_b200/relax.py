"""Structure relaxation on the device: ASE's FIRE, optionally with ASE's Frechet cell filter, inside one captured step.

The reference's recipe (docs/integrations/ase.md) relaxes a list of structures one at a time, each wrapped in
``FrechetCellFilter`` and driven by an ASE optimiser, with one host round trip per force call.  ``GraphedRelax``
captures the whole step -- the FIRE update of positions and cell, the cell packed into the device neighbour list
(``NeighborListPlan.set_cell_device``), the list, the model with stress, the generalised forces, the convergence test
and one row of a log -- as one CUDA graph for a batch of frames, and ``run(max_steps, block=K)`` replays it K times
per host read (DESIGN.md section 4.15).  Units are the model's: Angstrom, eV; FIRE's time step is in ASE's units
(unit masses).
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import torch

from . import _capi, ops
from .md import _MAX_CTAS, _THREADS, BlockDriver

#: the per-frame fields of a log row, in the order of ``nqb_relax_finish``
LOG_FIELDS = ("e_pot", "enthalpy", "fmax", "volume")
#: ASE's FIRE defaults (ase.optimize.FIRE)
FIRE_DEFAULTS = dict(dt=0.1, maxstep=0.2, dtmax=1.0, Nmin=5, finc=1.1, fdec=0.5, astart=0.1, fa=0.99, a=0.1)
_ISTATE = 5  # NQB_RELAX_ISTATE: {Nsteps, first, converged, failed, steps}


def _positive(name: str, v) -> float:
    v = float(v)
    if not (math.isfinite(v) and v > 0):
        raise ValueError(f"GraphedRelax: {name} must be finite and positive, got {v}")
    return v


class GraphedRelax(BlockDriver):
    """Relax a batch of structures on the device: ``r = GraphedRelax(model, example); res = r.run(max_steps)``.

    ``example`` holds what ``GraphedMDStep`` takes: ``pos`` [N, 3], ``atom_types`` [N], ``cell`` or none, ``pbc``, and
    ``batch`` / ``num_atoms`` for a batch of F frames (one frame is a batch of one).  Each frame is an independent FIRE
    optimisation (ASE's ``FIRE.step``, unit masses) with its own ``dt``, ``a`` and step counter, run until the largest
    row norm of its generalised forces is below ``fmax`` (eV/Angstrom).  The FIRE parameters are keyword arguments with
    ASE's defaults (``FIRE_DEFAULTS``).

    ``cell_filter=None`` moves the positions only (any frame: periodic, slab, molecule).  ``cell_filter="frechet"``
    (every frame periodic in all three directions) adds ASE's ``FrechetCellFilter``: the atoms' DOF are s with
    r = s Fd^T, the cell's are Q = c log Fd with cell = C0 Fd^T (C0 the initial cell, c = ``exp_cell_factor``, by
    default N_f), and the forces on them are the exact negative derivatives of the enthalpy E + pV with
    p = ``scalar_pressure`` (eV/Angstrom^3).  A frame is ``failed`` when a force is non-finite or its largest row norm
    exceeds ``fail_force``.  Converged and failed frames are frozen: their positions and cell no longer change,
    though their energy is still evaluated.  ``capacity`` is the edge capacity as in ``GraphedMDStep``.  Invalid
    arguments raise ``ValueError`` before any CUDA work.

    The forces, virial and convergence test at the initial structure come from one eager call, so a frame that starts
    converged takes zero steps.  ``run(max_steps, block=50)`` replays blocks of ``block`` steps with one host read
    each (``host_reads``) and stops after the first block in which every frame is converged or failed, or at
    ``max_steps``.  A block whose neighbour list overflowed is rolled back and re-captured with a larger capacity, as
    in ``GraphedMD``; a block in which a frame's cell became non-finite or singular is discarded and raises
    ``RuntimeError`` naming the frame.  It returns host tensors: ``converged``, ``failed`` [F] bool, ``steps`` [F] (the
    FIRE updates each frame took), ``pos`` [N, 3], ``cell`` [F, 3, 3] and ``log``, a dict of [n, F] float64 named by
    ``LOG_FIELDS`` (row s describes the structure after step s + 1 of the call): the model's energy, the enthalpy
    E + pV, the largest row norm of the generalised forces and the cell volume |det cell| (the cell of an open frame is
    the identity)."""

    LOG_FIELDS = LOG_FIELDS

    def __init__(self, model, example: Dict[str, torch.Tensor], fmax: float = 0.05, cell_filter: Optional[str] = None,
                 scalar_pressure: float = 0.0, exp_cell_factor=None, fail_force: float = 1e6,
                 capacity: Optional[int] = None, *, warmup: int = 3, **fire_params):
        unknown = set(fire_params) - set(FIRE_DEFAULTS)
        if unknown:
            raise ValueError(f"GraphedRelax: unknown FIRE parameters {sorted(unknown)}")
        fp = dict(FIRE_DEFAULTS, **fire_params)
        for k in ("dt", "maxstep", "dtmax", "finc", "fdec"):
            _positive(k, fp[k])
        for k in ("astart", "fa", "a"):
            if not (math.isfinite(float(fp[k])) and 0.0 <= float(fp[k]) <= 1.0):
                raise ValueError(f"GraphedRelax: {k} must be in [0, 1], got {fp[k]}")
        if int(fp["Nmin"]) != fp["Nmin"] or int(fp["Nmin"]) < 0:
            raise ValueError(f"GraphedRelax: Nmin must be a non-negative integer, got {fp['Nmin']}")
        self.fmax = _positive("fmax", fmax)
        self.fail_force = _positive("fail_force", fail_force)
        if cell_filter not in (None, "frechet"):
            raise ValueError(f"GraphedRelax: cell_filter must be None or 'frechet', got {cell_filter!r}")
        self.cell_filter = cell_filter
        self.pressure = float(scalar_pressure)
        if not math.isfinite(self.pressure):
            raise ValueError("GraphedRelax: scalar_pressure must be finite")
        if cell_filter is None and (self.pressure != 0.0 or exp_cell_factor is not None):
            raise ValueError("GraphedRelax: scalar_pressure and exp_cell_factor need cell_filter='frechet'")
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
            raise ValueError(f"GraphedRelax: num_atoms sums to {int(counts.sum())}, pos has {N} atoms")
        cell = example.get("cell")
        if cell is not None:
            cell = torch.as_tensor(cell)
            if cell.numel() != 9 * F:
                raise ValueError(f"GraphedRelax: cell must be [3, 3] or [{F}, 3, 3], got {tuple(cell.shape)}")
            cell = cell.reshape(F, 3, 3)
        pbc = example.get("pbc")
        pbc = torch.as_tensor(cell is not None if pbc is None else pbc).cpu()
        _, pbc_np, cells0 = ops._nl_frame_args(cell, pbc, batch.cpu(), N)
        if cell_filter is not None and not pbc_np.all():
            raise ValueError("GraphedRelax: cell_filter needs every frame periodic in all three directions")
        for f in range(F):
            ops._nl_check_cell(cells0[f], "GraphedRelax")
        if exp_cell_factor is None:
            cfac = counts.double().clamp_min(1.0)
        else:
            cfac = torch.as_tensor(exp_cell_factor, dtype=torch.float64).reshape(-1).expand(F).clone()
            if not bool((torch.isfinite(cfac) & (cfac > 0)).all()):
                raise ValueError("GraphedRelax: exp_cell_factor must be finite and positive")
        if pos.device.type != "cuda":
            raise RuntimeError("GraphedRelax needs CUDA tensors (there is no CPU path)")

        dev = pos.device
        self.num_frames = F
        self._init_blocks(dev)
        self._fire_host = (ctypes.c_double * 7)(*[float(fp[k]) for k in
                                                  ("maxstep", "dtmax", "finc", "fdec", "astart", "fa", "Nmin")])
        self._has_cell = cell_filter is not None
        self._nblk = max(1, min(_MAX_CTAS, -(-int(counts.max()) // _THREADS)))
        atom_ptr = torch.zeros(F + 1, dtype=torch.int64)
        atom_ptr[1:] = torch.cumsum(counts, 0)
        self._atom_ptr = atom_ptr.to(dev)
        f64 = dict(dtype=torch.float64, device=dev)
        self._pos = pos.detach().double().clone().to(dev)
        self._s = self._pos.clone() if self._has_cell else torch.zeros(0, 3, **f64)
        self._vel = torch.zeros(N, 3, **f64)
        self._g = torch.zeros(N, 3, **f64)
        self._part = torch.zeros(F, self._nblk, 4, **f64)
        self._cell = torch.from_numpy(cells0.copy()).to(dev)
        self._C0 = self._cell.clone()
        self._Q = torch.zeros(F, 3, 3, **f64)
        self._vcell = torch.zeros(F, 3, 3, **f64)
        self._gcell = torch.zeros(F, 3, 3, **f64)
        self._Fd = torch.eye(3, **f64).expand(F, 3, 3).contiguous()
        self._cfac = cfac.to(dev)
        self._fs = torch.tensor([[float(fp["dt"]), float(fp["a"])]] * F, **f64).reshape(F, 2)
        self._is = torch.zeros(F, _ISTATE, dtype=torch.int64, device=dev)
        self._is[:, 1] = 1  # first step
        self._coef = torch.zeros(F, 4, **f64)
        self._is_host = torch.zeros(F, _ISTATE, dtype=torch.int64).pin_memory()
        self._cerr_host = torch.zeros(F, dtype=torch.int32).pin_memory()
        self._snap = [t.clone() for t in self._state_list()]

        ex = {"pos": self._pos, "atom_types": example["atom_types"].to(dev).reshape(-1),
              "batch": batch.to(dev).long(), "num_atoms": counts.to(dev),
              "pbc": torch.as_tensor(pbc_np)}
        if cell is not None:
            ex["cell"] = self._cell
        self._initial(model, ex)
        super().__init__(model, ex, capacity=capacity, warmup=warmup, variable_cell=self._has_cell)
        if self._has_cell:
            self.plan.cell_error.zero_()

    # ---- state --------------------------------------------------------------------------------------------------
    def _state_list(self):
        return [self._pos, self._s, self._vel, self._g, self._part, self._Q, self._vcell, self._gcell, self._Fd,
                self._cell, self._fs, self._is, self._step]

    @property
    def state(self) -> Dict[str, torch.Tensor]:
        return {"pos": self._pos, "cell": self._cell, "vel": self._vel, "g": self._g, "Q": self._Q,
                "vcell": self._vcell, "gcell": self._gcell, "Fd": self._Fd, "fire": self._fs, "istate": self._is,
                "step": self._step}

    def _block_reads(self) -> list:
        reads = [(self._is, self._is_host)]
        if self._has_cell and self.plan is not None:
            reads.append((self.plan.cell_error, self._cerr_host))
        return reads

    # ---- the generalised forces, convergence test and log row ---------------------------------------------------
    def _finish(self, out, num_edges, overflow, sorted_flag) -> None:
        L, st, P = _capi.lib(), ops._stream(), ops._ptr
        F, nb, hc = self.num_frames, self._nblk, int(self._has_cell)
        f_new = out["forces"].detach().double().contiguous()
        _capi.check(L.nqb_relax_gforce(F, nb, P(self._atom_ptr), hc, P(self._Fd), P(f_new), P(self._vel), P(self._g),
                                       P(self._part), st), "nqb_relax_gforce")
        e_pot = out["total_energy"].detach().double().reshape(-1).contiguous()
        virial = out["virial"].detach().double().contiguous() if self._has_cell else None
        _capi.check(L.nqb_relax_finish(F, nb, P(self._part), hc, self.pressure, P(self._cfac), P(self._Q), P(self._Fd),
                                       P(self._cell), P(virial), P(e_pot), self.fmax, self.fail_force, P(self._gcell),
                                       P(self._is), P(num_edges), P(overflow), P(sorted_flag), self._log.shape[0],
                                       P(self._step), P(self._log), P(self._sticky), st), "nqb_relax_finish")

    def _initial(self, model, ex) -> None:
        """Forces, virial and convergence flags at the initial structure: one eager list and model call."""
        dev = self._pos.device
        nl = ops.neighbor_list(self._pos, ex.get("cell"), ex["pbc"], model.r_max,
                               **self._edge_type_args(model, ex), batch=ex["batch"])
        d = {"pos": self._pos, "atom_types": ex["atom_types"], "edge_index": nl["edge_index"],
             "edge_cell_shift": nl["edge_cell_shift"], "batch": ex["batch"], "num_atoms": ex["num_atoms"]}
        if ex.get("cell") is not None:
            d["cell"] = ex["cell"]
        out = model(d, compute_stress=True) if self._has_cell else model(d)
        zero64, zero32 = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev)
        self._finish(out, zero64, zero32, self._one)
        self._step.zero_()
        self._sticky.copy_(self._sticky0)
        self._is_host.copy_(self._is)

    # ---- the captured step --------------------------------------------------------------------------------------
    def _capture(self, model, example: Dict[str, torch.Tensor], capacity: int) -> None:
        super()._capture(model, example, capacity)
        if self._has_cell:
            self.plan.cell_error.zero_()  # the warm-up moved the cell from the state it was restored to

    def _run(self):
        L, st, P = _capi.lib(), ops._stream(), ops._ptr
        F, nb, hc = self.num_frames, self._nblk, int(self._has_cell)
        # the list and the model read the state's position (and cell) buffers themselves, which FIRE moves
        self.static["pos"] = self._pos
        if self._has_cell:
            self.static["cell"] = self._cell
        _capi.check(L.nqb_relax_fire(F, nb, P(self._part), self._fire_host, hc, P(self._cfac), P(self._C0),
                                     P(self._gcell), P(self._Q), P(self._vcell), P(self._Fd), P(self._cell),
                                     P(self._fs), P(self._is), P(self._coef), st), "nqb_relax_fire")
        _capi.check(L.nqb_relax_move(F, nb, P(self._atom_ptr), P(self._coef), hc, P(self._Fd), P(self._g),
                                     P(self._vel), P(self._s), P(self._pos), st), "nqb_relax_move")
        if self._has_cell:
            self.plan.set_cell_device(self._cell)
        out = super()._run()
        self._finish(out, self._out["num_edges"], self._out["overflow"], self._sorted_flag())
        return out

    def _check_block(self) -> None:
        super()._check_block()
        if self._has_cell and bool((self._cerr_host != 0).any()):
            bad = torch.nonzero(self._cerr_host).flatten().tolist()
            for s, t in zip(self._snap, self._state_list()):
                t.copy_(s)
            self.plan.cell_error.zero_()
            raise RuntimeError(f"GraphedRelax: the cell of frame(s) {bad} became non-finite or singular; the block "
                               "was discarded")

    def _all_done(self) -> bool:
        return bool(((self._is_host[:, 2] != 0) | (self._is_host[:, 3] != 0)).all())

    def run(self, max_steps: int, block: int = 50) -> Dict[str, object]:
        if max_steps < 0 or block < 1:
            raise ValueError(f"GraphedRelax.run: needs max_steps >= 0 and block >= 1, got {max_steps}, {block}")
        self._fit_log(block)
        rows = []
        done = 0
        while done < max_steps and not self._all_done():
            k = min(block, max_steps - done)
            rows.append(self._run_block(k))
            done += k
        log = (torch.cat(rows) if rows
               else torch.zeros(0, self.num_frames, len(LOG_FIELDS), dtype=torch.float64))
        torch.cuda.synchronize(self._pos.device)
        return {"converged": self._is_host[:, 2] != 0, "failed": self._is_host[:, 3] != 0,
                "steps": self._is_host[:, 4].clone(), "pos": self._pos.cpu(), "cell": self._cell.cpu(),
                "log": {name: log[:, :, j].clone() for j, name in enumerate(LOG_FIELDS)}}
