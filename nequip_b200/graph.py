"""CUDA-graph replay of the energy + forces step for a fixed (atoms, edges) shape.

One eager step of the 4-layer model is ~260 kernel launches, and the gaps between them add up.  The whole step -- edge embedding, every
interaction layer, readout and the backward pass that yields the forces -- is captured once into a CUDA
graph and replayed; inputs are copied into static buffers, outputs are read from static buffers.

The reference reaches the same goal with a tracing compiler (``nequip-compile`` -> AOTInductor,
nequip/scripts/_compile_utils.py, nequip/nn/compile.py); here the hand-written kernels are captured
as they are.

A graph is valid for one (num_atoms, num_edges) pair and for edge lists grouped by destination (what the
reference's neighbour lists produce, nequip/data/transforms/neighborlist.py:120-157); the sortedness flag
is computed inside the graph and verified when the results are read.  Anything else: use the eager
``model(data)`` call (same kernels, more launch overhead).

``GraphedMDStep`` lifts the shape restriction for molecular dynamics in a fixed cell (periodic, partly periodic
like a slab, or none for a molecule in vacuum): the device neighbour
list (``ops.NeighborListPlan``) is part of the graph and writes a list of fixed length ``capacity`` whose unused
slots hold null edges, which contribute exactly zero (DESIGN.md section 4.8).  So one graph replays every step
whatever the step's edge count, and a step that needs more than ``capacity`` edges is re-captured.  With
``variable_cell=True`` the cell is an input of every step as well (constant-pressure MD): the neighbour list reads it
from a device parameter block that is refreshed before each replay, and the step also returns stress and virial.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ops

_INPUT_KEYS = ("pos", "cell", "atom_types", "edge_index", "edge_cell_shift")


class GraphedEnergyForces:
    """``g = GraphedEnergyForces(model, example); out = g(data)`` with ``data`` of the example's shapes.

    ``out`` holds ``total_energy`` [1] and ``forces`` [N, 3] -- views of static buffers that the next call
    overwrites (clone them to keep them)."""

    def __init__(self, model, example: Dict[str, torch.Tensor], warmup: int = 3):
        dev = example["pos"].device
        if dev.type != "cuda":
            raise RuntimeError("GraphedEnergyForces needs CUDA tensors (there is no CPU path)")
        self.model = model
        self.static: Dict[str, torch.Tensor] = {k: example[k].clone() for k in _INPUT_KEYS if k in example}
        self.extra = {k: v for k, v in example.items() if k not in self.static}
        self.shapes = {k: tuple(v.shape) for k, v in self.static.items()}
        self.graph = torch.cuda.CUDAGraph()
        self._sorted_flags = []
        # warm-up on a side stream (lazy library loads, cudaFuncSetAttribute, allocator pools)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        ops.csr_cache.clear()
        from . import _capi

        n0 = _capi.launch_count()
        with torch.cuda.graph(self.graph):
            with ops.deferred_sorted_check() as chk:
                out = self._run()
            self._sorted_flags = list(chk.flags)
            self.energy = out["total_energy"]
            self.forces = out["forces"]
            self.sorted_flag = (torch.stack([f.view(()) for f in self._sorted_flags]).min().view(1)
                                if self._sorted_flags else torch.ones(1, dtype=torch.int32, device=dev))
        ops.csr_cache.clear()  # the cached CSR lives in the graph's private pool
        self.launches_per_replay = _capi.launch_count() - n0  # nequip_b200 kernels captured (torch's are extra)
        self.replays = 0
        # the "edges grouped by destination" flag of every replay is copied to pinned host memory right after
        # the graph and checked when the NEXT replay is issued (or by check_sorted()): an unsorted neighbour
        # list of the captured shape can therefore never go unnoticed for more than one step
        self._flag_host = torch.ones(1, dtype=torch.int32).pin_memory()
        self._flag_event: Optional[torch.cuda.Event] = None

    def _run(self):
        d = dict(self.extra)
        d.update(self.static)
        return self.model(d)


    def matches(self, data: Dict[str, torch.Tensor]) -> bool:
        return all(k in data and tuple(data[k].shape) == s for k, s in self.shapes.items())

    def load(self, data: Dict[str, torch.Tensor]) -> None:
        """Copy a frame into the static input buffers (host tensors: asynchronous H2D when pinned)."""
        for k, buf in self.static.items():
            src = data[k]
            if tuple(src.shape) != tuple(buf.shape):
                raise ValueError(f"GraphedEnergyForces was captured for {k} of shape {tuple(buf.shape)}, got {tuple(src.shape)}")
            buf.copy_(src, non_blocking=True)

    def _verify_previous(self) -> None:
        if self._flag_event is not None:
            self._flag_event.synchronize()
            self._flag_event = None
            if int(self._flag_host[0]) != 1:
                raise RuntimeError("GraphedEnergyForces: the previous frame's edge_index was not grouped by "
                                   "destination -- its energies/forces are invalid; use the eager model call")

    def replay(self) -> Dict[str, torch.Tensor]:
        self._verify_previous()
        self.graph.replay()
        self.replays += 1
        self._flag_host.copy_(self.sorted_flag, non_blocking=True)
        self._flag_event = torch.cuda.Event()
        self._flag_event.record()
        return {"total_energy": self.energy, "forces": self.forces, "edges_sorted": self.sorted_flag}

    def __call__(self, data: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        if data is not None:
            self.load(data)
        return self.replay()

    def check_sorted(self) -> None:
        """Host-side verification of the in-graph sortedness flag (synchronises)."""
        self._verify_previous()
        if int(self.sorted_flag.item()) != 1:
            raise RuntimeError("GraphedEnergyForces: edge_index is not grouped by destination; use the eager model call")


class GraphedShardedEnergyForces(GraphedEnergyForces):
    """The same replay for ONE RANK of a spatially decomposed frame (nequip_b200/parallel.py): the captured step
    contains the per-layer NCCL halo exchanges, the energy all-reduce and the reverse exchange that returns the
    ghost-position gradients to their owners (NCCL collectives are capturable).  ``forces`` are those of the
    OWNED atoms ``[n_own, 3]``.  Every rank must construct and replay it collectively."""

    def __init__(self, model, local: Dict[str, torch.Tensor], plan, halo, warmup: int = 3):
        self.plan, self.halo = plan, halo
        super().__init__(model, local, warmup=warmup)

    def _run(self):
        from . import parallel as P

        d = dict(self.extra)
        d.update(self.static)
        e, f = P.sharded_energy_forces(self.model, d, self.plan, self.halo, reduce_forces="owner")
        return {"total_energy": e, "forces": f}


#: default edge capacity of GraphedMDStep: E0 * (1 + CAPACITY_SLACK), E0 = the example frame's edge count
CAPACITY_SLACK = 0.02


class GraphedMDStep(GraphedEnergyForces):
    """One CUDA graph for a whole MD step: positions -> device neighbour list -> energy -> forces.
    ``g = GraphedMDStep(model, example); out = g(pos)``.

    ``example`` holds CUDA tensors ``pos`` [N,3], ``atom_types`` [N] and, for a periodic system, ``cell`` [3,3].
    The periodicity is ``example["pbc"]`` ([3] or [1, 3] bools) when present; otherwise all three directions are
    periodic with a cell and all open without one (a molecule in vacuum).  Along open directions the neighbour list
    finds the positions' bounding box on the device at every replay (``ops.NeighborListPlan(open_boundaries=True)``),
    and the captured model call reads the plan's cell (``plan.cell``, the identity without a cell), to which the null
    edges' shift refers.  By default the cell is captured (NVE / NVT).  ``capacity`` is the length of the edge buffer,
    by default ``E0 + ceil(CAPACITY_SLACK * E0)`` with E0 the example's edge count (``ops.neighbor_list`` with the
    example's cell and periodicity); unused slots hold null edges.

    ``g(pos)`` takes host (pinned) or device positions and returns ``total_energy`` [1,1], ``atomic_energy`` [N,1],
    ``forces`` [N,3] and ``num_edges`` [1] -- views of static buffers that the next call overwrites.  Every call
    reads the step's edge count and overflow flag back (12 bytes, one event wait) and checks that the list was grouped
    by destination.  If the step needed more than ``capacity`` edges, the graph is re-captured with
    ``capacity = ceil(1.02 * needed)`` and the same positions are computed again, so a returned result never comes
    from a truncated list; ``capacity`` only grows and ``recaptures`` counts the re-captures.

    A model with per-edge-type cutoffs (``per_edge_type_cutoff``) gets a neighbour list pruned by its table: the
    default capacity is sized from the pruned count, and the atom types of ``example`` are fixed for the graph.

    ``variable_cell=True`` (NPT): ``g(pos, cell)`` also takes the step's cell ([3,3], host or device; a device cell
    costs one device-to-host read).  It is copied into the static ``cell`` input the model reads and handed to the
    neighbour list (``ops.NeighborListPlan.set_cell``) before the replay.  The captured call is
    ``model(d, compute_stress=True)``, so the outputs also hold ``stress`` and ``virial`` [1,3,3].  A re-capture
    happens at the current cell, with a bin grid chosen for it.  ``variable_cell`` needs all three directions periodic
    (``ValueError`` otherwise).

    A batch of independent frames (torch-sim's input): ``example`` also holds ``batch`` [N] (non-decreasing) and
    ``num_atoms`` [F], ``cell`` is [F, 3, 3] or absent and ``pbc``, when present, is [F, 3] (or [3] for every frame).
    One graph then holds the step of every frame: one batched device list of one ``capacity``
    (``ops.NeighborListPlan(batch=)``, each frame with its own cell, grid and null-edge shift) and one model call on
    ``plan.cell`` [F, 3, 3].  The default capacity is sized from the batched ``ops.neighbor_list`` count.  ``g(pos)``
    returns ``total_energy`` [F, 1]; with ``variable_cell=True``, ``g(pos, cells)`` takes [F, 3, 3] and returns
    ``stress`` and ``virial`` [F, 3, 3].  The frames and their atom counts are fixed for the graph (a different batch
    needs a new ``GraphedMDStep``); ``batch`` and ``num_atoms`` are copied into the graph's static inputs, so the
    captured model call reads the frame count without a host synchronisation."""

    def __init__(self, model, example: Dict[str, torch.Tensor], capacity: Optional[int] = None, warmup: int = 3,
                 variable_cell: bool = False):
        cell = example.get("cell")
        self.pbc = self._periodicity(example)
        if cell is None and any(self._flags()):
            raise ValueError("GraphedMDStep: a periodic direction needs a cell")
        if variable_cell and not all(self._flags()):
            raise ValueError("GraphedMDStep: variable_cell needs all three directions periodic")
        if example["pos"].device.type != "cuda":
            raise RuntimeError("GraphedMDStep needs CUDA tensors (there is no CPU path)")
        self._frames = None
        if example.get("batch") is not None:
            dev = example["pos"].device
            self._frames = {"batch": example["batch"].to(dev).view(-1).clone(),
                            "num_atoms": torch.as_tensor(example["num_atoms"]).to(dev).view(-1).clone()}
        if capacity is None:
            e0 = int(ops.neighbor_list(example["pos"], cell, self.pbc, model.r_max,
                                       **self._edge_type_args(model, example),
                                       **({} if self._frames is None else {"batch": self._frames["batch"]})
                                       )["edge_index"].shape[1])
            capacity = e0 + math.ceil(CAPACITY_SLACK * e0)
        self.variable_cell = bool(variable_cell)
        self.recaptures = 0
        self._warmup = warmup
        self._num_edges_host = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._overflow_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._capture(model, {k: example[k] for k in ("pos", "atom_types", "cell") if example.get(k) is not None},
                      int(capacity))

    def _flags(self) -> list:
        """Every periodicity flag of the step (3, or 3 per frame of a batch)."""
        return [b for row in self.pbc for b in (row if isinstance(row, tuple) else (row,))]

    @staticmethod
    def _periodicity(example: Dict[str, torch.Tensor]) -> tuple:
        """3 bools: ``example["pbc"]`` ([3] or [1, 3], or one bool) when present, else all periodic with a cell and
        all open without one.  A batch (``example["batch"]``) with ``pbc`` [F, 3]: F tuples of 3 bools."""
        pbc = example.get("pbc")
        if pbc is None:
            return (example.get("cell") is not None,) * 3
        if example.get("batch") is not None and torch.as_tensor(pbc).dim() == 2:
            return tuple(tuple(bool(b) for b in row) for row in torch.as_tensor(pbc).tolist())
        flags = [bool(b) for b in torch.as_tensor(pbc).reshape(-1).tolist()]
        if len(flags) == 1:
            flags *= 3
        if len(flags) != 3:
            raise ValueError(f"GraphedMDStep: pbc must hold 3 flags, got {len(flags)}")
        return tuple(flags)

    @staticmethod
    def _edge_type_args(model, example: Dict[str, torch.Tensor]) -> dict:
        """The neighbour list's per-edge-type cutoffs: the model's table and the frame's (static) atom types."""
        table = getattr(model, "per_edge_type_cutoff", None)
        return {} if table is None else dict(atom_types=example["atom_types"], edge_type_cutoff=table)

    def _capture(self, model, example: Dict[str, torch.Tensor], capacity: int) -> None:
        self.capacity = capacity
        is_open = not all(self._flags())
        frames = {}
        if self._frames is not None:
            example = dict(example, **self._frames)
            frames = {"batch": self._frames["batch"]}
        self.plan = ops.NeighborListPlan(example["pos"].shape[0], example.get("cell"), self.pbc, model.r_max, capacity,
                                         device=example["pos"].device, variable_cell=self.variable_cell,
                                         **self._edge_type_args(model, example), open_boundaries=is_open, **frames)
        if is_open or frames:
            # the null edges' shift refers to plan.cell (the identity without a cell, [F, 3, 3] for a batch): the
            # model must see it
            example = dict(example, cell=self.plan.cell)
        super().__init__(model, example, warmup=self._warmup)
        ops.src_csr_cache.clear()  # like csr_cache: an entry made during the capture lives in the graph's pool
        out, self._out = self._out, None
        self.atomic_energy, self.num_edges, self.overflow = out["atomic_energy"], out["num_edges"], out["overflow"]
        self.stress, self.virial = out.get("stress"), out.get("virial")

    def _run(self):
        nl = self.plan.run(self.static["pos"])
        d = dict(self.extra)
        d.update(self.static)
        d["edge_index"], d["edge_cell_shift"] = nl["edge_index"], nl["edge_cell_shift"]
        out = self.model(d, compute_stress=True) if self.variable_cell else self.model(d)
        self._out = {"atomic_energy": out["atomic_energy"], "num_edges": nl["num_edges"], "overflow": nl["overflow"]}
        if self.variable_cell:
            self._out.update(stress=out["stress"], virial=out["virial"])
        return out

    def _recapture(self, capacity: int) -> None:
        example = {k: v.clone() for k, v in self.static.items()}  # the positions that overflowed
        replays = self.replays
        # drop every reference into the old graph's memory pool so that it is released with the graph
        self.graph = self.plan = None
        self.energy = self.forces = self.atomic_energy = self.num_edges = self.overflow = self.sorted_flag = None
        self.stress = self.virial = None
        self._sorted_flags = []
        self._flag_event = None
        self._capture(self.model, example, capacity)
        self.replays = replays
        self.recaptures += 1

    def __call__(self, pos: torch.Tensor, cell: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        if self.variable_cell:
            if cell is None:
                raise ValueError("GraphedMDStep(variable_cell=True) needs the step's cell: g(pos, cell)")
            self.plan.set_cell(cell)  # checks the cell before anything is copied
            self.static["cell"].copy_(torch.as_tensor(cell).reshape(self.static["cell"].shape), non_blocking=True)
        elif cell is not None:
            raise ValueError("this GraphedMDStep was captured for a fixed cell; build it with variable_cell=True")
        self.static["pos"].copy_(pos, non_blocking=True)
        while True:
            self.replay()
            self._num_edges_host.copy_(self.num_edges, non_blocking=True)
            self._overflow_host.copy_(self.overflow, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
            self._verify_previous()
            if int(self._overflow_host[0]) == 0:
                break
            needed = int(self._num_edges_host[0])
            self._recapture(max(self.capacity + 1, math.ceil(1.02 * needed)))
        out = {"total_energy": self.energy, "atomic_energy": self.atomic_energy, "forces": self.forces,
               "num_edges": self.num_edges}
        if self.variable_cell:
            out.update(stress=self.stress, virial=self.virial)
        return out
