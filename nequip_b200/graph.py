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
"""
from __future__ import annotations

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
