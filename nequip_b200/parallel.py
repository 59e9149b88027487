"""Spatial decomposition of one frame over GPUs with a per-layer halo exchange (host side).

The reference's only sharded-inference design is LAMMPS domain decomposition surfaced to the
model as owned + ghost atoms and a per-layer ghost-feature exchange hook
(``nequip/nn/_ghost_exchange_base.py:8-57``, ``nequip/nn/_ghost_exchange_lmp_mliap.py:11-64``,
``nequip/nn/interaction_block.py:159-199``; inputs in the ML-IAP convention,
``nequip/integrations/lammps_mliap/lmp_mliap_wrapper.py:202-219``).  This module is the
H100-native equivalent with ``torch.distributed`` (NCCL over NVLink; gloo in the CPU tests):

* atoms are split into ``gx x gy x gz`` bricks of equal atom counts (``brick_grid`` picks the
  factorisation with the smallest halo volume: slabs for an elongated box, 3-D bricks for a cubic
  one); a rank *owns* its brick and additionally holds *ghost* copies of every non-owned atom that
  is the source of an edge whose destination it owns -- so every scatter destination is local and
  the TP+scatter kernel never crosses ranks;
* before every interaction layer >= 1 the owners' current features are sent to the ranks
  that hold ghosts of them (``all_to_all_single`` with split sizes, received straight into the
  tail of the feature buffer); the backward of that exchange is the transposed exchange with
  accumulation into the owner rows (what LAMMPS' ``reverse_exchange`` does);
* energies: sum over owned atoms then one 8-byte all-reduce; forces stay with their owners: the
  gradient w.r.t. ghost positions travels back through one more transposed exchange
  (``owner_reduce``, O(N / P) per rank).  A dense ``[N, 3]`` all-reduce (``reduce_forces="global"``)
  is kept for tests and small frames.
* the whole sharded step is capturable as one CUDA graph per rank (``graph.GraphedShardedEnergyForces``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
import torch.distributed as dist


@dataclass
class ShardPlan:
    rank: int
    world: int
    num_global: int
    owned: torch.Tensor  # [n_own] global ids (ascending)
    ghosts: torch.Tensor  # [n_ghost] global ids, grouped by owner rank (ascending rank, then id)
    local_ids: torch.Tensor  # [n_own + n_ghost] global ids of the local numbering
    edge_index: torch.Tensor  # [2, E_loc] local numbering; dst (row 0) always < n_own
    edge_ids: torch.Tensor  # [E_loc] positions in the global edge list
    send_idx: torch.Tensor  # [sum send] local owned indices to send, grouped by destination rank
    send_splits: List[int]
    recv_splits: List[int]  # ghosts received from each rank (matches the grouping of ``ghosts``)

    @property
    def n_own(self) -> int:
        return int(self.owned.numel())

    @property
    def n_ghost(self) -> int:
        return int(self.ghosts.numel())


def slab_owner(pos: torch.Tensor, world: int, axis: int = 0) -> torch.Tensor:
    """Owner rank of every atom: equal-count slabs along ``axis`` (stable in atom order)."""
    N = pos.shape[0]
    order = torch.argsort(pos[:, axis], stable=True)
    owner = torch.empty(N, dtype=torch.long)
    bounds = [(N * r) // world for r in range(world + 1)]
    for r in range(world):
        owner[order[bounds[r]: bounds[r + 1]]] = r
    return owner


def brick_grid(world: int, lengths, halo: float = 5.0) -> tuple:
    """Factorisation (gx, gy, gz) of ``world`` whose bricks of a box with edge ``lengths`` have the smallest
    halo volume (= fewest ghost atoms) for a halo of thickness ``halo``: elongated boxes get slabs, cubic
    boxes 3-D bricks."""
    best, best_v = (world, 1, 1), None
    for gx in range(1, world + 1):
        if world % gx:
            continue
        for gy in range(1, world // gx + 1):
            if (world // gx) % gy:
                continue
            gz = world // gx // gy
            dims = [lengths[0] / gx, lengths[1] / gy, lengths[2] / gz]
            # a direction that is split (or periodic with one brick thinner than the box) grows by the halo on both sides
            grown = [min(L, d + 2 * halo) if g > 1 else d for d, g, L in zip(dims, (gx, gy, gz), lengths)]
            vol = grown[0] * grown[1] * grown[2] - dims[0] * dims[1] * dims[2]
            if best_v is None or vol < best_v - 1e-9:
                best, best_v = (gx, gy, gz), vol
    return best


def brick_owner(pos: torch.Tensor, grid) -> torch.Tensor:
    """Owner rank of every atom for a ``grid = (gx, gy, gz)`` brick decomposition with equal atom counts:
    equal-count slabs along x, each cut into equal-count columns along y, each cut along z
    (rank = (ix * gy + iy) * gz + iz).  ``grid = (world, 1, 1)`` reproduces ``slab_owner``."""
    N = pos.shape[0]
    owner = torch.zeros(N, dtype=torch.long)

    def split(ids: torch.Tensor, axis: int, parts: int):
        order = ids[torch.argsort(pos[ids, axis], stable=True)]
        n = order.numel()
        return [order[(n * r) // parts: (n * (r + 1)) // parts] for r in range(parts)]

    gx, gy, gz = (int(g) for g in grid)
    for ix, sx in enumerate(split(torch.arange(N), 0, gx)):
        for iy, sy in enumerate(split(sx, 1, gy)):
            for iz, sz in enumerate(split(sy, 2, gz)):
                owner[sz] = (ix * gy + iy) * gz + iz
    return owner


def make_plans(edge_index: torch.Tensor, owner: torch.Tensor, world: int) -> List[ShardPlan]:
    """All ranks' plans from the global edge list (host-side preprocessing, like the neighbour list).
    ``edge_index[0]`` = destination/centre, ``edge_index[1]`` = source/neighbour."""
    N = owner.numel()
    dst, src = edge_index[0], edge_index[1]
    plans: List[ShardPlan] = []
    need: List[List[torch.Tensor]] = [[None] * world for _ in range(world)]  # need[r][s]: ids owned by s that r ghosts
    owned_ids, ghost_ids, edges, eids = [], [], [], []
    for r in range(world):
        own = torch.nonzero(owner == r).view(-1)
        emask = owner[dst] == r
        e_ids = torch.nonzero(emask).view(-1)
        s_glob = src[e_ids]
        gsrc = torch.unique(s_glob[owner[s_glob] != r])
        # group ghosts by owner rank
        gowner = owner[gsrc]
        order = torch.argsort(gowner * (N + 1) + gsrc)
        gsrc = gsrc[order]
        for s in range(world):
            need[r][s] = gsrc[owner[gsrc] == s]
        owned_ids.append(own)
        ghost_ids.append(gsrc)
        eids.append(e_ids)
    for r in range(world):
        own, gh = owned_ids[r], ghost_ids[r]
        local_ids = torch.cat([own, gh])
        g2l = torch.full((N,), -1, dtype=torch.long)
        g2l[local_ids] = torch.arange(local_ids.numel())
        e_ids = eids[r]
        ei = torch.stack([g2l[dst[e_ids]], g2l[src[e_ids]]])
        assert int(ei.min()) >= 0 and (int(ei[0].max()) < own.numel() if e_ids.numel() else True)
        send_lists = [need[s][r] for s in range(world)]  # what rank s needs from me
        send_idx = torch.cat([g2l[t] for t in send_lists]) if world > 0 else torch.empty(0, dtype=torch.long)
        plans.append(
            ShardPlan(
                rank=r, world=world, num_global=N, owned=own, ghosts=gh, local_ids=local_ids, edge_index=ei,
                edge_ids=e_ids, send_idx=send_idx, send_splits=[int(t.numel()) for t in send_lists],
                recv_splits=[int(need[r][s].numel()) for s in range(world)],
            )
        )
    return plans


def shard_data(data: Dict[str, torch.Tensor], plan: ShardPlan) -> Dict[str, torch.Tensor]:
    """AtomicDataDict-shaped local view: owned atoms first, then ghosts (ML-IAP convention)."""
    out = {
        "pos": data["pos"][plan.local_ids],
        "atom_types": data["atom_types"][plan.local_ids],
        "edge_index": plan.edge_index,
    }
    if "cell" in data:
        out["cell"] = data["cell"]
        out["edge_cell_shift"] = data["edge_cell_shift"][plan.edge_ids]
    return out


class _HaloExchangeFn(torch.autograd.Function):
    """x_own [n_own, D] -> x_full [n_own + n_ghost, D]; backward adds ghost grads into the owners."""

    @staticmethod
    def forward(ctx, x_own, send_idx, send_splits, recv_splits, group):
        ctx.send_idx, ctx.send_splits, ctx.recv_splits, ctx.group = send_idx, send_splits, recv_splits, group
        ctx.n_own = x_own.shape[0]
        send = x_own.index_select(0, send_idx)
        # owned rows and received ghost rows share ONE buffer: the collective writes its tail in place
        # (no torch.cat copy of the whole feature matrix)
        full = x_own.new_empty((ctx.n_own + sum(recv_splits),) + tuple(x_own.shape[1:]))
        full[: ctx.n_own].copy_(x_own)
        dist.all_to_all_single(full[ctx.n_own:], send, output_split_sizes=recv_splits, input_split_sizes=send_splits,
                               group=group)
        return full

    @staticmethod
    def backward(ctx, g_full):
        g_own = g_full[: ctx.n_own].clone()
        g_ghost = g_full[ctx.n_own:].contiguous()
        back = g_full.new_empty((sum(ctx.send_splits),) + tuple(g_full.shape[1:]))
        dist.all_to_all_single(back, g_ghost, output_split_sizes=ctx.send_splits, input_split_sizes=ctx.recv_splits,
                               group=ctx.group)
        g_own.index_add_(0, ctx.send_idx, back)
        return g_own, None, None, None, None


class HaloExchange:
    def __init__(self, plan: ShardPlan, device, group=None):
        self.plan, self.group = plan, group
        self.send_idx = plan.send_idx.to(device)

    def __call__(self, x_own: torch.Tensor) -> torch.Tensor:
        if self.plan.world == 1:
            return x_own
        return _HaloExchangeFn.apply(x_own, self.send_idx, self.plan.send_splits, self.plan.recv_splits, self.group)


def owner_reduce(g_local: torch.Tensor, plan: ShardPlan, halo: "HaloExchange") -> torch.Tensor:
    """Per-atom quantity over owned + ghost atoms -> owned atoms: the ghost rows travel back to their owners
    (transposed halo exchange) and are added there.  ``[n_own + n_ghost, C] -> [n_own, C]``."""
    g_own = g_local[: plan.n_own].clone()
    if plan.world > 1:
        back = g_local.new_empty((sum(plan.send_splits),) + tuple(g_local.shape[1:]))
        dist.all_to_all_single(back, g_local[plan.n_own:].contiguous(), output_split_sizes=plan.send_splits,
                               input_split_sizes=plan.recv_splits, group=halo.group)
        g_own.index_add_(0, halo.send_idx, back)
    return g_own


def sharded_energy_forces(model, local: Dict[str, torch.Tensor], plan: ShardPlan, halo: HaloExchange,
                          reduce_forces=True):
    """Energy + forces of one frame sharded over ``plan.world`` ranks.

    ``model`` is a ``NequIPEnergyModel``; ``local`` the rank's ``shard_data`` on its device.
    Returns ``(total_energy [1] f64 -- identical on all ranks, forces)`` where ``forces`` depends on
    ``reduce_forces``:

    * ``"owner"`` -- ``[n_own, 3]``: the forces of the atoms this rank owns.  The gradient that the local
      energy has w.r.t. the positions of GHOST atoms is sent back to their owners with the transposed halo
      exchange (``[n_ghost, 3]`` doubles per rank -- what LAMMPS' reverse communication does,
      nequip/integrations/lammps_mliap/lmp_mliap_wrapper.py:202-219), so the cost per rank is O(N / P);
    * ``True`` / ``"global"`` -- ``[N_global, 3]`` on every rank (dense all-reduce; for tests and small frames);
    * ``False`` -- the raw local gradient ``-dE_local/dpos`` over owned + ghost atoms.
    """
    pos = local["pos"].detach().requires_grad_(True)
    d = dict(local)
    d["pos"] = pos
    with torch.enable_grad():
        e_atom_own = model.energy_owned(d, plan.n_own, halo)
        e_loc = e_atom_own.sum()
        (g,) = torch.autograd.grad([e_loc], [pos])
    e = e_loc.detach().reshape(1).clone()
    if plan.world > 1:
        dist.all_reduce(e, group=halo.group)
    if reduce_forces is False:
        return e, -g
    if reduce_forces == "owner":
        return e, -owner_reduce(g, plan, halo)
    f = torch.zeros((plan.num_global, 3), dtype=g.dtype, device=g.device)
    f.index_add_(0, plan.local_ids.to(g.device), -g)
    if plan.world > 1:
        dist.all_reduce(f, group=halo.group)
    return e, f
