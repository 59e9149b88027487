"""Host-side (PyTorch) mirror of the NequIP energy model around the fused kernels.

This is *plumbing*: the module order, irreps bookkeeping, initialisation and
normalisation constants of the reference's model builder, so that the hot-path
kernels can be driven end to end (energy + forces) on identical
``AtomicDataDict``-shaped batches without e3nn/nequip installed.  Everything on the
per-edge hot path goes through ``nequip_b200.ops`` (CUDA); node-side dense algebra
uses torch matmul (cuBLAS, fp32, TF32 off).

Reference files mirrored (under /root/reference):
  model assembly          nequip/model/nequip_models.py:116-210 (NequIPGNNModel), :214-399 (Full...)
  ConvNetLayer            nequip/nn/convnetlayer.py:74-170
  InteractionBlock        nequip/nn/interaction_block.py:21-207
  ScalarMLPFunction       nequip/nn/mlp.py:80-195, ScalarLinearLayer :223-271
  AvgNumNeighborsNorm     nequip/nn/norm.py:7-68
  NodeTypeEmbed           nequip/nn/embedding/node.py:146-175
  PerTypeScaleShift       nequip/nn/atomwise.py:236-284;  AtomwiseReduce :92-113
  ForceStressOutput       nequip/nn/grad_output.py:107-298 (forces only)
  e3nn o3.Linear / FullyConnectedTensorProduct / nn.Gate semantics: SURVEY.md Appendix A.4
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from .. import ops
from ..irreps import Irrep, Irreps, build_tp_instructions, tp_path_exists
from .pair import ZBL, ZBL_TARGET, parse_pair_potential
from .tp_scatter import B200TensorProductScatter

# e3nn.math.normalize2mom constants: (E_{z~N(0,1)} act(z)^2)^(-1/2) estimated from
# torch.randn(1_000_000, generator=Generator("cpu").manual_seed(0), dtype=float64)
C_SILU = 1.6791767923989418
C_TANH = 1.5937334472592692

# AtomicDataDict keys used here (nequip/data/_keys.py:14-115)
POSITIONS_KEY = "pos"
EDGE_INDEX_KEY = "edge_index"
EDGE_CELL_SHIFT_KEY = "edge_cell_shift"
CELL_KEY = "cell"
ATOM_TYPE_KEY = "atom_types"
TOTAL_ENERGY_KEY = "total_energy"
PER_ATOM_ENERGY_KEY = "atomic_energy"
FORCE_KEY = "forces"
STRESS_KEY = "stress"
VIRIAL_KEY = "virial"
EDGE_VECTORS_KEY = "edge_vectors"
EDGE_FORCE_KEY = "edge_forces"
BATCH_KEY = "batch"
BATCH_PTR_KEY = "ptr"
NUM_NODES_KEY = "num_atoms"


# ---------------------------------------------------------------------------------------
# irreps bookkeeping of the conv stack
# ---------------------------------------------------------------------------------------
def feature_widths(l_max: int, num_features) -> List[int]:
    """One width per degree 0..l_max: an int applies to every degree, a list is taken as is
    (nequip_models.py:164-169)."""
    if isinstance(num_features, int):
        return [num_features] * (l_max + 1)
    widths = [int(f) for f in num_features]
    if len(widths) != l_max + 1:
        raise ValueError(f"num_features: expected an int or l_max + 1 = {l_max + 1} widths, got {list(num_features)}")
    return widths


def hidden_irreps(l_max: int, num_features, parity: bool) -> Irreps:
    """``feature_irreps_hidden`` of NequIPGNNModel (nequip_models.py:176-187); ``num_features`` is an int or one
    width per degree."""
    widths = feature_widths(l_max, num_features)
    items = []
    for l in range(l_max + 1):
        ps = (1, -1) if parity else ((1,) if l % 2 == 0 else (-1,))
        for p in ps:
            items.append((widths[l], Irrep(l, p)))
    return Irreps(items)


def gate_irreps(prev: Irreps, edge_attr: Irreps, hidden: Irreps):
    """Irreps decisions of ConvNetLayer.__init__ (convnetlayer.py:74-114) for the gate nonlinearity.
    Returns (irreps_scalars, irreps_gates, irreps_gated, conv_irreps_out, layer_out)."""
    scalars = Irreps([(mul, ir) for mul, ir in hidden if ir.l == 0 and tp_path_exists(prev, edge_attr, ir)])
    gated = Irreps([(mul, ir) for mul, ir in hidden if ir.l > 0 and tp_path_exists(prev, edge_attr, ir)])
    gate_ir = Irrep(0, 1) if tp_path_exists(prev, edge_attr, Irrep(0, 1)) else Irrep(0, -1)
    gates = Irreps([(mul, gate_ir) for mul, _ in gated])
    conv_out = (scalars + gates + gated).simplify()
    # Gate.irreps_out = scalars + gated (with gates of even parity the gated irreps are unchanged)
    gated_out = Irreps([(mul, Irrep(ir.l, ir.p * gate_ir.p)) for mul, ir in gated])
    layer_out = scalars + gated_out
    return scalars, gates, gated, conv_out, layer_out


def layer_irreps(l_max: int, num_features, num_layers: int, parity: bool = True, type_embed_num_features=None):
    """[(feature_irreps_in, irreps_edge_attr, conv_irreps_out, (scalars, gates, gated))] per layer."""
    widths = feature_widths(l_max, num_features)
    f0 = type_embed_num_features or widths[0]
    edge_attr = Irreps.spherical_harmonics(l_max)
    prev = Irreps([(f0, Irrep(0, 1))])
    hid = hidden_irreps(l_max, widths, parity)
    hiddens = [hid] * (num_layers - 1) + [Irreps([(widths[0], Irrep(0, 1))])]
    out = []
    for h in hiddens:
        scalars, gates, gated, conv_out, layer_out = gate_irreps(prev, edge_attr, h)
        out.append((prev, edge_attr, conv_out, (scalars, gates, gated)))
        prev = layer_out
    return out


# ---------------------------------------------------------------------------------------
# dense pieces (torch)
# ---------------------------------------------------------------------------------------
class ScalarLinearLayer(torch.nn.Module):
    """mlp.py:223-271: ``mm(input, weight * alpha)``, weight ~ U(-sqrt3, sqrt3)."""

    def __init__(self, in_features: int, out_features: int, alpha: float = 1.0):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.register_buffer("alpha", torch.tensor(alpha), persistent=False)
        self.weight = torch.nn.Parameter(torch.empty((in_features, out_features)))
        torch.nn.init.uniform_(self.weight, -math.sqrt(3), math.sqrt(3))

    def forward(self, x):
        return torch.mm(x, self.weight * self.alpha)


class ScalarMLPFunction(torch.nn.Module):
    """mlp.py:80-195 with ``bias=False, forward_weight_init=True, nonlinearity="silu"``."""

    def __init__(self, input_dim: int, output_dim: int, hidden_layers_depth: int = 0,
                 hidden_layers_width: Optional[int] = None, nonlinearity: Optional[str] = "silu"):
        super().__init__()
        dims = [input_dim] + hidden_layers_depth * [hidden_layers_width] + [output_dim]
        self.dims = dims
        layers: List[torch.nn.Module] = []
        nl = len(dims) - 1
        for layer, (h_in, h_out) in enumerate(zip(dims, dims[1:])):
            gain = 1.0 if nonlinearity is None or layer == 0 else math.sqrt(2)
            layers.append(ScalarLinearLayer(h_in, h_out, alpha=gain / math.sqrt(h_in)))
            if layer != nl - 1 and nonlinearity is not None:
                layers.append(torch.nn.SiLU())
        self.mlp = torch.nn.Sequential(*layers)

    def forward(self, x):
        return self.mlp(x)


class Linear(torch.nn.Module):
    """e3nn ``o3.Linear(irreps_in, irreps_out)`` (internal shared weights, no bias,
    path_normalization="element"): out_b = (1/sqrt(sum_a mul_a)) sum_a x_a W_ab over equal irreps."""

    def __init__(self, irreps_in, irreps_out, layout: str = "mul_ir"):
        super().__init__()
        self.layout = layout
        self.irreps_in, self.irreps_out = Irreps(irreps_in), Irreps(irreps_out)
        self.instr: List[Tuple[int, int, int, float]] = []  # (i_in, i_out, weight offset, path weight)
        off = 0
        pairs = [
            (i, o)
            for i, (_, ir_i) in enumerate(self.irreps_in)
            for o, (_, ir_o) in enumerate(self.irreps_out)
            if ir_i == ir_o
        ]
        for (i, o) in pairs:
            fan = sum(self.irreps_in[i2][0] for (i2, o2) in pairs if o2 == o)
            self.instr.append((i, o, off, 1.0 / math.sqrt(fan)))
            off += self.irreps_in[i][0] * self.irreps_out[o][0]
        self.weight_numel = off
        self.weight = torch.nn.Parameter(torch.randn(off))
        self._in_sl, self._out_sl = self.irreps_in.slices(), self.irreps_out.slices()

    def forward(self, x):
        N = x.shape[0]
        outs: List[Optional[torch.Tensor]] = [None] * len(self.irreps_out)
        for (i, o, off, pw) in self.instr:
            mi, ir = self.irreps_in[i]
            mo = self.irreps_out[o][0]
            W = self.weight[off: off + mi * mo].view(mi, mo) * pw
            if self.layout == "ir_mul":
                # chunk = [d, mi] per node: one GEMM over all (node, component) rows
                r = torch.matmul(x[:, self._in_sl[i]].reshape(N * ir.dim, mi), W).reshape(N, ir.dim * mo)
            else:
                xi = x[:, self._in_sl[i]].reshape(N, mi, ir.dim)
                # [N, d, mi] @ [mi, mo] -> [N, d, mo] -> [N, mo, d]
                r = torch.matmul(xi.transpose(1, 2), W).transpose(1, 2).reshape(N, mo * ir.dim)
            outs[o] = r if outs[o] is None else outs[o] + r
        for o, (mo, ir) in enumerate(self.irreps_out):
            if outs[o] is None:
                outs[o] = x.new_zeros(N, mo * ir.dim)
        return torch.cat(outs, dim=1)


class SelfConnection(torch.nn.Module):
    """e3nn ``FullyConnectedTensorProduct(feature_irreps_in, F0 x 0e, feature_irreps_out)``
    (interaction_block.py:140-146): out_b[w,k] = (1/sqrt(sum_a mul_a F0)) sum_a sum_uv W_ab[u,v,w] x_a[u,k] attr[v]."""

    def __init__(self, irreps_in, num_attr: int, irreps_out, layout: str = "mul_ir"):
        super().__init__()
        self.layout = layout
        self.irreps_in, self.irreps_out, self.num_attr = Irreps(irreps_in), Irreps(irreps_out), num_attr
        pairs = [
            (i, o)
            for i, (_, ir_i) in enumerate(self.irreps_in)
            for o, (_, ir_o) in enumerate(self.irreps_out)
            if ir_i == ir_o
        ]
        self.instr: List[Tuple[int, int, int, float]] = []
        off = 0
        for (i, o) in pairs:
            fan = sum(self.irreps_in[i2][0] * num_attr for (i2, o2) in pairs if o2 == o)
            self.instr.append((i, o, off, 1.0 / math.sqrt(fan)))
            off += self.irreps_in[i][0] * num_attr * self.irreps_out[o][0]
        self.weight_numel = off
        self.weight = torch.nn.Parameter(torch.randn(off))
        self._in_sl = self.irreps_in.slices()

    def forward(self, x, node_attrs, types=None, type_table=None):
        """Generic form: ``node_attrs`` [N, F0].  When the attributes are a per-type table
        (``node_attrs == type_table[types]``, which is how NequIP builds them,
        nequip/nn/embedding/node.py:146-175) the bilinear form collapses to one GEMM per irrep
        pair with the per-type effective weights  Weff[t] = sum_v W[:, v, :] table[t, v]."""
        N = x.shape[0]
        outs: List[Optional[torch.Tensor]] = [None] * len(self.irreps_out)
        fast = types is not None and type_table is not None
        if fast:
            T = type_table.shape[0]
            onehot = torch.nn.functional.one_hot(types, T).to(x.dtype)  # [N, T]
        for (i, o, off, pw) in self.instr:
            mi, ir = self.irreps_in[i]
            mo = self.irreps_out[o][0]
            W = self.weight[off: off + mi * self.num_attr * mo].view(mi, self.num_attr, mo)
            if self.layout == "ir_mul":
                xk = x[:, self._in_sl[i]].reshape(N, ir.dim, mi)  # [N, d, mi]
                if fast:
                    weff = torch.einsum("uvw,tv->tuw", W, type_table).reshape(T * mi, mo) * pw
                    xe = (onehot.view(N, 1, T, 1) * xk.unsqueeze(2)).reshape(N * ir.dim, T * mi)
                    r = torch.matmul(xe, weff).reshape(N, ir.dim * mo)
                else:
                    r = pw * torch.einsum("uvw,nku,nv->nkw", W, xk, node_attrs).reshape(N, ir.dim * mo)
                outs[o] = r if outs[o] is None else outs[o] + r
                continue
            xi = x[:, self._in_sl[i]].reshape(N, mi, ir.dim)
            if fast:
                weff = torch.einsum("uvw,tv->tuw", W, type_table).reshape(T * mi, mo) * pw
                # [N, d, T*mi] @ [T*mi, mo]
                xe = (onehot.view(N, 1, T, 1) * xi.transpose(1, 2).unsqueeze(2)).reshape(N, ir.dim, T * mi)
                r = torch.matmul(xe, weff).transpose(1, 2).reshape(N, mo * ir.dim)
            else:
                r = pw * torch.einsum("uvw,nuk,nv->nwk", W, xi, node_attrs).reshape(N, mo * ir.dim)
            outs[o] = r if outs[o] is None else outs[o] + r
        for o, (mo, ir) in enumerate(self.irreps_out):
            if outs[o] is None:
                outs[o] = x.new_zeros(N, mo * ir.dim)
        return torch.cat(outs, dim=1)


class Gate(torch.nn.Module):
    """e3nn ``nn.Gate`` with normalize2mom'd SiLU (even) / tanh (odd) (convnetlayer.py:42-56,104-112)."""

    def __init__(self, irreps_scalars, irreps_gates, irreps_gated, layout: str = "mul_ir"):
        super().__init__()
        self.layout = layout
        self.irreps_scalars, self.irreps_gates, self.irreps_gated = (
            Irreps(irreps_scalars), Irreps(irreps_gates), Irreps(irreps_gated))
        self.irreps_in = self.irreps_scalars + self.irreps_gates + self.irreps_gated
        gp = self.irreps_gates[0][1].p if len(self.irreps_gates) else 1
        self.irreps_out = self.irreps_scalars + Irreps([(m, Irrep(ir.l, ir.p * gp)) for m, ir in self.irreps_gated])
        self.use_fused = True  # CUDA: fused kernels; the torch formulation below is the readable definition
        self._tabs = None

    @staticmethod
    def _act(x, p: int):
        return torch.nn.functional.silu(x) * C_SILU if p == 1 else torch.tanh(x) * C_TANH

    def forward(self, x):
        if x.is_cuda and self.use_fused:
            # one kernel per direction (nqb_gate_fwd/bwd) instead of ~30 strided elementwise ops
            key = (x.device, self.layout)
            if self._tabs is None or self._tabs[0] != key:
                self._tabs = (key, ops.GateTables(self.irreps_scalars, self.irreps_gates, self.irreps_gated,
                                                  self.layout, x.device))
            return ops.gate(x, self._tabs[1])
        N = x.shape[0]
        ns, ng = self.irreps_scalars.dim, self.irreps_gates.dim
        parts = []
        off = 0
        for mul, ir in self.irreps_scalars:
            parts.append(self._act(x[:, off: off + mul], ir.p))
            off += mul
        if len(self.irreps_gated):
            gates = []
            goff = ns
            for mul, ir in self.irreps_gates:
                gates.append(self._act(x[:, goff: goff + mul], ir.p))
                goff += mul
            gates = torch.cat(gates, dim=1)
            off = ns + ng
            g0 = 0
            for mul, ir in self.irreps_gated:
                if self.layout == "ir_mul":
                    ch = x[:, off: off + mul * ir.dim].reshape(N, ir.dim, mul)
                    parts.append((ch * gates[:, g0: g0 + mul].unsqueeze(1)).reshape(N, mul * ir.dim))
                else:
                    ch = x[:, off: off + mul * ir.dim].reshape(N, mul, ir.dim)
                    parts.append((ch * gates[:, g0: g0 + mul].unsqueeze(-1)).reshape(N, mul * ir.dim))
                off += mul * ir.dim
                g0 += mul
        return torch.cat(parts, dim=1)


# ---------------------------------------------------------------------------------------
# graph modules
# ---------------------------------------------------------------------------------------
class InteractionBlock(torch.nn.Module):
    """interaction_block.py:21-207 (no ghost exchange here; see nequip_b200.parallel for the sharded path)."""

    def __init__(self, feature_irreps_in, irreps_edge_attr, feature_irreps_out, num_edge_embed: int,
                 num_node_attrs: int, radial_mlp_depth: int, radial_mlp_width: int, use_sc: bool,
                 avg_num_neighbors: float, is_first_layer: bool = False, layout: str = "mul_ir"):
        super().__init__()
        self.is_first_layer = is_first_layer
        self.layout = layout
        fin, fe, fout = Irreps(feature_irreps_in), Irreps(irreps_edge_attr), Irreps(feature_irreps_out)
        self.feature_irreps_in, self.irreps_edge_attr, self.feature_irreps_out = fin, fe, fout
        # AvgNumNeighborsNorm (nequip/nn/norm.py:7-68): a global value, or one per atom type (a sequence in
        # type order / the reference's dict after ordering by type_names); norm_const = 1 / sqrt(avg_num_neighbors)
        ann = [float(avg_num_neighbors)] if isinstance(avg_num_neighbors, (int, float)) else [float(v) for v in avg_num_neighbors]
        self.register_buffer("norm_const", torch.tensor([1.0 / math.sqrt(v) for v in ann]).reshape(-1, 1), persistent=False)
        self.norm_shortcut = len(ann) == 1
        self.linear_1 = Linear(fin, fin, layout)
        irreps_mid, instructions = build_tp_instructions(fin, fe, fout)
        self.irreps_mid, self.instructions = irreps_mid, instructions
        self.tp_scatter = B200TensorProductScatter(fin, fe, irreps_mid, instructions, layout=layout)
        self.edge_mlp = ScalarMLPFunction(num_edge_embed, self.tp_scatter.weight_numel,
                                          hidden_layers_depth=radial_mlp_depth,
                                          hidden_layers_width=radial_mlp_width, nonlinearity="silu")
        self.linear_2 = Linear(irreps_mid.simplify(), fout, layout)
        self.sc = SelfConnection(fin, num_node_attrs, fout, layout) if use_sc else None
        self.use_tensor_cores = True
        self.use_fused_radial_tp = "auto"  # SURVEY 8f-1 kernel (mul % 32 == 0, K <= 128): True / False / "auto" (timed once)
        self._fused_choice = None
        self.strict_fast_path = False
        self._tc_cache = None

    def _edge_weights(self, edge_embedding):
        """Radial MLP, plain torch.mm formulation of the reference (mlp.py:262-268) -- the path for trainable
        weights, float64 and unusual shapes; frozen float32 ir_mul models use ``_tensor_core_blocks``."""
        return self.edge_mlp(edge_embedding)

    def _use_fused(self, tc, edge_embedding, x, edge_attrs, edge_index, pairs=None) -> bool:
        """``use_fused_radial_tp``: True / False, or "auto" (default) = time the fused kernel against the unfused pair
        (grouped GEMM + TP kernel) ONCE per layer on the first real call and keep the faster one.  The fused kernel
        never materialises the [E, W] weights in the forward pass, but its path-parallel decomposition gives up the
        sharing of the x_i Y_j products between paths: which one wins depends on the signature (measurements in
        DESIGN.md section 4.7)."""
        mode = self.use_fused_radial_tp
        if mode is True or mode is False:
            return mode
        if self._fused_choice is None:
            if torch.cuda.is_current_stream_capturing():
                return False
            with torch.no_grad():
                def t(fn):
                    fn()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(2):
                        fn()
                    e1.record()
                    torch.cuda.synchronize()
                    return e0.elapsed_time(e1) / 2

                xd, yd, ed = x.detach(), edge_attrs.detach(), edge_embedding.detach()
                tf = t(lambda: tc["fused"](ed, xd, yd, edge_index[0], edge_index[1]))
                tu = t(lambda: self.tp_scatter(x=xd, edge_attr=yd, edge_weight=tc["mlp"](ed, pairs), edge_dst=edge_index[0],
                                               edge_src=edge_index[1]))
            self._fused_choice = bool(tf < tu)
            self.fused_timing_ms = {"fused": tf, "unfused": tu}
        return self._fused_choice

    def _note_fallback(self, reason: str):
        """The library (torch.matmul / cuBLAS) formulation is about to run instead of the wgmma blocks: say so
        once per block and reason, or raise when the model was built with ``strict_fast_path=True`` (bench.py,
        smoke(): a silent library fallback would be timed as if it were the product)."""
        if getattr(self, "strict_fast_path", False):
            raise RuntimeError(f"nequip_b200 InteractionBlock: tensor-core fast path unavailable ({reason}) and "
                               "strict_fast_path=True")
        seen = self.__dict__.setdefault("_fallback_seen", set())
        if reason not in seen:
            seen.add(reason)
            import warnings

            warnings.warn(f"nequip_b200 InteractionBlock: dense blocks run through torch.matmul (cuBLAS), not the "
                          f"wgmma kernels: {reason}", RuntimeWarning, stacklevel=3)

    def forward(self, x, node_attrs, edge_attrs, edge_embedding, edge_index, types=None, type_table=None,
                n_own: Optional[int] = None, halo=None, pairs=None, pair_grad: bool = True):
        """``n_own``/``halo``: sharded frames (owned atoms first, then ghosts).  As in the reference
        (interaction_block.py:159-199) the first layer sees the type embedding of owned + ghost atoms;
        later layers work on owned rows, refresh the ghosts through ``halo`` right before the
        TP+scatter and truncate to the owned rows right after it.  ``pairs``: the reverse-edge pair map of the
        edge list (``ops.edge_pairs``), with which the radial MLP computes one row per pair, and with ``pair_grad``
        also its backward (``RadialMLPGemm``)."""
        if n_own is not None and not self.is_first_layer:
            x = x[:n_own]
            node_attrs = node_attrs[:n_own]
            types = None if types is None else types[:n_own]
        tc = self._tensor_core_blocks(x, types, type_table)
        if tc is not None:
            # inference fast path: every dense block is one grouped 3xTF32 wgmma GEMM launch
            x_in = x
            # 1/sqrt(avg_num_neighbors): folded into the prepared weights (global) or a per-atom row scale (per type)
            x = tc["lin1"](x) if self.norm_shortcut else tc["lin1"](x, self.norm_const.view(-1)[types].view(1, -1).contiguous())
            if halo is not None and not self.is_first_layer:
                x = halo(x)
            if tc["fused"] is not None and self._use_fused(tc, edge_embedding, x, edge_attrs, edge_index, pairs):
                # one kernel: last radial layer (wgmma, weights resident in shared memory) -> TP -> scatter
                y = tc["fused"](edge_embedding, x, edge_attrs, edge_index[0], edge_index[1])
                if y is not None:
                    x = y
                    if n_own is not None:
                        x = x[:n_own]
                    x = tc["lin2"](x)
                    if tc["sc"] is not None:
                        x = tc["sc"](x_in, types, x)
                    return x
            if tc["mlp"] is not None:
                w = tc["mlp"](edge_embedding, pairs, pair_grad)
            else:
                self._note_fallback("radial MLP shape not supported by the grouped GEMM (needs at least one hidden "
                                    "layer, num_bessels and widths multiples of 4)")
                w = self._edge_weights(edge_embedding)
            x = self.tp_scatter(x=x, edge_attr=edge_attrs, edge_weight=w, edge_dst=edge_index[0], edge_src=edge_index[1])
            if n_own is not None:
                x = x[:n_own]
            x = tc["lin2"](x)
            if tc["sc"] is not None:
                x = tc["sc"](x_in, types, x)  # accumulates the self-connection onto linear_2's output
            return x
        sc = self.sc(x, node_attrs, types, type_table) if self.sc is not None else None
        x = self.linear_1(x)
        x = x * (self.norm_const.view(()) if self.norm_shortcut else self.norm_const[types])
        if halo is not None and not self.is_first_layer:
            x = halo(x)
        w = self._edge_weights(edge_embedding)
        x = self.tp_scatter(x=x, edge_attr=edge_attrs, edge_weight=w, edge_dst=edge_index[0], edge_src=edge_index[1])
        if n_own is not None:
            x = x[:n_own]
        x = self.linear_2(x)
        if sc is not None:
            x = x + sc
        return x

    def _tensor_core_blocks(self, x, types, type_table):
        """Lazily prepared tensor-core versions of linear_1 / radial MLP / linear_2 / self-connection
        (nequip_b200/nn/dense.py); None when not applicable (training, float64, mul_ir, odd multiplicities)."""
        from . import dense

        if not self.use_tensor_cores or not x.is_cuda:
            return None
        if x.dtype != torch.float32 or self.layout != "ir_mul":
            self._note_fallback(f"dtype {x.dtype} / layout {self.layout} (needs float32, ir_mul)")
            return None
        if any(p.requires_grad for p in self.parameters()) or (type_table is not None and type_table.requires_grad):
            self._note_fallback("parameters require grad (training); freeze them for the inference path")
            return None
        if (self.sc is not None or not self.norm_shortcut) and (types is None or type_table is None):
            self._note_fallback("self-connection / per-type normalisation need atom types + type table")
            return None
        key = tuple((p.data_ptr(), p._version) for p in self.parameters()) + (
            (type_table.data_ptr(), type_table._version) if type_table is not None else ())
        if self._tc_cache is not None and self._tc_cache[0] == key:
            if self._tc_cache[1] is None:
                self._note_fallback("a multiplicity is not a multiple of 4")
            return self._tc_cache[1]
        ok = dense.IrrepsLinearGemm.supported(self.linear_1) and dense.IrrepsLinearGemm.supported(self.linear_2)
        if self.sc is not None:
            ok = ok and dense.SelfConnectionGemm.supported(self.sc)
        if not ok:
            self._note_fallback("a multiplicity is not a multiple of 4")
            self._tc_cache = (key, None)
            return None
        dev = x.device
        lins = [m for m in self.edge_mlp.mlp if isinstance(m, ScalarLinearLayer)]
        mlp = fused = None
        if len(lins) >= 2 and dense.RadialMLPGemm.supported(lins[0], lins[-1], x.dtype, middle=lins[1:-1]):
            mlp = dense.RadialMLPGemm(lins[0], lins[-1], dev, middle=lins[1:-1])
            # the fused block shares the layer's mlp (its hidden layers and backward GEMMs)
            if dense.FusedRadialTP.supported(lins[0], lins[-1], self.tp_scatter._plan, x.dtype):
                fused = dense.FusedRadialTP(mlp, lins[-1], self.tp_scatter._plan, dev)
        blocks = dict(
            fused=fused,
            lin1=(dense.IrrepsLinearGemm(self.linear_1, dev, extra_scale=float(self.norm_const.view(-1)[0]))
                  if self.norm_shortcut else dense.IrrepsLinearGemm(self.linear_1, dev, row_scaled=True)),
            lin2=dense.IrrepsLinearGemm(self.linear_2, dev),
            sc=dense.SelfConnectionGemm(self.sc, type_table, dev) if self.sc is not None else None,
            mlp=mlp,
        )
        self._tc_cache = (key, blocks)
        return blocks


class ConvNetLayer(torch.nn.Module):
    """convnetlayer.py:26-170 (gate nonlinearity, no resnet)."""

    def __init__(self, prev: Irreps, edge_attr: Irreps, hidden: Irreps, **conv_kwargs):
        super().__init__()
        scalars, gates, gated, conv_out, layer_out = gate_irreps(prev, edge_attr, hidden)
        self.equivariant_nonlin = Gate(scalars, gates, gated, conv_kwargs.get("layout", "mul_ir"))
        self.conv = InteractionBlock(prev, edge_attr, conv_out, **conv_kwargs)
        self.irreps_out = layer_out

    def forward(self, x, node_attrs, edge_attrs, edge_embedding, edge_index, types=None, type_table=None,
                n_own=None, halo=None, pairs=None, pair_grad=True):
        x = self.conv(x, node_attrs, edge_attrs, edge_embedding, edge_index, types, type_table, n_own, halo, pairs,
                      pair_grad)
        return self.equivariant_nonlin(x)


# The named architectures of the NequIP foundation potentials: _NEQUIP_GNN_PRESETS (nequip_models.py:30-51) on top
# of _NEQUIP_GNN_STANDARD_PRESET (nequip_models.py:53-58), combined as PresetNequIPGNNModel does (:98-115).
NEQUIP_PRESETS: Dict[str, dict] = {
    "S": dict(num_layers=2, l_max=1, num_features=[128, 64]),
    "M": dict(num_layers=4, l_max=2, num_features=[128, 64, 32]),
    "L": dict(num_layers=6, l_max=3, num_features=[128, 64, 32, 32]),
    "XL": dict(num_layers=6, l_max=4, num_features=[320, 96, 64, 32, 32]),
}
NEQUIP_STANDARD_PRESET = dict(parity=False, type_embed_num_features=32, radial_mlp_depth=1, radial_mlp_width=128)


def parse_per_edge_type_cutoff(spec: dict, type_names: Sequence[str], r_max: float) -> torch.Tensor:
    """The reference's ``per_edge_type_cutoff`` (nn/embedding/utils.py:15-83) as a [T, T] float64 table
    ``rc[source, target]``: ``spec`` maps a source type name to one cutoff (every target) or to a dict {target type
    name: cutoff}; missing sources and targets get ``r_max``.  The table may be asymmetric.  Raises ``ValueError`` for
    unknown type names, cutoffs outside 0 < rc <= r_max and any other nesting."""
    names = list(type_names)
    if not isinstance(spec, dict):
        raise ValueError(f"per_edge_type_cutoff: expected a dict, got {type(spec).__name__}")

    def value(v, where):
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            raise ValueError(f"per_edge_type_cutoff[{where}]: expected a number, got {v!r}")
        v = float(v)
        if not 0.0 < v <= r_max:
            raise ValueError(f"per_edge_type_cutoff[{where}] = {v}: must satisfy 0 < rc <= r_max = {r_max}")
        return v

    table = torch.full((len(names), len(names)), float(r_max), dtype=torch.float64)
    for src, entry in spec.items():
        if src not in names:
            raise ValueError(f"per_edge_type_cutoff: unknown source type {src!r} (types: {names})")
        a = names.index(src)
        if isinstance(entry, dict):
            for tgt, v in entry.items():
                if tgt not in names:
                    raise ValueError(f"per_edge_type_cutoff[{src!r}]: unknown target type {tgt!r} (types: {names})")
                table[a, names.index(tgt)] = value(v, f"{src!r}][{tgt!r}")
        else:
            table[a, :] = value(entry, repr(src))
    return table


def preset_kwargs(name: str, **overrides) -> dict:
    """Constructor arguments of preset ``name`` (case-insensitive): standard preset < named preset < ``overrides``."""
    key = name.upper()
    if key not in NEQUIP_PRESETS:
        raise ValueError(f"unknown preset {name!r}: expected one of {sorted(NEQUIP_PRESETS)}")
    return {**NEQUIP_STANDARD_PRESET, **NEQUIP_PRESETS[key], **overrides}


class NequIPEnergyModel(torch.nn.Module):
    """``NequIPGNNModel`` (nequip_models.py:116-210) wrapped in the force part of
    ``ForceStressOutput`` (grad_output.py:215-232).  ``forward(data) -> data`` on an
    AtomicDataDict-shaped dict: needs ``pos`` [N,3] f64, ``edge_index`` [2,E] i64,
    ``atom_types`` [N] i64 and, for periodic systems, ``cell`` [3,3] + ``edge_cell_shift`` [E,3]."""

    def __init__(self, *, r_max: float, type_names: Sequence[str], num_layers: int = 4, l_max: int = 1,
                 parity: bool = True, num_features: Union[int, Sequence[int]] = 32,
                 type_embed_num_features: Optional[int] = None, radial_mlp_depth: int = 1,
                 radial_mlp_width: int = 128, num_bessels: int = 8, polynomial_cutoff_p: float = 6.0,
                 avg_num_neighbors: float = 1.0, per_type_energy_scales: Optional[Sequence[float]] = None,
                 per_type_energy_shifts: Optional[Sequence[float]] = None, model_dtype=torch.float32,
                 seed: int = 123, node_layout: str = "ir_mul", strict_fast_path: bool = False,
                 pair_potential: Optional[dict] = None, per_edge_type_cutoff: Optional[dict] = None):
        """``num_features``: one width for every degree, or a list of l_max + 1 widths (one per degree, e.g.
        ``[128, 64, 32]`` = 128x0e + 64x1o + 32x2e for l_max = 2 without parity), as in nequip_models.py:164-190.
        ``type_embed_num_features``: width of the type embedding, which is also the first layer's input and the
        self-connection's attribute width (nequip_models.py:171-174, 294); defaults to ``num_features[0]``.
        ``pair_potential``: the reference's config block of a pair potential (energy_modules.py:10-35), e.g.
        ``{"_target_": "nequip.nn.pair_potential.ZBL", "units": "metal", "chemical_species": ["C", "H", "O", "Cu"]}``
        (``_target_`` may be left out; optional ``polynomial_cutoff_p``, default 6, independent of the model's).  Its
        per-atom energies are added after the per-type scale and shift, before the sum (submodule ``pair_potential``).
        ``per_edge_type_cutoff``: the reference's partial table of cutoffs per ordered type pair (source = centre
        ``edge_index[0]``, target = neighbour), e.g. ``{"H": 2.0, "C": {"H": 4.0, "C": 3.5}}``; missing entries are
        ``r_max``, every entry satisfies 0 < rc <= r_max (``parse_per_edge_type_cutoff``).  The edge embedding and the
        ZBL envelope then take the normalised length ``r / rc[t_i, t_j]`` (the Bessel prefactor keeps ``r_max``), so an
        edge at or beyond its pair's cutoff contributes exactly zero; the full table is ``self.per_edge_type_cutoff``
        [T, T] f64, its reciprocal the buffer ``rmax_recip`` [T * T] f64 (the reference's ``edge_norm._rmax_recip``).
        Neighbour lists built with the table (``ops.neighbor_list(..., atom_types=, edge_type_cutoff=)``) drop those
        edges, and every per-edge cost shrinks with them.
        """
        super().__init__()
        pair_spec = parse_pair_potential(pair_potential, len(type_names))
        cutoff_table = (None if per_edge_type_cutoff is None
                        else parse_per_edge_type_cutoff(per_edge_type_cutoff, type_names, float(r_max)))
        widths = feature_widths(l_max, num_features)
        f_embed = int(type_embed_num_features) if type_embed_num_features is not None else widths[0]
        self.r_max, self.l_max, self.num_bessels, self.poly_p = float(r_max), l_max, num_bessels, float(polynomial_cutoff_p)
        self.model_dtype = model_dtype
        self.node_layout = node_layout  # internal layout of node features between the kernels
        self.config = dict(r_max=r_max, type_names=list(type_names), num_layers=num_layers, l_max=l_max, parity=parity,
                           num_features=num_features if isinstance(num_features, int) else widths,
                           type_embed_num_features=f_embed, radial_mlp_depth=radial_mlp_depth,
                           radial_mlp_width=radial_mlp_width, num_bessels=num_bessels,
                           polynomial_cutoff_p=polynomial_cutoff_p, avg_num_neighbors=avg_num_neighbors)
        prev_default = torch.get_default_dtype()
        torch.set_default_dtype(model_dtype)
        try:
            torch.manual_seed(seed)  # model_builder seeds before construction (model/utils.py:104-230)
            ntypes = len(type_names)
            if isinstance(avg_num_neighbors, dict):  # per type, keyed by type name (nequip/nn/norm.py:28-31)
                if set(avg_num_neighbors) != set(type_names):
                    raise ValueError("avg_num_neighbors: keys must be the type names")
                avg_num_neighbors = [float(avg_num_neighbors[k]) for k in type_names]
            elif not isinstance(avg_num_neighbors, (int, float)):
                avg_num_neighbors = [float(v) for v in avg_num_neighbors]
                if len(avg_num_neighbors) not in (1, ntypes):
                    raise ValueError(f"avg_num_neighbors: expected a scalar or {ntypes} values")
            self.config["avg_num_neighbors"] = avg_num_neighbors
            self.type_embed = torch.nn.Embedding(ntypes, f_embed)
            edge_attr = Irreps.spherical_harmonics(l_max)
            prev = Irreps([(f_embed, Irrep(0, 1))])
            hid = hidden_irreps(l_max, widths, parity)
            hiddens = [hid] * (num_layers - 1) + [Irreps([(widths[0], Irrep(0, 1))])]
            layers = []
            for li, h in enumerate(hiddens):
                layer = ConvNetLayer(prev, edge_attr, h, num_edge_embed=num_bessels, num_node_attrs=f_embed,
                                     radial_mlp_depth=radial_mlp_depth, radial_mlp_width=radial_mlp_width,
                                     use_sc=(li != 0), avg_num_neighbors=avg_num_neighbors,
                                     is_first_layer=(li == 0), layout=node_layout)
                layers.append(layer)
                prev = layer.irreps_out
            self.layers = torch.nn.ModuleList(layers)
            self.readout = ScalarMLPFunction(prev.dim, 1, hidden_layers_depth=0)
        finally:
            torch.set_default_dtype(prev_default)
        # PerTypeScaleShift (atomwise.py:236-284): a float or a one-element list applies to every type
        # (the reference's scales_shortcut / shifts_shortcut); otherwise one value per type
        def table(v, what):
            if v is None:
                return torch.empty(0, dtype=torch.float64)
            t = torch.as_tensor(v, dtype=torch.float64).reshape(-1)
            if t.numel() == 1:
                t = t.expand(ntypes).clone()
            if t.numel() != ntypes:
                raise ValueError(f"{what}: expected a scalar or {ntypes} values (one per type), got {t.numel()}")
            return t.reshape(-1, 1)

        self.register_buffer("scales", table(per_type_energy_scales, "per_type_energy_scales"))
        self.register_buffer("shifts", table(per_type_energy_shifts, "per_type_energy_shifts"))
        self.pair_potential = None
        if pair_spec is not None:
            self.pair_potential = ZBL(type_names, model_dtype=model_dtype, **pair_spec)
            self.config["pair_potential"] = dict(_target_=ZBL_TARGET, **pair_spec)
        self.per_edge_type_cutoff: Optional[torch.Tensor] = cutoff_table
        # the radial MLP's backward on the pair slots needs both edges of a pair to have the same embedding
        # derivative: an asymmetric table gives i -> j and j -> i different cutoffs, so it keeps the per-edge backward
        self._pair_grad = cutoff_table is None or bool(torch.equal(cutoff_table, cutoff_table.t()))
        if cutoff_table is not None:
            self.register_buffer("rmax_recip", cutoff_table.reciprocal().reshape(-1))
            self.config["per_edge_type_cutoff"] = {k: (dict(v) if isinstance(v, dict) else v)
                                                   for k, v in per_edge_type_cutoff.items()}
        self.set_strict_fast_path(strict_fast_path)

    @classmethod
    def from_preset(cls, name: str, **kwargs) -> "NequIPEnergyModel":
        """One of the reference's named architectures ``S``, ``M``, ``L``, ``XL`` (``NEQUIP_PRESETS``); ``kwargs``
        must include ``r_max`` and ``type_names`` and override any preset value."""
        return cls(**preset_kwargs(name, **kwargs))

    def set_strict_fast_path(self, on: bool = True):
        """Raise instead of warning when an interaction block cannot use the wgmma dense blocks."""
        for layer in self.layers:
            layer.conv.strict_fast_path = bool(on)
        return self

    def _edge_pairs(self, edge_index, shift, edge_embedding, num_nodes):
        """The reverse-edge pair map (``ops.edge_pairs``) that every layer's radial MLP shares, built on every call
        (the edge list changes between MD steps); None when the radial MLP cannot use it (it needs the [8, 128] ->
        [128, W] tensor-core MLP on float32)."""
        if not (self.num_bessels == 8 and self.config["radial_mlp_depth"] == 1 and self.config["radial_mlp_width"] == 128
                and edge_embedding.dtype == torch.float32 and self.node_layout == "ir_mul"):
            return None
        dst = edge_index[0]
        csr = ops.csr_cache.get(dst if dst.dtype == torch.int64 else dst.long().contiguous(), num_nodes)
        return ops.edge_pairs(edge_index, shift, edge_embedding, csr)

    def _edge_type_kwargs(self, types) -> dict:
        """Keyword arguments of the edge embedding for the per-edge-type cutoffs ({} without a table)."""
        if self.per_edge_type_cutoff is None:
            return {}
        return dict(types=types, edge_type_recip=self.rmax_recip)

    def _pair_kwargs(self) -> dict:
        return {} if self.per_edge_type_cutoff is None else dict(edge_type_recip=self.rmax_recip)

    @staticmethod
    def _frame_kwargs(data: Dict[str, torch.Tensor], cell) -> dict:
        """``batch=`` for the edge embedding and ZBL when a batch comes with one cell per frame ([F, 3, 3], F > 1);
        {} otherwise, so that a single frame and frames sharing one cell take the single-cell kernels."""
        batch = data.get(BATCH_KEY)
        if batch is None or cell is None or cell.dim() != 3 or cell.shape[0] == 1:
            return {}
        return dict(batch=batch)

    @staticmethod
    def _reduce_energy(e_atom: torch.Tensor, data: Dict[str, torch.Tensor]) -> torch.Tensor:
        """AtomwiseReduce (atomwise.py:92-113): per-graph sum -> [num_graphs, 1]; one frame without ``batch``."""
        batch = data.get(BATCH_KEY)
        if batch is None:
            return e_atom.sum(dim=0, keepdim=True)
        if NUM_NODES_KEY in data:
            ng = int(data[NUM_NODES_KEY].numel())
        elif BATCH_PTR_KEY in data:
            ng = int(data[BATCH_PTR_KEY].numel()) - 1
        else:
            ng = int(batch.max().item()) + 1 if batch.numel() else 0
        out = torch.zeros((ng, 1), dtype=e_atom.dtype, device=e_atom.device)
        return out.index_add_(0, batch.view(-1).long(), e_atom)

    # the energy part (SequentialGraphNetwork order of nequip_models.py:288-399)
    def energy(self, data: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        pos = data[POSITIONS_KEY]
        edge_index = data[EDGE_INDEX_KEY]
        types = data[ATOM_TYPE_KEY].view(-1)
        node_attrs = self.type_embed(types)
        x = node_attrs
        shift, cell = data.get(EDGE_CELL_SHIFT_KEY), data.get(CELL_KEY)
        if cell is None:
            shift = None
        pre = (2 * math.pi) / (self.r_max * self.r_max)
        sink = data.get("_edge_grad_sink")
        if EDGE_VECTORS_KEY in data:
            # the caller (LAMMPS ML-IAP) supplies the edge vectors: with_edge_vectors_ keeps them (nn/utils.py:68-118)
            # the types of an edge come from the real edge_index (the kernel's own index list names made-up positions)
            et = self._edge_type_kwargs(types)
            if et:
                et["edge_index"] = edge_index
            edge_attrs, edge_embedding = ops.edge_embed_from_vectors(
                data[EDGE_VECTORS_KEY], lmax=self.l_max, num_bessel=self.num_bessels, r_max=self.r_max,
                poly_p=self.poly_p, prefactor=pre, out_dtype=self.model_dtype, **et)
        else:
            _vec, edge_attrs, edge_embedding = ops.edge_embed(
                pos, edge_index, shift, cell, lmax=self.l_max, num_bessel=self.num_bessels, r_max=self.r_max,
                poly_p=self.poly_p, prefactor=pre, out_dtype=self.model_dtype, edge_grad_sink=sink,
                **self._edge_type_kwargs(types), **self._frame_kwargs(data, cell))
        pairs = self._edge_pairs(edge_index, None if EDGE_VECTORS_KEY in data else shift, edge_embedding, types.numel())
        # ML-IAP edge forces are dE/d(edge vector) per edge: moving a partner's gradient onto its representative
        # would change them, so that input keeps the per-edge radial-MLP backward
        pair_grad = self._pair_grad and EDGE_VECTORS_KEY not in data
        for layer in self.layers:
            x = layer(x, node_attrs, edge_attrs, edge_embedding, edge_index, types, self.type_embed.weight, pairs=pairs,
                      pair_grad=pair_grad)
        e_atom = self.readout(x).to(torch.float64)
        if self.scales.numel():
            e_atom = e_atom * self.scales[types]
        if self.shifts.numel():
            e_atom = e_atom + self.shifts[types]
        if self.pair_potential is not None:
            if EDGE_VECTORS_KEY in data:
                e_pair = self.pair_potential(types, edge_index, self.r_max, edge_vectors=data[EDGE_VECTORS_KEY],
                                             **self._pair_kwargs())
            else:
                e_pair = self.pair_potential(types, edge_index, self.r_max, pos=pos, shift=shift, cell=cell,
                                             edge_grad_sink=sink, **self._pair_kwargs(),
                                             **self._frame_kwargs(data, cell))
            e_atom = e_atom + e_pair
        data[PER_ATOM_ENERGY_KEY] = e_atom
        data[TOTAL_ENERGY_KEY] = self._reduce_energy(e_atom, data)
        return data

    def energy_owned(self, data: Dict[str, torch.Tensor], n_own: int, halo) -> torch.Tensor:
        """Per-atom energies [n_own, 1] f64 of the OWNED atoms of a sharded frame (``data`` holds owned
        atoms first, then ghosts; every edge's destination is owned) -- see nequip_b200/parallel.py."""
        pos, edge_index = data[POSITIONS_KEY], data[EDGE_INDEX_KEY]
        types = data[ATOM_TYPE_KEY].view(-1)
        node_attrs = self.type_embed(types)
        x = node_attrs
        shift, cell = data.get(EDGE_CELL_SHIFT_KEY), data.get(CELL_KEY)
        if cell is None:
            shift = None
        _vec, edge_attrs, edge_embedding = ops.edge_embed(
            pos, edge_index, shift, cell, lmax=self.l_max, num_bessel=self.num_bessels, r_max=self.r_max,
            poly_p=self.poly_p, prefactor=(2 * math.pi) / (self.r_max * self.r_max), out_dtype=self.model_dtype,
            **self._edge_type_kwargs(types))
        pairs = self._edge_pairs(edge_index, shift, edge_embedding, types.numel())
        for layer in self.layers:
            x = layer(x, node_attrs, edge_attrs, edge_embedding, edge_index, types, self.type_embed.weight, n_own, halo,
                      pairs, self._pair_grad)
        e_atom = self.readout(x).to(torch.float64)
        t_own = types[:n_own]
        if self.scales.numel():
            e_atom = e_atom * self.scales[t_own]
        if self.shifts.numel():
            e_atom = e_atom + self.shifts[t_own]
        if self.pair_potential is not None:
            # every edge's centre is owned: the owned rows are complete, the ghost rows (no edges) are 0
            e_atom = e_atom + self.pair_potential(types, edge_index, self.r_max, pos=pos, shift=shift, cell=cell,
                                                  **self._pair_kwargs())[:n_own]
        return e_atom

    @staticmethod
    def _frame_stress(vec: torch.Tensor, g_edge: torch.Tensor, data: Dict[str, torch.Tensor]):
        """(stress, virial) [F, 3, 3] of a batch: dE/d(eps_f) = sym(sum over the edges e whose centre is in frame f of
        r_e (x) g_e), divided by |det cell_f| (one cell serves every frame).  F is the row count of the energy."""
        F = data[TOTAL_ENERGY_KEY].shape[0]
        cell = data[CELL_KEY].double().reshape(-1, 3, 3)
        if cell.shape[0] not in (1, F):
            raise ValueError(f"compute_stress: {cell.shape[0]} cells for {F} frames")
        frame_e = data[BATCH_KEY].view(-1).long()[data[EDGE_INDEX_KEY][0].long()]
        rg = (vec.unsqueeze(2) * g_edge.unsqueeze(1)).reshape(-1, 9)
        v = torch.zeros((F, 9), dtype=torch.float64, device=vec.device).index_add_(0, frame_e, rg).view(F, 3, 3)
        v = 0.5 * (v + v.transpose(1, 2))
        vol = torch.linalg.det(cell).abs().view(-1, 1, 1)
        return v / vol, torch.neg(v)

    def forward(self, data: Dict[str, torch.Tensor], compute_forces: bool = True,
                compute_stress: bool = False) -> Dict[str, torch.Tensor]:
        """``ForceStressOutput.forward`` (nequip/nn/grad_output.py:107-298):

        * positions given: ``forces = -dE/dpos``; with ``compute_stress`` (needs ``cell``) also
          ``stress = (1/|det cell|) dE/d(eps)`` and ``virial = -dE/d(eps)`` ([1,3,3]) for the symmetric strain
          ``eps`` applied to positions and cell.  With ``batch`` (a batch of frames, ``cell`` [F,3,3] or one cell for
          all) each frame has its own strain: ``stress`` and ``virial`` are [F,3,3], frame f sums the edges whose
          centre is in f and divides by its own ``|det cell_f|`` (grad_output.py:117-260).  The cell/strain gradient is not taken through a displaced
          copy of the inputs: every edge vector transforms as ``r -> r (1 + eps)``, so
          ``dE/d(eps) = sym( sum_e r_e (x) dE/dr_e )`` and the per-edge gradients are a by-product of the
          edge-embedding backward kernel;
        * ``edge_vectors`` given (LAMMPS ML-IAP): ``edge_forces = dE/d(edge_vectors)``, no sign flip (:270-296).
        """
        data = dict(data)
        if not compute_forces:
            return self.energy(data)
        if EDGE_VECTORS_KEY in data:
            with torch.enable_grad():
                vec = data[EDGE_VECTORS_KEY].detach().double().requires_grad_(True)
                data[EDGE_VECTORS_KEY] = vec
                data = self.energy(data)
                (g,) = torch.autograd.grad([data[TOTAL_ENERGY_KEY].sum()], [vec])
            data[EDGE_FORCE_KEY] = g
            data[EDGE_VECTORS_KEY] = vec.detach()
            data[TOTAL_ENERGY_KEY] = data[TOTAL_ENERGY_KEY].detach()
            data[PER_ATOM_ENERGY_KEY] = data[PER_ATOM_ENERGY_KEY].detach()
            return data
        if compute_stress and data.get(CELL_KEY) is None:
            raise ValueError("compute_stress needs a cell")
        pos = data[POSITIONS_KEY]
        sink = {} if compute_stress else None
        with torch.enable_grad():
            pos = pos.detach().requires_grad_(True)
            data[POSITIONS_KEY] = pos
            if sink is not None:
                data["_edge_grad_sink"] = sink
            data = self.energy(data)
            (g,) = torch.autograd.grad([data[TOTAL_ENERGY_KEY].sum()], [pos])
        data.pop("_edge_grad_sink", None)
        data[FORCE_KEY] = torch.neg(g)
        if sink is not None:
            g_edge = sink["edge_vector_grad"]
            if "pair_edge_vector_grad" in sink:  # the pair potential's share of dE/d(edge vector)
                g_edge = g_edge + sink["pair_edge_vector_grad"]
            if data.get(BATCH_KEY) is None:
                v = torch.einsum("ea,eb->ab", sink["edge_vectors"], g_edge)
                v = 0.5 * (v + v.t())
                vol = torch.linalg.det(data[CELL_KEY].double().view(3, 3)).abs()
                data[STRESS_KEY] = (v / vol).view(1, 3, 3)
                data[VIRIAL_KEY] = torch.neg(v).view(1, 3, 3)
            else:
                data[STRESS_KEY], data[VIRIAL_KEY] = self._frame_stress(sink["edge_vectors"], g_edge, data)
        data[POSITIONS_KEY] = pos.detach()
        data[TOTAL_ENERGY_KEY] = data[TOTAL_ENERGY_KEY].detach()
        data[PER_ATOM_ENERGY_KEY] = data[PER_ATOM_ENERGY_KEY].detach()
        return data
