"""Dense blocks of the interaction layer on the tensor cores (inference: frozen weights, float32,
channel-contiguous ``ir_mul`` node layout).

Each block is ONE launch of the grouped 3xTF32 GEMM (``nequip_b200/csrc/nqb_gemm.cu``) per
direction; the weights are prepared (scaled, split hi/lo, tiled) once.  Reference ops:

* ``RadialMLPGemm``      ScalarMLPFunction, depth >= 1 (one launch per layer, SiLU in the GEMM epilogue)
                         nequip/nn/mlp.py:80-195, 262-268
* ``IrrepsLinearGemm``   e3nn o3.Linear (linear_1, linear_2)   nequip/nn/interaction_block.py:82-87,129-138
* ``SelfConnectionGemm`` e3nn FullyConnectedTensorProduct(x, node_attrs) with node_attrs =
                         type_embed[atom_types]                nequip/nn/interaction_block.py:140-146,175

In ir_mul every (chunk pair, irrep component) is a strided GEMM over the atoms:
``out[:, oo + i*mo : oo + (i+1)*mo] (+)= x[:, io + i*mi : io + (i+1)*mi] @ W``.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from .. import ops
from ..irreps import Irreps


def _aligned(*vals) -> bool:
    return all(v % 4 == 0 for v in vals)


# ---------------------------------------------------------------------------------------
class _GemmLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, fwd: ops.GroupedGemm, bwd: ops.GroupedGemm, d_out: int, zero_out: bool, d_in: int, zero_in: bool,
                rowscale, out_init):
        M = x.shape[0]
        if out_init is not None:
            out = out_init  # accumulate into an existing tensor (self-connection added onto linear_2's output)
        else:
            out = (torch.zeros if zero_out else torch.empty)((M, d_out), dtype=x.dtype, device=x.device)
        fwd.run(x, out, M, rowscale)
        ctx.bwd, ctx.d_in, ctx.zero_in, ctx.rowscale = bwd, d_in, zero_in, rowscale
        ctx.has_init = out_init is not None
        if out_init is not None:
            ctx.mark_dirty(out_init)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        gout = gout.contiguous()
        M = gout.shape[0]
        gx = (torch.zeros if ctx.zero_in else torch.empty)((M, ctx.d_in), dtype=gout.dtype, device=gout.device)
        ctx.bwd.run(gout, gx, M, ctx.rowscale)
        return gx, None, None, None, None, None, None, None, (gout if ctx.has_init else None)


class IrrepsLinearGemm:
    """``o3.Linear`` in ir_mul layout from a ``nequip_b200.nn.model.Linear`` module's weights."""

    def __init__(self, lin, device, extra_scale: float = 1.0, row_scaled: bool = False):
        """``row_scaled``: every problem multiplies its output rows by row 0 of the ``rowscale`` matrix given at call
        time (the per-atom-type AvgNumNeighborsNorm factor, nequip/nn/norm.py:48-68)."""
        fin, fout = lin.irreps_in, lin.irreps_out
        rs = 0 if row_scaled else -1
        self.row_scaled = row_scaled
        in_off, out_off = fin.offsets(), fout.offsets()
        self.d_in, self.d_out = fin.dim, fout.dim
        fwd: List[ops.GemmProblem] = []
        bwd: List[ops.GemmProblem] = []
        # problems of one launch run concurrently: a target written by more than one problem is
        # zero-initialised and every writer adds with red.global.add; single writers store plainly
        n_out = {o: sum(1 for (_, o2, _, _) in lin.instr if o2 == o) for o in range(len(fout))}
        n_in = {i: sum(1 for (i2, _, _, _) in lin.instr if i2 == i) for i in range(len(fin))}
        for (i, o, off, pw) in lin.instr:
            mi, ir = fin[i]
            mo = fout[o][0]
            W = lin.weight.detach()[off: off + mi * mo].view(mi, mo)
            for c in range(ir.dim):
                a_off, c_off = in_off[i] + c * mi, out_off[o] + c * mo
                fwd.append(ops.GemmProblem(a_off, self.d_in, c_off, self.d_out, W, scale=pw * extra_scale,
                                           atomic=n_out[o] > 1, rs_off=rs))
                bwd.append(ops.GemmProblem(c_off, self.d_out, a_off, self.d_in, W, scale=pw * extra_scale, transposed=True,
                                           atomic=n_in[i] > 1, rs_off=rs))
        self.zero_out = any(n != 1 for n in n_out.values())
        self.zero_in = any(n != 1 for n in n_in.values())
        self.fwd = ops.GroupedGemm(fwd, device)
        self.bwd = ops.GroupedGemm(bwd, device)

    @staticmethod
    def supported(lin) -> bool:
        muls = [m for m, _ in lin.irreps_in] + [m for m, _ in lin.irreps_out]
        return lin.layout == "ir_mul" and all(m % 4 == 0 for m in muls) and lin.weight.dtype == torch.float32

    def __call__(self, x, rowscale=None):
        if self.row_scaled != (rowscale is not None):
            raise ValueError("IrrepsLinearGemm: rowscale must be given exactly when built with row_scaled=True")
        return _GemmLinearFn.apply(x.contiguous(), self.fwd, self.bwd, self.d_out, self.zero_out, self.d_in, self.zero_in,
                                   rowscale, None)


class SelfConnectionGemm:
    """FCTP(x, type_embed[types]) as per-type effective-weight GEMMs with a one-hot row scale; the result
    is ACCUMULATED onto ``base`` (the linear_2 output), i.e. ``x = linear_2(x) + sc`` in one pass."""

    def __init__(self, sc, type_table: torch.Tensor, device):
        fin, fout = sc.irreps_in, sc.irreps_out
        in_off, out_off = fin.offsets(), fout.offsets()
        self.d_in, self.d_out = fin.dim, fout.dim
        self.T = type_table.shape[0]
        fwd: List[ops.GemmProblem] = []
        bwd: List[ops.GemmProblem] = []
        tt = type_table.detach()
        for (i, o, off, pw) in sc.instr:
            mi, ir = fin[i]
            mo = fout[o][0]
            W = sc.weight.detach()[off: off + mi * sc.num_attr * mo].view(mi, sc.num_attr, mo)
            weff = torch.einsum("uvw,tv->tuw", W, tt)  # [T, mi, mo]
            for t in range(self.T):
                for c in range(ir.dim):
                    a_off, c_off = in_off[i] + c * mi, out_off[o] + c * mo
                    # row scale = row t of one-hot^T [T, M]
                    # forward: each atom row belongs to exactly one type -> the T problems of one (pair,
                    # component) write disjoint rows; read-modify-write onto linear_2's output is race free
                    # as long as only ONE in-chunk feeds an out chunk, otherwise add atomically
                    multi_o = sum(1 for (_, o2, _, _) in sc.instr if o2 == o) > 1
                    fwd.append(ops.GemmProblem(a_off, self.d_in, c_off, self.d_out, weff[t].contiguous(), scale=pw,
                                               accumulate=not multi_o, atomic=multi_o, rs_off=t, skip_zero_rows=True))
                    multi_i = sum(1 for (i2, _, _, _) in sc.instr if i2 == i) > 1
                    bwd.append(ops.GemmProblem(c_off, self.d_out, a_off, self.d_in, weff[t].contiguous(), scale=pw,
                                               transposed=True, accumulate=not multi_i, atomic=multi_i, rs_off=t,
                                               skip_zero_rows=True))
        self.zero_in = True  # backward accumulates (row-masked) into a zero-initialised gradient
        self.fwd = ops.GroupedGemm(fwd, device)
        self.bwd = ops.GroupedGemm(bwd, device)

    @staticmethod
    def supported(sc) -> bool:
        muls = [m for m, _ in sc.irreps_in] + [m for m, _ in sc.irreps_out]
        return sc.layout == "ir_mul" and all(m % 4 == 0 for m in muls) and sc.weight.dtype == torch.float32

    def __call__(self, x, types, base):
        onehot_t = torch.nn.functional.one_hot(types, self.T).to(x.dtype).t().contiguous()  # [T, M]
        return _GemmLinearFn.apply(x.contiguous(), self.fwd, self.bwd, self.d_out, False, self.d_in, self.zero_in,
                                   onehot_t, base)


# ---------------------------------------------------------------------------------------
class _RadialMLPGemmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, emb, mlp: "RadialMLPGemm", need_bwd: bool, pairs, pair_grad: bool):
        E = emb.shape[0]
        out = torch.empty((E, mlp.W), dtype=emb.dtype, device=emb.device)
        pre = [] if need_bwd else None
        shared = pairs is not None and mlp.shares_pairs
        if shared:
            # one row of h and of the GEMM per slot of the pair map, stored to both edges of the slot
            h = torch.empty((E, mlp.w1s.shape[1]), dtype=emb.dtype, device=emb.device)  # rows < count are used
            ops.mlp_hidden_fwd_rows(emb, mlp.w1s, pairs, h)
            mlp.fwd.run_pairs(h, out, pairs)
        else:
            mlp.fwd.run(mlp.hidden(emb, pre), out, E)
        ctx.mlp = mlp
        ctx.pairs = pairs if shared and pair_grad else None
        if need_bwd:
            ctx.save_for_backward(emb, *pre)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gw):
        emb, *pre = ctx.saved_tensors
        return ctx.mlp.grad_emb(emb, gw, pre, ctx.pairs), None, None, None, None


class RadialMLPGemm:
    """ScalarMLPFunction of any depth >= 1 (no bias, SiLU between layers) on the project's kernels.

    ``first`` [num_bessels, H], ``middle`` [H, H] each, ``last`` [H, W] (``ScalarLinearLayer`` modules).
    Forward: the first layer runs on ``k_hidden_fwd`` when it is [8, 128], otherwise as a ``k_gemm3x`` problem with
    the SiLU epilogue (K = num_bessels); every middle layer is one such problem; the last layer is a plain problem.
    With a backward pass ahead, each hidden layer on ``k_gemm3x`` also stores its pre-activation ([E, H] float32).
    Given the reverse-edge pair map (``ops.edge_pairs``), an [8, 128] -> [128, W] MLP computes one row per slot
    (``k_hidden_fwd`` on the slots' representative edges, then the paired ``k_gemm3x`` that stores each result row to
    both edges of its slot), and by default its backward on the slots too (``grad_emb`` with ``pairs``); deeper MLPs
    keep the per-edge forward and backward.
    Backward: the transposed GEMM of each layer multiplies by silu' of the saved pre-activation of the layer below;
    into an [8, 128] first layer it gives grad_h for ``k_hidden_bwd`` (pre-activation recomputed), and a generic
    first layer ends with a plain transposed GEMM into grad_emb [E, num_bessels]."""

    def __init__(self, first, last, device, middle=()):
        self.w1s = (first.weight.detach() * first.alpha).contiguous()
        self.W = last.weight.shape[1]
        plan = self.plan(first, last, middle)
        self._hidden_kernel = plan["hidden_kernel"]

        def gemm(p):
            return ops.GroupedGemm([p], device)

        self.fwd = gemm(plan["fwd"])
        # the last layer's plain transposed GEMM, grad_h = gw @ (W_last a)^T
        self.bwd = gemm(plan["bwd"])
        self._hidden = [(gemm(save), gemm(plain), save.B.shape[1]) for save, plain in plan["hidden"]]
        self._chain = [(self.bwd if p is plan["bwd"] else gemm(p), width, pre) for p, width, pre in plan["chain"]]
        # the forward can share rows between the two edges of a pair slot (no per-edge pre-activation is kept)
        self.shares_pairs = self._hidden_kernel and not self._hidden

    @staticmethod
    def uses_hidden_kernel(first) -> bool:
        """The CUDA-core hidden-layer kernels are built for [E, 8] x [8, 128] only."""
        return tuple(first.weight.shape) == (8, 128)

    @classmethod
    def plan(cls, first, last, middle=()):
        """The grouped-GEMM problems of the forward and backward pass (needs no device):

        * ``hidden``: per hidden layer on ``k_gemm3x``, in order, its ("silu_save", "silu") problems;
        * ``fwd`` / ``bwd``: the last layer's problem and its plain transposed problem;
        * ``chain``: the backward launches in order, (problem, output width, index into the saved pre-activations
          of the ``hidden`` layers or None);
        * ``hidden_kernel``: the first layer runs on ``k_hidden_fwd`` / ``k_hidden_bwd``."""

        def prob(lin, act="none", transposed=False):
            k, n = lin.weight.shape
            lda, ldc = (n, k) if transposed else (k, n)
            return ops.GemmProblem(0, lda, 0, ldc, lin.weight.detach(), scale=float(lin.alpha), transposed=transposed,
                                   act=act)

        layers = [first, *middle, last]
        kernel = cls.uses_hidden_kernel(first)
        skip = 1 if kernel else 0  # hidden layers before the first one on k_gemm3x
        bwd = prob(last, transposed=True)
        chain = []
        for i in range(len(layers) - 1, 0, -1):  # layer i's transposed GEMM, then silu' of hidden layer i - 1
            pre = i - 1 - skip
            if pre >= 0:
                p = prob(layers[i], "silu_grad", True)
            else:  # into k_hidden_bwd: plain grad_h
                p = bwd if i == len(layers) - 1 else prob(layers[i], transposed=True)
            chain.append((p, layers[i].weight.shape[0], pre if pre >= 0 else None))
        if not kernel:
            chain.append((prob(first, transposed=True), first.weight.shape[0], None))
        return dict(hidden_kernel=kernel, hidden=[(prob(l, "silu_save"), prob(l, "silu")) for l in layers[skip:-1]],
                    fwd=prob(last), bwd=bwd, chain=chain)

    @staticmethod
    def supported(first, last, dtype, middle=()) -> bool:
        """float32, and num_bessels and every width a multiple of 4 (the grouped GEMM's K, N and strides)."""
        dims = [first.weight.shape[0]] + [l.weight.shape[1] for l in (first, *middle, last)]
        return dtype == torch.float32 and all(d % 4 == 0 for d in dims)

    def hidden(self, emb, pre: Optional[list] = None):
        """The last hidden activation ``silu(... silu(emb @ w1s) ...)``.  ``pre``: a list that receives the
        pre-activation of every hidden layer on ``k_gemm3x`` (what ``grad_emb`` needs); None keeps none."""
        E = emb.shape[0]
        x = emb
        if self._hidden_kernel:
            x = torch.empty((E, self.w1s.shape[1]), dtype=emb.dtype, device=emb.device)
            ops.mlp_hidden_fwd(emb, self.w1s, x)
        for save, plain, width in self._hidden:
            h = torch.empty((E, width), dtype=emb.dtype, device=emb.device)
            if pre is None:
                plain.run(x, h, E)
            else:
                p = torch.empty((E, width), dtype=emb.dtype, device=emb.device)
                save.run(x, h, E, aux=p)
                pre.append(p)
            x = h
        return x

    def grad_emb(self, emb, gw, pre=(), pairs: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        """Gradient of ``emb`` from the gradient ``gw`` of the edge weights, with ``pre`` the pre-activations that
        ``hidden`` saved.

        ``pairs`` (MLPs with ``shares_pairs`` only): the backward of the pair-shared forward.  Both edges of a slot got
        the slot's output, so the slot's grad_h is ``(gw[rep] + gw[partner]) @ (W a)^T`` (the sum is formed inside the
        GEMM), ``k_hidden_bwd`` writes the representative's ``grad_emb`` row from it and zeros to the partner's row.
        The two edges have bitwise-equal embedding rows, so in exact arithmetic this moves the partner's embedding
        gradient onto the representative; it leaves forces and ``sym(sum_e r_e (x) dE/dr_e)`` unchanged where the
        embedding's derivative is the same for both edges (a function of |r| with one cutoff for the pair), not the
        per-edge ``dE/d(edge vector)``."""
        E = emb.shape[0]
        g = gw.contiguous()
        if pairs is not None:
            if not self.shares_pairs:
                raise ValueError("RadialMLPGemm.grad_emb: pairs given, but this MLP does not share rows between pairs")
            gh = torch.empty((E, self.w1s.shape[1]), dtype=g.dtype, device=g.device)  # rows < count are used
            self.bwd.run_pair_sum(g, gh, pairs)
            gemb = torch.empty_like(emb)
            ops.mlp_hidden_bwd_rows(emb, self.w1s, gh, pairs, gemb)
            return gemb
        for gemm, width, k in self._chain:
            out = torch.empty((E, width), dtype=g.dtype, device=g.device)
            gemm.run(g, out, E, aux=None if k is None else pre[k])
            g = out
        if self._hidden_kernel:
            gemb = torch.empty_like(emb)
            ops.mlp_hidden_bwd(emb, self.w1s, g, gemb)
            return gemb
        return g

    def __call__(self, emb, pairs: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, pair_grad: bool = True):
        """``pairs``: ``ops.edge_pairs`` of the edge list whose embedding ``emb`` is (the per-edge forward without).
        ``pair_grad``: with a pair-shared forward, also run the backward on the slots (``grad_emb``); False keeps the
        per-edge backward, for callers that need each edge's own ``dE/d(emb)`` (per-edge outputs such as ML-IAP edge
        forces, or an embedding whose derivative differs between the two edges of a pair)."""
        return _RadialMLPGemmFn.apply(emb.contiguous(), self, torch.is_grad_enabled() and emb.requires_grad, pairs,
                                      pair_grad)


# ---------------------------------------------------------------------------------------
class _FusedRadialTPFn(torch.autograd.Function):
    """``out = scatter(TP(x[src], y, silu(emb @ W1 a1) @ W2 a2))`` with the last radial layer fused into the
    tensor-product kernel (forward: the [E, W] weights are produced in registers and consumed in place;
    they are written once on the side only when a backward pass will need them)."""

    @staticmethod
    def forward(ctx, emb, x, y, edge_src, mod: "FusedRadialTP", csr, need_emb_grad: bool):
        pre = [] if need_emb_grad else None
        h = mod.mlp.hidden(emb, pre)
        need_bwd = any(ctx.needs_input_grad[:3])
        out, w = ops.tp_fused_fwd(mod.fw, x, y, h, edge_src, csr, want_w=need_bwd)
        ctx.mod, ctx.csr = mod, csr
        if need_bwd:
            ctx.save_for_backward(emb, x, y, w, edge_src, *(pre or ()))
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        emb, x, y, w, edge_src, *pre = ctx.saved_tensors
        mod = ctx.mod
        gx, gy, gw = ops.tp_scatter_bwd_raw(mod.plan, x, y, w, edge_src, ctx.csr, gout, need_x=ctx.needs_input_grad[1])
        gemb = mod.mlp.grad_emb(emb, gw, pre) if ctx.needs_input_grad[0] else None
        return gemb, gx, (gy if ctx.needs_input_grad[2] else None), None, None, None, None


class FusedRadialTP:
    """Radial MLP (any depth; the last layer fused) + TensorProductScatter of one interaction layer as a single
    forward kernel (``nqb_tp_fused_fwd``) after the hidden layers; backward = ``nqb_tp_scatter_bwd`` + the layer's
    ``RadialMLPGemm.grad_emb``."""

    def __init__(self, mlp: RadialMLPGemm, lin2, plan: ops.TPPlan, device):
        """``mlp``: the layer's unfused radial MLP (built from the same weights), whose hidden layer and backward GEMM
        this kernel shares."""
        self.plan = plan
        self.mlp = mlp
        self.fw = ops.FusedTPWeights(plan, lin2.weight.detach(), float(lin2.alpha), device)

    @staticmethod
    def supported(lin1, lin2, plan: ops.TPPlan, dtype) -> bool:
        hid, W = lin2.weight.shape
        if dtype != torch.float32 or hid > 128 or hid % 8 or W != plan.weight_numel or W % 4:
            return False
        return int(ops._capi.lib().nqb_tp_fused_slices(plan.handle)) > 0

    def __call__(self, emb, x, y, edge_dst, edge_src):
        csr = ops.csr_cache.get(edge_dst.long().contiguous() if edge_dst.dtype != torch.int64 else edge_dst, x.shape[0])
        if csr.perm is not None:
            return None  # unsorted neighbour list: the caller uses the unfused kernels (which take the permutation)
        return _FusedRadialTPFn.apply(emb.contiguous(), x.contiguous(), y.contiguous(), edge_src.long().contiguous(), self, csr,
                                      torch.is_grad_enabled() and emb.requires_grad)
