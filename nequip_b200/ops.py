"""Torch-facing operators over the C ABI (device memory, streams and autograd glue only).

``tp_scatter``  -- the fused tensor product + scatter that replaces
                   ``TensorProductScatter.forward`` (nequip/nn/_tp_scatter_base.py:35-38)
                   and its autograd (first order: what forces need,
                   nequip/nn/grad_output.py:217-221 with ``create_graph=False``).
``spherical_harmonics`` / ``edge_embed`` -- the edge-embedding kernels replacing
                   nequip/nn/embedding/_edge.py:65-80,136-150,193-198 + nequip/nn/utils.py:68-118.

There is no CPU or eager fallback: CPU tensors raise, a missing/unbuildable kernel
library raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from . import _capi, build
from .codegen import GenOptions, TPSignature
from .irreps import Irreps

_DT = {torch.float32: 0, torch.float64: 1}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _require_cuda(*ts: torch.Tensor):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError(
                "nequip_b200 kernels run on CUDA (sm_90a) only; got a CPU tensor and there is no CPU fallback"
            )


# ---------------------------------------------------------------------------------------
# plans
# ---------------------------------------------------------------------------------------
class TPPlan:
    """Immutable binding of one TensorProductScatter signature to its kernel library."""

    def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions, opts: Optional[GenOptions] = None):
        self.sig = TPSignature(Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out), list(instructions))
        self.opts = opts or GenOptions()
        self.spec_path = build.ensure_spec(self.sig, self.opts)
        L = _capi.lib()

        def arr(irr):
            a = (_capi.NqbIrrep * len(irr))()
            for i, (mul, ir) in enumerate(irr):
                a[i].mul, a[i].l, a[i].p = mul, ir.l, ir.p
            return a

        in1, in2, out = arr(self.sig.irreps_in1), arr(self.sig.irreps_in2), arr(self.sig.irreps_out)
        ins = (_capi.NqbInstruction * len(self.sig.instructions))()
        for i, (a, b, c) in enumerate(self.sig.instructions):
            ins[i].i_in1, ins[i].i_in2, ins[i].i_out = a, b, c
        h = C.c_void_p()
        _capi.check(
            L.nqb_plan_create(in1, len(in1), in2, len(in2), out, len(out), ins, len(ins),
                              self.spec_path.encode(), C.byref(h)),
            "nqb_plan_create",
        )
        self._h = h
        self.d_in, self.s_dim = self.sig.d_in, self.sig.s_dim
        self.weight_numel, self.d_out = self.sig.weight_numel, self.sig.d_out

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _capi.lib().nqb_plan_destroy(self._h)
                self._h = None
        except Exception:
            pass


_plans: Dict[str, TPPlan] = {}
_plans_lock = threading.Lock()


def get_plan(irreps_in1, irreps_in2, irreps_out, instructions, opts: Optional[GenOptions] = None) -> TPPlan:
    opts = opts or GenOptions()
    sig = TPSignature(Irreps(irreps_in1), Irreps(irreps_in2), Irreps(irreps_out), list(instructions))
    key = sig.canonical() + "|" + opts.tag()
    with _plans_lock:
        p = _plans.get(key)
        if p is None:
            p = TPPlan(irreps_in1, irreps_in2, irreps_out, instructions, opts)
            _plans[key] = p
        return p


# ---------------------------------------------------------------------------------------
# destination CSR
# ---------------------------------------------------------------------------------------
@dataclass
class EdgeCSR:
    row_ptr: torch.Tensor  # [N+1] int64
    perm: Optional[torch.Tensor]  # [E] int64 (slot -> edge id) or None when edges are already grouped
    num_nodes: int
    num_edges: int


def build_csr(edge_dst: torch.Tensor, num_nodes: int, assume_sorted: Optional[bool] = None) -> EdgeCSR:
    """CSR over edges grouped by destination.  ``assume_sorted=None`` checks on the
    device (one host sync); the reference's neighbour lists are grouped by centre atom
    (nequip/data/transforms/neighborlist.py:120-157) so the common case needs no sort."""
    _require_cuda(edge_dst)
    if edge_dst.dtype != torch.int64:
        edge_dst = edge_dst.long()
    edge_dst = edge_dst.contiguous()
    E = edge_dst.numel()
    L = _capi.lib()
    st = _stream()
    is_sorted = assume_sorted
    deferred = getattr(_sorted_tls, "flags", None)
    if deferred is None and _capture_flags and torch.cuda.is_current_stream_capturing():
        # the backward of a captured step runs in autograd's device thread, which has no thread-local context:
        # use the innermost deferred_sorted_check that is open in some thread
        deferred = _capture_flags[-1]
    if is_sorted is None and deferred is not None:
        # CUDA-graph capture (nequip_b200/graph.py): no host sync allowed -- run the check kernel, keep its
        # flag for the caller to verify after the replay, and build the CSR as if sorted
        flag = torch.empty(1, dtype=torch.int32, device=edge_dst.device)
        _capi.check(L.nqb_csr_check_sorted(_ptr(edge_dst), E, _ptr(flag), st), "nqb_csr_check_sorted")
        deferred.append(flag)
        is_sorted = True
    if is_sorted is None:
        flag = torch.empty(1, dtype=torch.int32, device=edge_dst.device)
        _capi.check(L.nqb_csr_check_sorted(_ptr(edge_dst), E, _ptr(flag), st), "nqb_csr_check_sorted")
        is_sorted = bool(flag.item())
    perm = None
    keys = edge_dst
    if not is_sorted:
        keys, perm = torch.sort(edge_dst, stable=True)
        perm = perm.contiguous()
        keys = keys.contiguous()
    row_ptr = torch.empty(num_nodes + 1, dtype=torch.int64, device=edge_dst.device)
    _capi.check(L.nqb_csr_from_sorted(_ptr(keys), E, num_nodes, _ptr(row_ptr), st), "nqb_csr_from_sorted")
    return EdgeCSR(row_ptr, perm, num_nodes, E)


_sorted_tls = threading.local()
_capture_flags: List[List[torch.Tensor]] = []  # flag lists of the open deferred_sorted_check contexts, any thread


class deferred_sorted_check:
    """Context manager: inside it ``build_csr`` does not synchronise to learn whether the edge list is grouped
    by destination; it records the device flags (1 = sorted) in ``self.flags`` and assumes sorted."""

    def __enter__(self):
        self.flags: List[torch.Tensor] = []
        self._prev = getattr(_sorted_tls, "flags", None)
        _sorted_tls.flags = self.flags
        _capture_flags.append(self.flags)
        return self

    def __exit__(self, *exc):
        _sorted_tls.flags = self._prev
        for k in range(len(_capture_flags) - 1, -1, -1):
            if _capture_flags[k] is self.flags:
                del _capture_flags[k]
                break
        return False


class _CSRCache:
    """Per-thread one-entry cache: all layers of one forward share the same edge_index."""

    def __init__(self):
        self._tls = threading.local()

    def get(self, edge_dst: torch.Tensor, num_nodes: int) -> EdgeCSR:
        key = (edge_dst.data_ptr(), edge_dst.numel(), edge_dst._version, num_nodes, edge_dst.device)
        ent = getattr(self._tls, "ent", None)
        if ent is not None and ent[0] == key:
            return ent[1]
        csr = build_csr(edge_dst, num_nodes)
        # hold a reference to edge_dst so the data_ptr cannot be recycled while cached
        self._tls.ent = (key, csr, edge_dst)
        return csr

    def clear(self):
        self._tls.ent = None


csr_cache = _CSRCache()


# ---------------------------------------------------------------------------------------
# fused TP + scatter
# ---------------------------------------------------------------------------------------
class _TPScatterFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, edge_attr, edge_weight, edge_src, plan: TPPlan, csr: EdgeCSR):
        L = _capi.lib()
        N, E = x.shape[0], edge_src.numel()
        out = torch.empty((N, plan.d_out), dtype=x.dtype, device=x.device)
        if N > 0:
            _capi.check(
                L.nqb_tp_scatter_fwd(plan.handle, _DT[x.dtype], _ptr(x), _ptr(edge_attr), _ptr(edge_weight),
                                     _ptr(csr.row_ptr), _ptr(csr.perm), _ptr(edge_src), N, E, _ptr(out), _stream()),
                "nqb_tp_scatter_fwd",
            )
        ctx.plan, ctx.csr = plan, csr
        ctx.save_for_backward(x, edge_attr, edge_weight, edge_src)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        x, y, w, edge_src = ctx.saved_tensors
        gx, gy, gw = tp_scatter_bwd_raw(ctx.plan, x, y, w, edge_src, ctx.csr, gout, need_x=ctx.needs_input_grad[0])
        return gx, (gy if ctx.needs_input_grad[1] else None), (gw if ctx.needs_input_grad[2] else None), None, None, None


def tp_scatter(plan: TPPlan, x, edge_attr, edge_weight, edge_dst, edge_src, csr: Optional[EdgeCSR] = None):
    """``out[n] = sum_{e: dst[e]=n} TP_uvu(x[src[e]], edge_attr[e], edge_weight[e])`` -> ``[x.size(0), D_mid]``."""
    _require_cuda(x, edge_attr, edge_weight, edge_dst, edge_src)
    if x.dtype not in _DT:
        raise TypeError(f"nequip_b200.tp_scatter: unsupported dtype {x.dtype}")
    dt = x.dtype
    if x.dim() != 2 or x.shape[1] != plan.d_in:
        raise ValueError(f"x must be [N, {plan.d_in}], got {tuple(x.shape)}")
    E = edge_src.numel()
    if tuple(edge_attr.shape) != (E, plan.s_dim) or tuple(edge_weight.shape) != (E, plan.weight_numel):
        raise ValueError(
            f"edge_attr/edge_weight must be [{E}, {plan.s_dim}] / [{E}, {plan.weight_numel}], got "
            f"{tuple(edge_attr.shape)} / {tuple(edge_weight.shape)}"
        )
    if edge_dst.numel() != E:
        raise ValueError("edge_dst and edge_src differ in length")
    x = x.contiguous()
    y = edge_attr.to(dt).contiguous()
    w = edge_weight.to(dt).contiguous()
    src = edge_src.long().contiguous()
    if csr is None:
        csr = csr_cache.get(edge_dst.long().contiguous() if edge_dst.dtype != torch.int64 else edge_dst, x.shape[0])
    elif csr.num_nodes != x.shape[0] or csr.num_edges != E:
        raise ValueError("EdgeCSR does not match x / edge_index")
    return _TPScatterFn.apply(x, y, w, src, plan, csr)


# ---------------------------------------------------------------------------------------
# fused last radial-MLP layer + TP + scatter (forward) -- nqb_tp_fused_fwd
# ---------------------------------------------------------------------------------------
class FusedTPWeights:
    """Second-layer radial-MLP weights ``W2 [K, W]`` (times ``alpha2``) permuted into the slice order of the
    signature's fused kernel, split into tf32 hi/lo parts and laid out in the order the kernel's shared memory holds
    them (once per model), plus the split of the grid (one CTA per SM) over the slices in proportion to their cost."""

    def __init__(self, plan: TPPlan, W2: torch.Tensor, alpha2: float, device):
        from .codegen import TPGenerator

        L = _capi.lib()
        self.plan = plan
        lay = TPGenerator(plan.sig, plan.opts).fused_layout()
        nslice = int(L.nqb_tp_fused_slices(plan.handle))
        if lay is None or nslice == 0 or nslice != len(lay["slices"]):
            raise RuntimeError("FusedTPWeights: this signature has no fused kernel")
        K, W = int(W2.shape[0]), int(W2.shape[1])
        if W != plan.weight_numel or K > 128 or K % 8:
            raise ValueError(f"FusedTPWeights: W2 must be [K <= 128 (multiple of 8), {plan.weight_numel}], got {tuple(W2.shape)}")
        self.K, self.nslice = K, nslice
        cols = torch.tensor(lay["cols"], dtype=torch.long, device=device)
        W2d = W2.detach().to(device=device, dtype=torch.float32)
        Wp = torch.zeros((K, cols.numel()), dtype=torch.float32, device=device)
        ok = cols >= 0
        Wp[:, ok] = W2d[:, cols[ok]]
        self.prepared = self.prepare(Wp * float(alpha2), nslice)
        G = torch.cuda.get_device_properties(device).multi_processor_count
        self.cta0, self.nctas = self.split_grid(lay["cost"], G)
        self.cta0_dev = torch.tensor(self.cta0, dtype=torch.int32, device=device)

    @staticmethod
    def prepare(Wp: torch.Tensor, nslice: int) -> torch.Tensor:
        """[K, 128 * nslice] -> per slice: hi and lo of W^T [128 rows, 128 k] (K zero padded), each in the canonical
        K-major core-matrix order of the wgmma A operand: element (r, k) at (r // 8) * 1024 + (k // 4) * 32 +
        (r % 8) * 4 + k % 4.  hi = round-to-nearest tf32 (ties away from zero), lo = the exact remainder."""
        K = Wp.shape[0]
        wt = torch.zeros((nslice, 128, 128), dtype=torch.float32, device=Wp.device)
        wt[:, :, :K] = Wp.t().reshape(nslice, 128, K)
        bits = wt.view(torch.int32)
        hi = ((bits + 0x1000) & -0x2000).view(torch.float32)
        lo = wt - hi
        both = torch.stack([hi, lo], 1)  # [slice, part, r, k]
        both = both.reshape(nslice, 2, 16, 8, 32, 4).permute(0, 1, 2, 4, 3, 5)  # [.., r // 8, k // 4, r % 8, k % 4]
        return both.contiguous().reshape(-1)

    @staticmethod
    def split_grid(cost, G: int):
        """CTAs per slice proportional to cost (every slice gets at least one); returns (prefix, total)."""
        S = len(cost)
        n = [1] * S
        for _ in range(max(0, G - S)):
            i = max(range(S), key=lambda j: cost[j] / n[j])
            n[i] += 1
        pre = [0]
        for v in n:
            pre.append(pre[-1] + v)
        return pre, pre[-1]


def tp_fused_fwd(fw: FusedTPWeights, x: torch.Tensor, y: torch.Tensor, h: torch.Tensor, edge_src: torch.Tensor,
                 csr: EdgeCSR, want_w: bool):
    """``out [N, D_mid]`` (and the per-edge weights ``w [E, W]`` when ``want_w``) of the fused kernel."""
    _require_cuda(x, y, h, edge_src)
    plan = fw.plan
    if csr.perm is not None:
        raise RuntimeError("tp_fused_fwd: edges must be grouped by destination (no permutation)")
    if x.dtype != torch.float32 or y.dtype != torch.float32 or h.dtype != torch.float32:
        raise TypeError("tp_fused_fwd: float32 only")
    N, E = x.shape[0], edge_src.numel()
    if x.shape[1] != plan.d_in or tuple(y.shape) != (E, plan.s_dim) or h.shape[0] != E or h.shape[1] != fw.K:
        raise ValueError("tp_fused_fwd: shape mismatch")
    x, y, h = x.contiguous(), y.contiguous(), h.contiguous()
    out = torch.empty((N, plan.d_out), dtype=torch.float32, device=x.device)
    w = torch.empty((E, plan.weight_numel), dtype=torch.float32, device=x.device) if want_w else None
    _capi.check(
        _capi.lib().nqb_tp_fused_fwd(plan.handle, _ptr(x), _ptr(y), _ptr(h), h.stride(0), fw.K, _ptr(fw.prepared),
                                     _ptr(csr.row_ptr), _ptr(edge_src), N, E, _ptr(out), _ptr(w), _ptr(fw.cta0_dev),
                                     int(fw.nctas), _stream()),
        "nqb_tp_fused_fwd",
    )
    return out, w


_DETERMINISTIC = os.environ.get("NQB_DETERMINISTIC", "0") not in ("", "0")


def set_deterministic(on: bool = True) -> None:
    """Bitwise-repeatable backward of the fused TP+scatter (also implied by ``torch.use_deterministic_algorithms``):
    grad_x goes through a per-edge buffer and a source-sorted segmented sum, grad_Y through one slice per writer,
    instead of ``red.global.add`` in arrival order (the default, like the reference's OpenEquivariance back-end)."""
    global _DETERMINISTIC
    _DETERMINISTIC = bool(on)


def deterministic() -> bool:
    return _DETERMINISTIC or torch.are_deterministic_algorithms_enabled()


class _SrcCSRCache:
    """Source-sorted view of the edge list (the reference's edge_transpose_perm): one entry per thread."""

    def __init__(self):
        self._tls = threading.local()

    def get(self, edge_src: torch.Tensor, num_nodes: int):
        key = (edge_src.data_ptr(), edge_src.numel(), edge_src._version, num_nodes, edge_src.device)
        ent = getattr(self._tls, "ent", None)
        if ent is not None and ent[0] == key:
            return ent[1], ent[2]
        keys, perm = torch.sort(edge_src, stable=True)
        seg = torch.empty(num_nodes + 1, dtype=torch.int64, device=edge_src.device)
        _capi.check(_capi.lib().nqb_csr_from_sorted(_ptr(keys.contiguous()), edge_src.numel(), num_nodes, _ptr(seg), _stream()),
                    "nqb_csr_from_sorted")
        self._tls.ent = (key, perm.contiguous(), seg, edge_src)
        return self._tls.ent[1], seg

    def clear(self):
        self._tls.ent = None


src_csr_cache = _SrcCSRCache()


def tp_scatter_bwd_raw(plan: TPPlan, x, y, w, edge_src, csr: EdgeCSR, gout, need_x: bool = True,
                       force_deterministic: Optional[bool] = None):
    """Backward kernels of the fused TP+scatter on raw tensors: (grad_x or None, grad_y, grad_w)."""
    L = _capi.lib()
    N, E = x.shape[0], edge_src.numel()
    det = deterministic() if force_deterministic is None else bool(force_deterministic)
    gw = torch.empty_like(w)
    if N == 0 or E == 0:
        gw.zero_()
        return (torch.zeros_like(x) if need_x else None), torch.zeros_like(y), gw
    gout = gout.contiguous()
    dt = _DT[x.dtype]
    if not det:
        gx = torch.zeros_like(x) if need_x else None
        gy = torch.zeros_like(y)
        _capi.check(L.nqb_tp_scatter_bwd(plan.handle, dt, _ptr(x), _ptr(y), _ptr(w), _ptr(csr.row_ptr), _ptr(csr.perm),
                                         _ptr(edge_src), _ptr(gout), N, E, _ptr(gx), _ptr(gy), _ptr(gw), 0, _stream()),
                    "nqb_tp_scatter_bwd")
        return gx, gy, gw
    ns = int(L.nqb_tp_scatter_gy_slices(plan.handle, dt))
    if ns <= 0:
        raise RuntimeError("nequip_b200: this kernel library has no deterministic backward")
    gxe = torch.empty((E, x.shape[1]), dtype=x.dtype, device=x.device) if need_x else None
    gys = torch.zeros((ns, E, y.shape[1]), dtype=y.dtype, device=y.device)
    _capi.check(L.nqb_tp_scatter_bwd(plan.handle, dt, _ptr(x), _ptr(y), _ptr(w), _ptr(csr.row_ptr), _ptr(csr.perm),
                                     _ptr(edge_src), _ptr(gout), N, E, _ptr(gxe), _ptr(gys), _ptr(gw), 1, _stream()),
                "nqb_tp_scatter_bwd")
    gx = None
    if need_x:
        perm_t, seg_t = src_csr_cache.get(edge_src, N)
        gx = torch.empty_like(x)
        _capi.check(L.nqb_segment_sum(dt, _ptr(gxe), x.shape[1], _ptr(perm_t), _ptr(seg_t), N, _ptr(gx), _stream()),
                    "nqb_segment_sum")
    gy = gys[0]
    for q in range(1, ns):  # fixed order
        gy = gy + gys[q]
    return gx, gy, gw


# ---------------------------------------------------------------------------------------
# spherical harmonics / edge embedding
# ---------------------------------------------------------------------------------------
class _SHFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, vec, lmax: int, out_dtype):
        L = _capi.lib()
        E = vec.shape[0]
        y = torch.empty((E, (lmax + 1) ** 2), dtype=out_dtype, device=vec.device)
        _capi.check(L.nqb_sh_fwd(lmax, _ptr(vec), E, _DT[out_dtype], _ptr(y), _stream()), "nqb_sh_fwd")
        ctx.lmax, ctx.out_dtype = lmax, out_dtype
        ctx.save_for_backward(vec)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy):
        (vec,) = ctx.saved_tensors
        L = _capi.lib()
        E = vec.shape[0]
        gvec = torch.empty_like(vec)
        gy = gy.to(ctx.out_dtype).contiguous()
        _capi.check(L.nqb_sh_bwd(ctx.lmax, _ptr(vec), E, _DT[ctx.out_dtype], _ptr(gy), _ptr(gvec), _stream()),
                    "nqb_sh_bwd")
        return gvec, None, None


def spherical_harmonics(vec: torch.Tensor, lmax: int, out_dtype=torch.float32) -> torch.Tensor:
    """``o3.SphericalHarmonics(lmax, normalize=True, "component")`` of ``[E,3]`` float64 edge vectors."""
    _require_cuda(vec)
    if vec.dim() != 2 or vec.shape[1] != 3:
        raise ValueError("vec must be [E, 3]")
    return _SHFn.apply(vec.double().contiguous(), int(lmax), out_dtype)


class _EdgeEmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pos, edge_index, shift, cell, lmax, num_bessel, r_max, poly_p, prefactor, out_dtype, sink=None,
                types=None, recip=None, frame=None):
        L = _capi.lib()
        N, E = pos.shape[0], edge_index.shape[1]
        dev = pos.device
        vec = torch.empty((E, 3), dtype=torch.float64, device=dev)
        y = torch.empty((E, (lmax + 1) ** 2), dtype=out_dtype, device=dev)
        emb = torch.empty((E, num_bessel), dtype=out_dtype, device=dev)
        if frame is not None:
            _capi.check(
                L.nqb_edge_embed_fwd_frames(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(pos), _ptr(edge_index),
                                            _ptr(shift), _ptr(cell), _ptr(frame), N, E, _ptr(types),
                                            0 if recip is None else _ptr(edge_index), _ptr(recip),
                                            0 if recip is None else _edge_type_count(recip), _DT[out_dtype], _ptr(vec),
                                            _ptr(y), _ptr(emb), _stream()),
                "nqb_edge_embed_fwd_frames",
            )
        elif recip is None:
            _capi.check(
                L.nqb_edge_embed_fwd(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(pos), _ptr(edge_index), _ptr(shift),
                                     _ptr(cell), N, E, _DT[out_dtype], _ptr(vec), _ptr(y), _ptr(emb), _stream()),
                "nqb_edge_embed_fwd",
            )
        else:
            _capi.check(
                L.nqb_edge_embed_fwd_typed(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(pos), _ptr(edge_index),
                                           _ptr(shift), _ptr(cell), N, E, _ptr(types), _ptr(edge_index), _ptr(recip),
                                           _edge_type_count(recip), _DT[out_dtype], _ptr(vec), _ptr(y), _ptr(emb),
                                           _stream()),
                "nqb_edge_embed_fwd_typed",
            )
        ctx.args = (lmax, num_bessel, r_max, poly_p, prefactor, out_dtype, N)
        ctx.sink = sink
        ctx.save_for_backward(vec, edge_index, types, recip)
        ctx.mark_non_differentiable(vec)
        return vec, y, emb

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, _gvec, gy, gemb):
        vec, edge_index, types, recip = ctx.saved_tensors
        lmax, num_bessel, r_max, poly_p, prefactor, out_dtype, N = ctx.args
        L = _capi.lib()
        E = vec.shape[0]
        gpos = torch.zeros((N, 3), dtype=torch.float64, device=vec.device)
        gy = None if gy is None else gy.to(out_dtype).contiguous()
        gemb = None if gemb is None else gemb.to(out_dtype).contiguous()
        # the per-edge gradient dE/d(edge vector) is what the virial is made of (sum_e r_e (x) g_e): keep it
        # when the caller asked for it
        gvec = torch.empty_like(vec) if ctx.sink is not None else None
        if recip is None:
            _capi.check(
                L.nqb_edge_embed_bwd(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(vec), _ptr(edge_index), N, E,
                                     _DT[out_dtype], _ptr(gy), _ptr(gemb), _ptr(gpos), _ptr(gvec), _stream()),
                "nqb_edge_embed_bwd",
            )
        else:
            _capi.check(
                L.nqb_edge_embed_bwd_typed(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(vec), _ptr(edge_index), N, E,
                                           _ptr(types), _ptr(edge_index), _ptr(recip), _edge_type_count(recip),
                                           _DT[out_dtype], _ptr(gy), _ptr(gemb), _ptr(gpos), _ptr(gvec), _stream()),
                "nqb_edge_embed_bwd_typed",
            )
        if ctx.sink is not None:
            ctx.sink["edge_vectors"], ctx.sink["edge_vector_grad"] = vec, gvec
        return gpos, None, None, None, None, None, None, None, None, None, None, None, None, None


class _EdgeEmbedVecFn(torch.autograd.Function):
    """Harmonics + radial embedding of GIVEN edge vectors (the ML-IAP branch: LAMMPS hands over the vectors,
    nequip/nn/grad_output.py:270-296); backward = dE/d(edge vectors)."""

    @staticmethod
    def forward(ctx, vec, lmax, num_bessel, r_max, poly_p, prefactor, out_dtype, types=None, type_index=None,
                recip=None):
        L = _capi.lib()
        E = vec.shape[0]
        dev = vec.device
        # the fused kernel computes pos[src] - pos[dst]: atoms 0..E-1 are the vectors, atom E is the origin
        pos = torch.cat([vec, torch.zeros((1, 3), dtype=torch.float64, device=dev)], 0)
        ar = torch.arange(E, dtype=torch.int64, device=dev)
        edge_index = torch.stack([torch.full_like(ar, E), ar]).contiguous()
        vec_out = torch.empty((E, 3), dtype=torch.float64, device=dev)
        y = torch.empty((E, (lmax + 1) ** 2), dtype=out_dtype, device=dev)
        emb = torch.empty((E, num_bessel), dtype=out_dtype, device=dev)
        if recip is None:
            _capi.check(
                L.nqb_edge_embed_fwd(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(pos), _ptr(edge_index), 0, 0, E + 1,
                                     E, _DT[out_dtype], _ptr(vec_out), _ptr(y), _ptr(emb), _stream()),
                "nqb_edge_embed_fwd",
            )
        else:
            # the types come from the real edge list, not from the made-up positions' index list
            _capi.check(
                L.nqb_edge_embed_fwd_typed(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(pos), _ptr(edge_index), 0, 0,
                                           E + 1, E, _ptr(types), _ptr(type_index), _ptr(recip), _edge_type_count(recip),
                                           _DT[out_dtype], _ptr(vec_out), _ptr(y), _ptr(emb), _stream()),
                "nqb_edge_embed_fwd_typed",
            )
        ctx.args = (lmax, num_bessel, r_max, poly_p, prefactor, out_dtype)
        ctx.save_for_backward(vec_out, edge_index, types, type_index, recip)
        return y, emb

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gy, gemb):
        vec, edge_index, types, type_index, recip = ctx.saved_tensors
        lmax, num_bessel, r_max, poly_p, prefactor, out_dtype = ctx.args
        E = vec.shape[0]
        gvec = torch.empty_like(vec)
        gy = None if gy is None else gy.to(out_dtype).contiguous()
        gemb = None if gemb is None else gemb.to(out_dtype).contiguous()
        if recip is None:
            _capi.check(
                _capi.lib().nqb_edge_embed_bwd(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(vec), _ptr(edge_index),
                                               E + 1, E, _DT[out_dtype], _ptr(gy), _ptr(gemb), 0, _ptr(gvec), _stream()),
                "nqb_edge_embed_bwd",
            )
        else:
            _capi.check(
                _capi.lib().nqb_edge_embed_bwd_typed(lmax, num_bessel, r_max, poly_p, prefactor, _ptr(vec),
                                                     _ptr(edge_index), E + 1, E, _ptr(types), _ptr(type_index),
                                                     _ptr(recip), _edge_type_count(recip), _DT[out_dtype], _ptr(gy),
                                                     _ptr(gemb), 0, _ptr(gvec), _stream()),
                "nqb_edge_embed_bwd_typed",
            )
        return gvec, None, None, None, None, None, None, None, None, None


def _edge_type_count(recip: torch.Tensor) -> int:
    """T of a [T * T] reciprocal-cutoff table."""
    T = int(round(recip.numel() ** 0.5))
    if T < 1 or T * T != recip.numel():
        raise ValueError(f"edge_type_recip must hold T * T values, got {recip.numel()}")
    return T


def _edge_type_args(types, edge_type_recip, what: str):
    """(types, recip) checked and laid out for the ``_typed`` kernels, or (None, None) without a table."""
    if (types is None) != (edge_type_recip is None):
        raise ValueError(f"{what}: types and edge_type_recip must be given together")
    if edge_type_recip is None:
        return None, None
    _require_cuda(types, edge_type_recip)
    recip = edge_type_recip.to(torch.float64).reshape(-1).contiguous()
    _edge_type_count(recip)
    return types.view(-1).long().contiguous(), recip


def edge_embed_from_vectors(vec, *, lmax: int, num_bessel: int = 8, r_max: float, poly_p: float = 6.0,
                            prefactor: float = 1.0, out_dtype=torch.float32, types=None, edge_index=None,
                            edge_type_recip=None):
    """``(edge_attrs [E,(lmax+1)^2], edge_embedding [E,num_bessel])`` of given ``[E,3]`` edge vectors,
    differentiable w.r.t. the vectors.

    Per-edge-type cutoffs: ``edge_type_recip`` [T * T] f64 holds ``1 / rc[source, target]`` and the normalised length
    of edge e is ``|vec_e| * edge_type_recip[T * types[edge_index[0, e]] + types[edge_index[1, e]]]``; ``types`` [N]
    and the edge list ``edge_index`` [2, E] the vectors belong to must come with it."""
    _require_cuda(vec)
    types, recip = _edge_type_args(types, edge_type_recip, "edge_embed_from_vectors")
    if recip is not None:
        if edge_index is None or tuple(edge_index.shape) != (2, vec.shape[0]):
            raise ValueError(f"edge_embed_from_vectors: edge_type_recip needs edge_index [2, {vec.shape[0]}]")
        _require_cuda(edge_index)
        edge_index = edge_index.long().contiguous()
    return _EdgeEmbedVecFn.apply(vec.double().contiguous(), int(lmax), int(num_bessel), float(r_max), float(poly_p),
                                 float(prefactor), out_dtype, types, None if recip is None else edge_index, recip)


def _frame_cells(cell, batch, num_atoms: int, what: str):
    """(cells [F, 3, 3] f64, frame [N] i64) of a batch of frames for the ``_frames`` kernels; ``ValueError`` for a
    malformed ``batch`` or a frame index outside [0, F) (one host synchronisation, skipped while the stream is
    capturing a CUDA graph)."""
    _require_cuda(cell, batch)
    if cell.dim() != 3 or tuple(cell.shape[1:]) != (3, 3):
        raise ValueError(f"{what}: cell must be [F, 3, 3] with batch, got {tuple(cell.shape)}")
    frame = batch.view(-1).long().contiguous()
    if frame.numel() != num_atoms:
        raise ValueError(f"{what}: batch must hold {num_atoms} frame indices, got {frame.numel()}")
    if num_atoms and not torch.cuda.is_current_stream_capturing():
        # a captured step (graph.GraphedMDStep) takes its batch from a NeighborListPlan that checked it when it was
        # made, and a read-back cannot be captured
        lo, hi = (int(v) for v in torch.aminmax(frame))
        if lo < 0 or hi >= cell.shape[0]:
            raise ValueError(f"{what}: batch holds frame indices outside [0, {cell.shape[0]})")
    return cell.double().contiguous(), frame


def _framed(cell, batch) -> bool:
    """Whether a call takes the ``_frames`` kernels: a batch with more than one cell.  One cell ([3, 3] or [1, 3, 3])
    serves every edge as it does without a batch."""
    return batch is not None and cell is not None and cell.dim() == 3 and cell.shape[0] > 1


def edge_embed(pos, edge_index, shift=None, cell=None, *, lmax: int, num_bessel: int = 8, r_max: float,
               poly_p: float = 6.0, prefactor: float = 1.0, out_dtype=torch.float32, edge_grad_sink=None,
               types=None, edge_type_recip=None, batch=None):
    """Edge vectors, harmonics and Bessel x cutoff embedding in one kernel.

    Returns ``(edge_vectors [E,3] f64, edge_attrs [E,(lmax+1)^2], edge_embedding [E,num_bessel])``.
    Differentiable w.r.t. ``pos`` (forces).  ``edge_grad_sink`` (a dict): the backward pass also stores the
    edge vectors and dE/d(edge vector) in it, from which the virial / cell gradient follows.
    ``types`` [N] + ``edge_type_recip`` [T * T] f64: per-edge-type cutoffs, the normalised length of edge e is
    ``r_e * edge_type_recip[T * types[edge_index[0, e]] + types[edge_index[1, e]]]`` instead of ``r_e / r_max``
    (``prefactor`` is the caller's).
    A batch of frames: ``cell`` [F, 3, 3] with ``batch`` [N] (the frame of each atom); edge e takes the cell of frame
    ``batch[edge_index[0, e]]`` (nequip/nn/utils.py:96-106) and its outputs are bitwise those of a call on its frame
    alone.  A single cell with or without ``batch`` takes the single-cell kernels."""
    _require_cuda(pos, edge_index)
    pos = pos.double().contiguous()
    edge_index = edge_index.long().contiguous()
    if (shift is None) != (cell is None):
        raise ValueError("shift and cell must be given together")
    frame = None
    if shift is not None:
        shift = shift.double().contiguous()
        if _framed(cell, batch):
            cell, frame = _frame_cells(cell, batch, pos.shape[0], "edge_embed")
        else:
            cell = cell.double().reshape(3, 3).contiguous()
    types, recip = _edge_type_args(types, edge_type_recip, "edge_embed")
    if frame is not None:
        return _EdgeEmbedFn.apply(pos, edge_index, shift, cell, int(lmax), int(num_bessel), float(r_max),
                                  float(poly_p), float(prefactor), out_dtype, edge_grad_sink, types, recip, frame)
    if recip is None:
        return _EdgeEmbedFn.apply(pos, edge_index, shift, cell, int(lmax), int(num_bessel), float(r_max),
                                  float(poly_p), float(prefactor), out_dtype, edge_grad_sink)
    return _EdgeEmbedFn.apply(pos, edge_index, shift, cell, int(lmax), int(num_bessel), float(r_max),
                              float(poly_p), float(prefactor), out_dtype, edge_grad_sink, types, recip)


# ---------------------------------------------------------------------------------------
# ZBL pair energy -- nqb_zbl_fwd / nqb_zbl_bwd
# ---------------------------------------------------------------------------------------
class _ZBLFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, geom, edge_index, shift, cell, types, table, r_max, poly_p, cutoff_f32, from_vectors, sink,
                recip=None, frame=None):
        N, E, T = types.numel(), edge_index.shape[1], table.shape[0]
        csr = csr_cache.get(edge_index[0], N)  # the CSR the first interaction layer already built
        pos, vec = (None, geom) if from_vectors else (geom, None)
        e_atom = torch.empty((N, 1), dtype=torch.float64, device=types.device)
        if frame is not None:
            _capi.check(
                _capi.lib().nqb_zbl_fwd_frames(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(frame),
                                               _ptr(types), _ptr(table), T, _ptr(csr.row_ptr), _ptr(csr.perm), N, E,
                                               r_max, poly_p, int(cutoff_f32), _ptr(recip), _ptr(e_atom), _stream()),
                "nqb_zbl_fwd_frames",
            )
        elif recip is None:
            _capi.check(
                _capi.lib().nqb_zbl_fwd(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(vec), _ptr(types),
                                        _ptr(table), T, _ptr(csr.row_ptr), _ptr(csr.perm), N, E, r_max, poly_p,
                                        int(cutoff_f32), _ptr(e_atom), _stream()),
                "nqb_zbl_fwd",
            )
        else:
            _capi.check(
                _capi.lib().nqb_zbl_fwd_typed(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(vec),
                                              _ptr(types), _ptr(table), T, _ptr(csr.row_ptr), _ptr(csr.perm), N, E,
                                              r_max, poly_p, int(cutoff_f32), _ptr(recip), _ptr(e_atom), _stream()),
                "nqb_zbl_fwd_typed",
            )
        ctx.args = (r_max, poly_p, cutoff_f32, from_vectors)
        ctx.sink = sink
        ctx.save_for_backward(geom, edge_index, shift, cell, types, table, recip, frame)
        return e_atom

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, ge):
        geom, edge_index, shift, cell, types, table, recip, frame = ctx.saved_tensors
        r_max, poly_p, cutoff_f32, from_vectors = ctx.args
        N, E = types.numel(), edge_index.shape[1]
        pos, vec = (None, geom) if from_vectors else (geom, None)
        gpos = None if from_vectors else torch.zeros_like(geom)
        gvec = torch.empty((E, 3), dtype=torch.float64, device=geom.device) \
            if from_vectors or ctx.sink is not None else None
        ge = ge.to(torch.float64).contiguous()
        if frame is not None:
            _capi.check(
                _capi.lib().nqb_zbl_bwd_frames(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(frame),
                                               _ptr(types), _ptr(table), table.shape[0], N, E, r_max, poly_p,
                                               int(cutoff_f32), _ptr(recip), _ptr(ge), _ptr(gpos), _ptr(gvec),
                                               _stream()),
                "nqb_zbl_bwd_frames",
            )
        elif recip is None:
            _capi.check(
                _capi.lib().nqb_zbl_bwd(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(vec), _ptr(types),
                                        _ptr(table), table.shape[0], N, E, r_max, poly_p, int(cutoff_f32), _ptr(ge),
                                        _ptr(gpos), _ptr(gvec), _stream()),
                "nqb_zbl_bwd",
            )
        else:
            _capi.check(
                _capi.lib().nqb_zbl_bwd_typed(_ptr(pos), _ptr(edge_index), _ptr(shift), _ptr(cell), _ptr(vec),
                                              _ptr(types), _ptr(table), table.shape[0], N, E, r_max, poly_p,
                                              int(cutoff_f32), _ptr(recip), _ptr(ge), _ptr(gpos), _ptr(gvec), _stream()),
                "nqb_zbl_bwd_typed",
            )
        if ctx.sink is not None:
            # kept apart from the edge embedding's gradient: the stress assembly adds the two once both backwards ran
            ctx.sink["pair_edge_vector_grad"] = gvec
        return (gvec if from_vectors else gpos), None, None, None, None, None, None, None, None, None, None, None, None


def zbl_energy(pos, edge_index, types, table, *, shift=None, cell=None, edge_vectors=None, r_max: float,
               poly_p: float = 6.0, cutoff_dtype=torch.float64, edge_grad_sink=None, edge_type_recip=None, batch=None):
    """ZBL per-atom energies ``[N, 1]`` f64 (``N = types.numel()``), summed onto the centre ``edge_index[0]``.

    ``table`` [T, T, 2] f64 holds ``0.5 * qqr2e * Z_i Z_j`` and ``Z_i^0.23 + Z_j^0.23`` per ordered type pair
    (``nn.pair.ZBL.table``).  The geometry comes from ``pos`` (+ ``shift``/``cell``) or, with ``pos=None``, from the
    given ``edge_vectors`` [E, 3] (the ML-IAP branch); the result is differentiable w.r.t. whichever was given.
    ``cutoff_dtype=torch.float32`` rounds the cutoff as a float32 model does.  ``edge_grad_sink`` (a dict): the backward
    pass also stores dE/d(edge vector) in it under ``pair_edge_vector_grad``.  ``edge_type_recip`` [T * T] f64
    (``1 / rc[source, target]``): per-edge-type cutoffs, the envelope takes ``r * edge_type_recip[T * t_i + t_j]``
    instead of ``r / r_max``.  ``cell`` [F, 3, 3] with ``batch`` [N]: a batch of frames, edge e takes the cell of frame
    ``batch[edge_index[0, e]]`` (as ``edge_embed``)."""
    _require_cuda(edge_index, types, table)
    edge_index = edge_index.long().contiguous()
    types = types.view(-1).long().contiguous()
    table = table.to(torch.float64).contiguous()
    if table.dim() != 3 or table.shape[0] != table.shape[1] or table.shape[2] != 2:
        raise ValueError(f"zbl_energy: table must be [T, T, 2], got {tuple(table.shape)}")
    if cutoff_dtype not in (torch.float32, torch.float64):
        raise ValueError(f"zbl_energy: cutoff_dtype must be float32 or float64, got {cutoff_dtype}")
    if (pos is None) == (edge_vectors is None):
        raise ValueError("zbl_energy: give exactly one of pos and edge_vectors")
    if (shift is None) != (cell is None):
        raise ValueError("shift and cell must be given together")
    if edge_vectors is not None:
        _require_cuda(edge_vectors)
        if shift is not None:
            raise ValueError("zbl_energy: edge_vectors already include the cell shifts")
        geom, from_vectors = edge_vectors.double().contiguous(), True
    else:
        _require_cuda(pos)
        geom, from_vectors = pos.double().contiguous(), False
        if geom.shape != (types.numel(), 3):
            raise ValueError(f"zbl_energy: pos must be [{types.numel()}, 3], got {tuple(geom.shape)}")
    frame = None
    if shift is not None:
        shift = shift.double().contiguous()
        if _framed(cell, batch):
            cell, frame = _frame_cells(cell, batch, types.numel(), "zbl_energy")
        else:
            cell = cell.double().reshape(3, 3).contiguous()
    recip = None
    if edge_type_recip is not None:
        _require_cuda(edge_type_recip)
        recip = edge_type_recip.to(torch.float64).reshape(-1).contiguous()
        if recip.numel() != table.shape[0] * table.shape[0]:
            raise ValueError(f"zbl_energy: edge_type_recip must hold T * T = {table.shape[0] ** 2} values")
    if frame is not None:
        return _ZBLFn.apply(geom, edge_index, shift, cell, types, table, float(r_max), float(poly_p),
                            cutoff_dtype == torch.float32, from_vectors, edge_grad_sink, recip, frame)
    if edge_type_recip is None:
        return _ZBLFn.apply(geom, edge_index, shift, cell, types, table, float(r_max), float(poly_p),
                            cutoff_dtype == torch.float32, from_vectors, edge_grad_sink)
    return _ZBLFn.apply(geom, edge_index, shift, cell, types, table, float(r_max), float(poly_p),
                        cutoff_dtype == torch.float32, from_vectors, edge_grad_sink, recip)


# ---------------------------------------------------------------------------------------
# grouped fp32-accurate GEMM on the tensor cores (wgmma 3xTF32) -- nqb_gemm_grouped
# ---------------------------------------------------------------------------------------
@dataclass
class GemmProblem:
    """C[M, N] (ldc, at c_off) (+)= rowscale[m] * A[M, K] (lda, at a_off) @ B[K, N]."""

    a_off: int
    lda: int
    c_off: int
    ldc: int
    B: torch.Tensor  # [K, N] (or [N, K] when transposed=True), float32
    scale: float = 1.0
    transposed: bool = False
    accumulate: bool = False  # C += ... (read-modify-write; at most ONE problem of the launch may touch an element)
    rs_off: int = -1  # row of the [R, M] row-scale matrix, -1 = none
    skip_zero_rows: bool = False  # rows with row scale 0 are left untouched (disjoint row-masked writers)
    atomic: bool = False  # C += ... with red.global.add (several problems of one launch add into the same C)
    # activation epilogue (nqb_gemm_grouped_act), v = the product above:
    #   "silu"       C = silu(v)
    #   "silu_save"  C = silu(v) and aux = v (the pre-activation, addressed like C)
    #   "silu_grad"  C = v * silu'(aux)  (aux = the pre-activation saved by "silu_save")
    act: str = "none"


# descriptor flag bits of each GemmProblem.act (nqb.h)
GEMM_ACT_FLAGS = {"none": 0, "silu": 8, "silu_save": 8 | 16, "silu_grad": 32}


class GroupedGemm:
    """A fixed list of GEMM problems sharing M, with their weights prepared once (split hi/lo, tiled)."""

    def __init__(self, problems, device):
        L = _capi.lib()
        self.problems = list(problems)
        rows = self.descriptor_rows(self.problems)
        blobs = []
        for p, row in zip(self.problems, rows):
            K, N = row[6], row[7]
            Bc = p.B.detach().to(device).contiguous()
            prep = torch.empty(int(L.nqb_gemm_prepared_floats(K, N)), dtype=torch.float32, device=device)
            _capi.check(L.nqb_gemm_prepare(_ptr(Bc), Bc.shape[1], K, N, int(p.transposed), float(p.scale), _ptr(prep),
                                           _stream()), "nqb_gemm_prepare")
            blobs.append(prep)
        self.act = any(p.act != "none" for p in self.problems)
        self.needs_aux = any(p.act in ("silu_save", "silu_grad") for p in self.problems)
        self.ntiles_total = rows[-1][10] + rows[-1][9]
        self.tile_ctas, self.sched_ctas = self._weighted_split(rows, device)
        self.prepared = torch.cat(blobs)
        self.descs = torch.tensor(rows, dtype=torch.int64, device=device)
        self.ndesc = len(rows)

    @staticmethod
    def descriptor_rows(problems) -> List[List[int]]:
        """The checked 12-int64 descriptor of each problem (nqb.h), with the weights laid out one after another."""
        if not problems:
            raise ValueError("GroupedGemm: empty problem list")
        L = _capi.lib()
        rows, b_off, tile0 = [], 0, 0
        for p in problems:
            K, N = (p.B.shape[1], p.B.shape[0]) if p.transposed else (p.B.shape[0], p.B.shape[1])
            if any(v % 4 for v in (K, N, p.lda, p.ldc, p.a_off, p.c_off)):
                raise ValueError("GroupedGemm: K, N, lda, ldc and offsets must be multiples of 4")
            if p.B.dtype != torch.float32:
                raise TypeError("GroupedGemm: float32 only")
            if p.act not in GEMM_ACT_FLAGS:
                raise ValueError(f"GroupedGemm: unknown act {p.act!r} (one of {', '.join(GEMM_ACT_FLAGS)})")
            if p.act != "none" and (p.accumulate or p.atomic):
                raise ValueError("GroupedGemm: an activation cannot be combined with accumulate or atomic")
            kchunks, ntiles = (K + 31) // 32, (N + 127) // 128
            rows.append([p.a_off, p.c_off, b_off, p.rs_off, p.lda, p.ldc, K, N, kchunks, ntiles, tile0,
                         (1 if p.accumulate else 0) | (2 if p.skip_zero_rows else 0) | (4 if p.atomic else 0)
                         | GEMM_ACT_FLAGS[p.act]])
            b_off += int(L.nqb_gemm_prepared_floats(K, N))
            tile0 += ntiles
        return rows

    @staticmethod
    def _weighted_split(rows, device):
        """CTAs per N-tile proportional to the tile's cost (pieces of K to multiply + columns to store, reduce-adds
        twice a store), for a grid of one CTA per SM.  None when there are more N-tiles than SMs."""
        if torch.device(device).type != "cuda":
            return None, 0
        G = torch.cuda.get_device_properties(device).multi_processor_count
        cost = []
        for (_a, _c, _b, _rs, _lda, _ldc, K, N, _kch, ntiles, _t0, flags) in rows:
            for t in range(ntiles):
                ncols = min(128, N - t * 128)
                cost.append(((K + 31) // 32) * 1000.0 + ((ncols + 31) // 32) * 650.0 * (2.0 if flags & 5 else 1.0))
        T = len(cost)
        # uniform launches (the radial-MLP GEMMs) keep the even split: its CTAs sweep the M-tiles in lockstep
        # and share every A tile in L2
        if T > G or T < 2 or max(cost) < 1.3 * min(cost):
            return None, 0
        n = [1] * T
        for _ in range(G - T):  # give the next CTA to the tile with the largest per-CTA load
            i = max(range(T), key=lambda j: cost[j] / n[j])
            n[i] += 1
        tab, c0 = [], 0
        for j in range(T):
            tab += [c0, n[j]]
            c0 += n[j]
        return torch.tensor(tab, dtype=torch.int32, device=device), c0

    def run(self, a: torch.Tensor, c: torch.Tensor, M: int, rowscale: Optional[torch.Tensor] = None,
            aux: Optional[torch.Tensor] = None):
        """``aux``: the pre-activation matrix of "silu_save" (written) / "silu_grad" (read) problems."""
        _require_cuda(a, c)
        if a.dtype != torch.float32 or c.dtype != torch.float32:
            raise TypeError("GroupedGemm.run: float32 only")
        rs_ld = int(rowscale.shape[-1]) if rowscale is not None else 0
        if not self.act:
            if aux is not None:
                raise ValueError("GroupedGemm.run: aux given, but no problem sets an activation")
            _capi.check(
                _capi.lib().nqb_gemm_grouped(_ptr(self.descs), self.ndesc, self.ntiles_total, _ptr(self.tile_ctas),
                                             int(self.sched_ctas), _ptr(a), _ptr(self.prepared), _ptr(c),
                                             _ptr(rowscale), rs_ld, int(M), _stream()),
                "nqb_gemm_grouped",
            )
            return c
        if self.needs_aux and aux is None:
            raise ValueError("GroupedGemm.run: silu_save / silu_grad problems need aux")
        if aux is not None:
            _require_cuda(aux)
            if aux.dtype != torch.float32:
                raise TypeError("GroupedGemm.run: float32 only")
        # "silu"-only launches never touch aux; the entry point still takes a valid base
        _capi.check(
            _capi.lib().nqb_gemm_grouped_act(_ptr(self.descs), self.ndesc, self.ntiles_total, _ptr(self.tile_ctas),
                                             int(self.sched_ctas), _ptr(a), _ptr(self.prepared), _ptr(c),
                                             _ptr(rowscale), rs_ld, int(M), _ptr(c if aux is None else aux), _stream()),
            "nqb_gemm_grouped_act",
        )
        return c

    def _check_pairs(self, a, c, pairs, who):
        pair_rows, count = pairs
        _require_cuda(a, c, pair_rows, count)
        if a.dtype != torch.float32 or c.dtype != torch.float32:
            raise TypeError(f"GroupedGemm.{who}: float32 only")
        if any(p.act != "none" or p.accumulate or p.atomic or p.skip_zero_rows or p.rs_off >= 0 for p in self.problems):
            raise ValueError(f"GroupedGemm.{who}: plain problems only (no row scale, accumulate, atomic or activation)")
        if pair_rows.dtype != torch.int64 or count.dtype != torch.int64 or pair_rows.dim() != 2 or pair_rows.shape[1] != 2:
            raise ValueError(f"GroupedGemm.{who}: pair_rows must be [E, 2] and count [1], int64")
        return pair_rows, count

    def run_pairs(self, a: torch.Tensor, c: torch.Tensor, pairs: Tuple[torch.Tensor, torch.Tensor]):
        """C on the slots of ``edge_pairs``: ``a`` holds one row per slot (rows < U are read) and result row u is
        stored to the C rows ``pair_rows[u]`` (the second when >= 0).  Plain problems only."""
        pair_rows, count = self._check_pairs(a, c, pairs, "run_pairs")
        _capi.check(
            _capi.lib().nqb_gemm_grouped_pairs(_ptr(self.descs), self.ndesc, self.ntiles_total, _ptr(self.tile_ctas),
                                               int(self.sched_ctas), _ptr(a), _ptr(self.prepared), _ptr(c),
                                               _ptr(pair_rows), _ptr(count), int(pair_rows.shape[0]), _stream()),
            "nqb_gemm_grouped_pairs",
        )
        return c

    def run_pair_sum(self, a: torch.Tensor, c: torch.Tensor, pairs: Tuple[torch.Tensor, torch.Tensor]):
        """The transpose of ``run_pairs``: result row u < U is ``(a[pair_rows[u, 0]] + a[pair_rows[u, 1]]) @ B`` (the
        second row only when >= 0), stored to row u of ``c`` (rows >= U untouched).  Plain problems only."""
        pair_rows, count = self._check_pairs(a, c, pairs, "run_pair_sum")
        _capi.check(
            _capi.lib().nqb_gemm_grouped_pair_sum(_ptr(self.descs), self.ndesc, self.ntiles_total, _ptr(self.tile_ctas),
                                                  int(self.sched_ctas), _ptr(a), _ptr(self.prepared), _ptr(c),
                                                  _ptr(pair_rows), _ptr(count), int(pair_rows.shape[0]), _stream()),
            "nqb_gemm_grouped_pair_sum",
        )
        return c


def edge_pairs(edge_index: torch.Tensor, shift: Optional[torch.Tensor], emb: torch.Tensor,
               csr: EdgeCSR) -> Tuple[torch.Tensor, torch.Tensor]:
    """Reverse-edge pair map of the radial MLP (``nqb_edge_pairs``): ``(pair_rows [E, 2], count [1])``, int64 on the
    device.  Slot u < count holds (representative edge, its reverse edge or -1); the two edges of a slot have bitwise
    equal ``emb`` rows, so the radial MLP computes the slot's row once.  ``shift`` [E, 3] or None; ``csr``: the
    destination CSR of ``edge_index[0]`` (``csr_cache``).  No host synchronisation (capturable)."""
    _require_cuda(edge_index, emb)
    if emb.dtype != torch.float32 or emb.dim() != 2:
        raise TypeError("edge_pairs: emb must be [E, num_bessel] float32")
    edge_index = edge_index.long().contiguous()
    E = edge_index.shape[1]
    if emb.shape[0] != E or csr.num_edges != E:
        raise ValueError("edge_pairs: emb / csr do not match edge_index")
    emb = emb.contiguous()
    if shift is not None:
        shift = shift.double().contiguous()
    L = _capi.lib()
    dev = edge_index.device
    pair_rows = torch.empty((E, 2), dtype=torch.int64, device=dev)
    count = torch.empty(1, dtype=torch.int64, device=dev)
    work = torch.empty(int(L.nqb_edge_pairs_work_size(E)), dtype=torch.int64, device=dev)
    _capi.check(L.nqb_edge_pairs(_ptr(edge_index), E, csr.num_nodes, _ptr(shift), _ptr(emb), emb.shape[1],
                                 _ptr(csr.row_ptr), _ptr(csr.perm), _ptr(work), _ptr(pair_rows), _ptr(count), _stream()),
                "nqb_edge_pairs")
    return pair_rows, count


def mlp_hidden_fwd_rows(emb: torch.Tensor, w1s: torch.Tensor, pairs: Tuple[torch.Tensor, torch.Tensor],
                        h: torch.Tensor) -> None:
    """``h[u] = silu(emb[pair_rows[u, 0]] @ w1s)`` for the slots u < count of ``edge_pairs``."""
    pair_rows, count = pairs
    _require_cuda(emb, w1s, pair_rows, count, h)
    _capi.check(_capi.lib().nqb_mlp_hidden_fwd_rows(_ptr(emb), _ptr(w1s), _ptr(pair_rows), _ptr(count),
                                                    pair_rows.shape[0], emb.shape[1], w1s.shape[1], _ptr(h), _stream()),
                "nqb_mlp_hidden_fwd_rows")


def mlp_hidden_fwd(emb: torch.Tensor, w1s: torch.Tensor, h: torch.Tensor, h_lo=None) -> None:
    """``h = silu(emb @ w1s)`` ([E,8] x [8,128]).  ``h_lo`` exists only so that ``bench.py``'s four-argument call
    keeps working; it must be None."""
    if h_lo is not None:
        raise ValueError("mlp_hidden_fwd: h_lo must be None")
    _require_cuda(emb, w1s, h)
    _capi.check(_capi.lib().nqb_mlp_hidden_fwd(_ptr(emb), _ptr(w1s), emb.shape[0], emb.shape[1], w1s.shape[1], _ptr(h),
                                               _stream()), "nqb_mlp_hidden_fwd")


def mlp_hidden_variant(variant: int = 0) -> int:
    """Returns 2: ``bench.py`` reports the hidden-layer kernels as ``"v%d" % mlp_hidden_variant(0)``, and this exists
    only for that call.  There is one kernel generation; any argument other than 0 or 2 raises ValueError."""
    if variant not in (0, 2):
        raise ValueError(f"mlp_hidden_variant: only variant 2 exists, got {variant!r}")
    return 2


def mlp_hidden_bwd(emb: torch.Tensor, w1s: torch.Tensor, gh: torch.Tensor, gemb: torch.Tensor) -> None:
    """``gemb = (gh * silu'(emb @ w1s)) @ w1s^T``."""
    _require_cuda(emb, w1s, gh, gemb)
    _capi.check(_capi.lib().nqb_mlp_hidden_bwd(_ptr(emb), _ptr(w1s), _ptr(gh), emb.shape[0], emb.shape[1], w1s.shape[1],
                                               _ptr(gemb), _stream()), "nqb_mlp_hidden_bwd")


def mlp_hidden_bwd_rows(emb: torch.Tensor, w1s: torch.Tensor, gh: torch.Tensor, pairs: Tuple[torch.Tensor, torch.Tensor],
                        gemb: torch.Tensor) -> None:
    """The backward of ``mlp_hidden_fwd_rows``: for the slots u < count of ``edge_pairs``,
    ``gemb[pair_rows[u, 0]] = (gh[u] * silu'(emb[pair_rows[u, 0]] @ w1s)) @ w1s^T`` and ``gemb[pair_rows[u, 1]] = 0``
    (when >= 0)."""
    pair_rows, count = pairs
    _require_cuda(emb, w1s, gh, pair_rows, count, gemb)
    _capi.check(_capi.lib().nqb_mlp_hidden_bwd_rows(_ptr(emb), _ptr(w1s), _ptr(gh), _ptr(pair_rows), _ptr(count),
                                                    pair_rows.shape[0], emb.shape[1], w1s.shape[1], _ptr(gemb),
                                                    _stream()),
                "nqb_mlp_hidden_bwd_rows")


# ---------------------------------------------------------------------------------------
# Gate nonlinearity -- nqb_gate_fwd / nqb_gate_bwd
# ---------------------------------------------------------------------------------------
class GateTables:
    """Column tables of the fused Gate kernels for ``irreps_in = scalars + gates + gated`` in ``layout``
    (e3nn ``nn.Gate``, nequip/nn/convnetlayer.py:104-112).  ``p`` of a scalar/gate irrep picks the activation:
    even -> c_silu * silu, odd -> c_tanh * tanh."""

    def __init__(self, irreps_scalars, irreps_gates, irreps_gated, layout: str, device):
        from .irreps import Irreps

        sc, ga, gd = Irreps(irreps_scalars), Irreps(irreps_gates), Irreps(irreps_gated)
        if sum(m for m, _ in ga) != sum(m for m, _ in gd):
            raise ValueError("Gate: one gate per gated multiplicity")
        ns, ng = sc.dim, ga.dim
        self.d_in = ns + ng + gd.dim
        self.d_out = ns + gd.dim
        src, gate, kind = [0] * self.d_out, [-1] * self.d_out, [0] * self.d_out
        tab = [[0] * 6 for _ in range(self.d_in)]
        off = 0
        for mul, ir in sc:  # scalars: out[j] = act(x[j])
            k = 0 if ir.p == 1 else 1
            for u in range(mul):
                src[off + u], kind[off + u] = off + u, k
                tab[off + u] = [0, off + u, 0, 0, 0, k]
            off += mul
        gate_kind = []
        for mul, ir in ga:
            gate_kind += [0 if ir.p == 1 else 1] * mul
        g0, in_off, out_off = 0, ns + ng, ns
        for mul, ir in gd:  # gated chunk: out = x * act(gate of its multiplicity index u)
            d = ir.dim
            stride = mul if layout == "ir_mul" else 1  # distance between the 2l+1 components of one u
            for u in range(mul):
                gcol, k = ns + g0 + u, gate_kind[g0 + u]
                first = u if layout == "ir_mul" else u * d
                tab[gcol] = [2, out_off + first, in_off + first, stride, d, k]
                for c in range(d):
                    pos = first + c * stride
                    src[out_off + pos], gate[out_off + pos], kind[out_off + pos] = in_off + pos, gcol, k
                    tab[in_off + pos] = [1, out_off + pos, gcol, 0, 0, k]
            g0 += mul
            in_off += mul * d
            out_off += mul * d
        mk = lambda v: torch.tensor(v, dtype=torch.int32, device=device).contiguous()
        self.src, self.gate, self.kind = mk(src), mk(gate), mk(kind)
        self.tab = mk([x for row in tab for x in row])


class _GateFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, tabs: GateTables):
        x = x.contiguous()
        out = torch.empty((x.shape[0], tabs.d_out), dtype=x.dtype, device=x.device)
        _capi.check(_capi.lib().nqb_gate_fwd(_DT[x.dtype], _ptr(x), x.shape[0], tabs.d_in, tabs.d_out, _ptr(tabs.src),
                                             _ptr(tabs.gate), _ptr(tabs.kind), _ptr(out), _stream()), "nqb_gate_fwd")
        ctx.tabs = tabs
        ctx.save_for_backward(x)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        (x,) = ctx.saved_tensors
        gout = gout.contiguous()
        gx = torch.empty_like(x)
        t = ctx.tabs
        _capi.check(_capi.lib().nqb_gate_bwd(_DT[x.dtype], _ptr(x), _ptr(gout), x.shape[0], t.d_in, t.d_out, _ptr(t.tab),
                                             _ptr(gx), _stream()), "nqb_gate_bwd")
        return gx, None


def gate(x: torch.Tensor, tabs: GateTables) -> torch.Tensor:
    """Fused Gate nonlinearity on ``x [N, scalars + gates + gated]`` (CUDA, float32/float64)."""
    _require_cuda(x)
    if x.dtype not in _DT or x.dim() != 2 or x.shape[1] != tabs.d_in:
        raise ValueError("gate: x must be [N, %d] float32/float64" % tabs.d_in)
    return _GateFn.apply(x, tabs)


# ---------------------------------------------------------------------------------------
# neighbour list on the device -- nqb_nl_bin / nqb_nl_count / nqb_nl_fill   (SURVEY 8f-2)
# ---------------------------------------------------------------------------------------
def _nl_cell(cell, pbc):
    """Host copies of the periodicity (3 bools), the cell (rows = lattice vectors) and its inverse."""
    import numpy as np

    if isinstance(pbc, bool):
        pbc = (pbc,) * 3
    pbc = [bool(b) for b in (pbc.tolist() if torch.is_tensor(pbc) else pbc)]
    if cell is None:
        if any(pbc):
            raise ValueError("Periodic boundary conditions requested but no cell was provided.")
        cell_np = np.eye(3)
    else:
        cell_np = (cell.detach().cpu().double().reshape(3, 3).numpy() if torch.is_tensor(cell) else np.asarray(cell, dtype=np.float64).reshape(3, 3)).copy()
    return pbc, cell_np, np.linalg.inv(cell_np)


def _nl_bin_cap(N: int) -> int:
    """Most bins per direction of the device list: round((4 N)^(1/3)), at least 1."""
    return max(1, int(round((4 * max(N, 1)) ** (1.0 / 3.0))))


def _nl_perp(inv_np):
    """Distance between opposite faces along each lattice direction = 1 / |column d of the inverse| (3 floats)."""
    import numpy as np

    return 1.0 / np.linalg.norm(inv_np, axis=0)


class _NlArgs:
    """Host-side arguments of the nqb_nl_* calls: cell, inverse, periodicity, bin grid and search range.

    ``nb`` (3 ints) fixes the bin grid instead of deriving it from the cell; the search range is still the one this
    cell needs with that grid (a variable-cell ``NeighborListPlan`` keeps its grid, and so its scratch sizes)."""

    def __init__(self, N: int, cell_np, inv_np, pbc, r_max: float, lo, width, nb=None):
        import numpy as np

        perp = _nl_perp(inv_np)
        fixed = nb is not None
        nb, sr = ([int(n) for n in nb] if fixed else [1, 1, 1]), [1, 1, 1]
        cap = _nl_bin_cap(N)
        for d in range(3):
            extent = perp[d] * (1.0 if pbc[d] else width[d])
            if not fixed:
                nb[d] = int(min(cap, max(1, np.floor(extent / r_max))))
            sr[d] = int(np.ceil(r_max / (extent / nb[d]) - 1e-12)) if pbc[d] else 1
            sr[d] = max(sr[d], 1)
        I3 = C.c_int * 3
        D9, D3 = C.c_double * 9, C.c_double * 3
        self.cell, self.inv = D9(*cell_np.reshape(-1)), D9(*inv_np.reshape(-1))
        self.pbc, self.nb, self.sr = I3(*[int(b) for b in pbc]), I3(*nb), I3(*sr)
        self.lo, self.width = D3(*lo), D3(*width)
        self.r_max = float(r_max)
        self.nbins = nb[0] * nb[1] * nb[2]


def _nl_scratch(N: int, nbins: int, dev) -> Dict[str, torch.Tensor]:
    """Buffers of the bin / sort / count / scan steps (``row_ptr`` is the exact list's destination CSR)."""
    return {
        "wpos": torch.empty((N, 3), dtype=torch.float64, device=dev),
        "base": torch.empty((N, 3), dtype=torch.int32, device=dev),
        "cidx": torch.empty((N, 3), dtype=torch.int32, device=dev),
        "binid": torch.empty((N,), dtype=torch.int64, device=dev),
        "sorted_bin": torch.empty((N,), dtype=torch.int64, device=dev),
        "order": torch.empty((N,), dtype=torch.int64, device=dev),
        "bins": torch.arange(nbins + 1, device=dev, dtype=torch.int64),
        "bin_start": torch.empty((nbins + 1,), dtype=torch.int64, device=dev),
        "counts": torch.zeros((N,), dtype=torch.int64, device=dev),
        "row_ptr": torch.zeros((N + 1,), dtype=torch.int64, device=dev),
    }


class _NlTypes:
    """Per-edge-type cutoffs of the device list: atom types [N] and ``rc2 = rc * rc`` [T * T] (float64, computed on
    the host) on the device; the pair (i, j) is a neighbour when ``d2 < rc2[T * types[i] + types[j]]``."""

    def __init__(self, atom_types, edge_type_cutoff, r_max: float, num_atoms: int, device):
        import numpy as np

        rc = (edge_type_cutoff.detach().cpu().double().numpy() if torch.is_tensor(edge_type_cutoff)
              else np.asarray(edge_type_cutoff, dtype=np.float64))
        if rc.ndim != 2 or rc.shape[0] != rc.shape[1] or rc.shape[0] < 1:
            raise ValueError(f"edge_type_cutoff must be a [T, T] table, got shape {tuple(rc.shape)}")
        if not (np.all(rc > 0) and np.all(rc <= r_max)):
            raise ValueError(f"edge_type_cutoff: every entry must satisfy 0 < rc <= r_max = {r_max}")
        if atom_types is None:
            raise ValueError("edge_type_cutoff needs atom_types")
        types = torch.as_tensor(atom_types).view(-1)
        if types.numel() != num_atoms:
            raise ValueError(f"atom_types must hold {num_atoms} types, got {types.numel()}")
        T = rc.shape[0]
        if num_atoms and (int(types.min()) < 0 or int(types.max()) >= T):
            raise ValueError(f"atom_types must lie in [0, {T})")
        self.T = T
        # a copy the list owns: a captured graph keeps its pointer
        self.types = types.to(device=device, dtype=torch.int64).contiguous().clone()
        self.rc2 = torch.from_numpy((rc * rc).reshape(-1)).to(device)


def _nl_rows(pos: torch.Tensor, a: _NlArgs, s: Dict[str, torch.Tensor],
             params_dev: Optional[torch.Tensor] = None, ty: Optional[_NlTypes] = None) -> None:
    """Bins, atoms sorted by bin, neighbours per atom and their exclusive scan into ``s["row_ptr"]``; all on the
    device, no host synchronisation.  ``params_dev``: read the cell-dependent arguments from this device parameter
    block (``nqb_nl_params_pack``) instead of passing ``a``'s by value.  ``ty``: per-edge-type cutoffs."""
    L = _capi.lib()
    N = pos.shape[0]
    st = _stream()
    if params_dev is None:
        _capi.check(L.nqb_nl_bin(_ptr(pos), N, a.cell, a.inv, a.pbc, a.nb, a.sr, a.lo, a.width, a.r_max,
                                 _ptr(s["wpos"]), _ptr(s["base"]), _ptr(s["binid"]), _ptr(s["cidx"]), st), "nqb_nl_bin")
    else:
        _capi.check(L.nqb_nl_bin_dp(_ptr(pos), N, _ptr(params_dev), _ptr(s["wpos"]), _ptr(s["base"]), _ptr(s["binid"]),
                                    _ptr(s["cidx"]), st), "nqb_nl_bin_dp")
    torch.sort(s["binid"], stable=True, out=(s["sorted_bin"], s["order"]))
    torch.searchsorted(s["sorted_bin"], s["bins"], out=s["bin_start"])
    if ty is not None and params_dev is None:
        _capi.check(L.nqb_nl_count_typed(N, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, _ptr(s["wpos"]), _ptr(s["cidx"]),
                                         _ptr(s["order"]), _ptr(s["bin_start"]), _ptr(ty.types), _ptr(ty.rc2), ty.T,
                                         _ptr(s["counts"]), st), "nqb_nl_count_typed")
    elif ty is not None:
        _capi.check(L.nqb_nl_count_dp_typed(N, _ptr(params_dev), _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["order"]),
                                            _ptr(s["bin_start"]), _ptr(ty.types), _ptr(ty.rc2), ty.T, _ptr(s["counts"]),
                                            st), "nqb_nl_count_dp_typed")
    elif params_dev is None:
        _capi.check(L.nqb_nl_count(N, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, _ptr(s["wpos"]), _ptr(s["cidx"]),
                                   _ptr(s["order"]), _ptr(s["bin_start"]), _ptr(s["counts"]), st), "nqb_nl_count")
    else:
        _capi.check(L.nqb_nl_count_dp(N, _ptr(params_dev), _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["order"]),
                                      _ptr(s["bin_start"]), _ptr(s["counts"]), st), "nqb_nl_count_dp")
    torch.cumsum(s["counts"], 0, out=s["row_ptr"][1:])


def neighbor_list(pos: torch.Tensor, cell=None, pbc=True, r_max: float = 5.0, transpose_perm: bool = False,
                  atom_types=None, edge_type_cutoff=None, batch=None):
    """Full neighbour list within ``r_max`` built on the GPU (cell list), in the layout the convolution wants.

    ``pos`` [N,3] float64 CUDA; ``cell`` [3,3] (rows = lattice vectors; host or device) or None; ``pbc`` bool or 3
    bools.  Returns a dict with ``edge_index`` [2,E] int64 (row 0 = centre / scatter destination, row 1 =
    neighbour), ``edge_cell_shift`` [E,3] float64 (edge vector = pos[j] - pos[i] + shift @ cell), ``row_ptr``
    [N+1] int64 (destination CSR: edges are sorted by (centre, neighbour)) and, on request,
    ``edge_transpose_perm`` [E] (argsort by (neighbour, centre), nequip/data/transforms/neighborlist.py:150-155).
    Same contract as the reference's host backends (nequip/data/_nl.py:60-152): both directions, no self edge in
    the home image.  One host synchronisation (the edge count); ``NeighborListPlan`` has none.

    Per-edge-type cutoffs: ``edge_type_cutoff`` [T, T] (``rc[source, target]``, 0 < rc <= r_max) with ``atom_types``
    [N] keeps the pair (i, j) when ``d2 < rc[t_i, t_j]^2`` (``rc * rc`` in float64); the bins are those of ``r_max``.

    A batch of independent frames (``batch`` [N] int, the frame of each atom, non-decreasing): ``cell`` [F, 3, 3] or
    None (every frame open), ``pbc`` a bool, [3] or [F, 3]; F is the number of cells, else of ``pbc`` rows, else
    ``batch.max() + 1``, and a frame may hold no atoms.  The result is the concatenation over frames of the single-frame
    lists, bit for bit, with atom indices offset by each frame's first atom (``row_ptr`` [N+1] over all atoms).  A frame
    open in every direction takes the identity cell, whatever its row of ``cell`` holds.  One set of launches for all
    frames; host synchronisations for the checks of ``batch``, one read-back of the per-frame atom counts and bounding
    boxes, and the edge count."""
    import numpy as np

    if batch is not None:
        return _neighbor_list_frames(pos, cell, pbc, r_max, transpose_perm, atom_types, edge_type_cutoff, batch)
    _require_cuda(pos)
    L = _capi.lib()
    pos = pos.detach().double().contiguous()
    N = pos.shape[0]
    dev = pos.device
    pbc, cell_np, inv_np = _nl_cell(cell, pbc)
    lo = np.zeros(3)
    width = np.ones(3)
    if not all(pbc) and N > 0:
        frac = pos @ torch.as_tensor(inv_np, device=dev)
        fmin, fmax = frac.min(0).values.cpu().numpy(), frac.max(0).values.cpu().numpy()
        for d in range(3):
            if not pbc[d]:
                lo[d], width[d] = fmin[d], max(fmax[d] - fmin[d], 1e-9) * (1 + 1e-9)
    a = _NlArgs(N, cell_np, inv_np, pbc, r_max, lo, width)
    ty = None
    if edge_type_cutoff is not None:
        ty = _NlTypes(atom_types, edge_type_cutoff, float(r_max), N, dev)
    elif atom_types is not None:
        raise ValueError("atom_types is only read with edge_type_cutoff")
    s = _nl_scratch(N, a.nbins, dev)
    if ty is None:
        _nl_rows(pos, a, s)
    else:
        _nl_rows(pos, a, s, ty=ty)
    row_ptr = s["row_ptr"]
    E = int(row_ptr[-1].item())
    edge_index = torch.empty((2, E), dtype=torch.int64, device=dev)
    shifts = torch.empty((E, 3), dtype=torch.float64, device=dev)
    if ty is None:
        _capi.check(L.nqb_nl_fill(N, E, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, _ptr(s["wpos"]), _ptr(s["cidx"]),
                                  _ptr(s["base"]), _ptr(s["order"]), _ptr(s["bin_start"]), _ptr(row_ptr),
                                  _ptr(edge_index), _ptr(shifts), _stream()), "nqb_nl_fill")
    else:
        _capi.check(L.nqb_nl_fill_typed(N, E, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, _ptr(s["wpos"]),
                                        _ptr(s["cidx"]), _ptr(s["base"]), _ptr(s["order"]), _ptr(s["bin_start"]),
                                        _ptr(row_ptr), _ptr(ty.types), _ptr(ty.rc2), ty.T, _ptr(edge_index),
                                        _ptr(shifts), _stream()), "nqb_nl_fill_typed")
    out = {"edge_index": edge_index, "edge_cell_shift": shifts, "row_ptr": row_ptr}
    if transpose_perm:
        out["edge_transpose_perm"] = torch.argsort(edge_index[1] * N + edge_index[0], stable=True)
    return out


def _nl_frame_args(cell, pbc, batch, num_atoms: int):
    """Host checks of a batched ``neighbor_list``: (F, pbc [F, 3] bool, cells [F, 3, 3] float64) with the identity
    as the cell of a frame open in every direction.  ``ValueError`` for a ``batch`` that is not [N] integers or
    decreases or leaves [0, F), a cell that is not [F, 3, 3], a ``pbc`` of another shape or row count, and a periodic
    frame without a cell."""
    import numpy as np

    b = torch.as_tensor(batch)
    if b.dim() != 1 or b.numel() != num_atoms or b.dtype.is_floating_point or b.dtype == torch.bool:
        raise ValueError(f"neighbor_list: batch must be [{num_atoms}] integers, got {tuple(b.shape)} {b.dtype}")
    if num_atoms > 1 and bool((b[1:] < b[:-1]).any()):
        raise ValueError("neighbor_list: batch must be non-decreasing (each frame is one contiguous range of atoms)")
    F = None
    if cell is not None:
        c = cell.detach().cpu().double().numpy() if torch.is_tensor(cell) else np.asarray(cell, dtype=np.float64)
        if c.ndim != 3 or c.shape[1:] != (3, 3):
            raise ValueError(f"neighbor_list: with batch, cell must be [F, 3, 3], got {tuple(c.shape)}")
        F = c.shape[0]
    p = pbc.detach().cpu().numpy() if torch.is_tensor(pbc) else np.asarray(pbc)
    if p.shape == ():
        p = np.full(3, bool(p))
    if p.shape == (3,):
        if F is None:
            F = int(b.max()) + 1 if num_atoms else 0
        p = np.broadcast_to(p, (F, 3))
    elif p.ndim == 2 and p.shape[1] == 3:
        if F is not None and p.shape[0] != F:
            raise ValueError(f"neighbor_list: pbc has {p.shape[0]} rows for {F} cells")
        F = p.shape[0]
    else:
        raise ValueError(f"neighbor_list: with batch, pbc must be a bool, [3] or [F, 3], got shape {tuple(p.shape)}")
    p = p.astype(bool)
    if cell is None:
        if p.any():
            raise ValueError("Periodic boundary conditions requested but no cell was provided.")
        c = np.zeros((F, 3, 3))
    if num_atoms and (int(b.min()) < 0 or int(b.max()) >= F):
        raise ValueError(f"neighbor_list: batch holds frame indices outside [0, {F})")
    c = c.copy()
    c[~p.any(axis=1)] = np.eye(3)  # an open frame's edges do not depend on its cell (nvalchemiops uses the identity)
    return F, p, c


def _neighbor_list_frames(pos, cell, pbc, r_max, transpose_perm, atom_types, edge_type_cutoff, batch):
    """``neighbor_list`` of a batch of frames: the ``_NlArgs`` of each frame as the single-frame call builds them,
    packed into one device block per frame (``nqb_nl_frames_pack``), and one bin / sort / count / scan / fill over
    all frames with each frame's bins at ``bin_base[f]`` of one global range."""
    import numpy as np

    N = pos.shape[0]
    F, pbc_np, cells = _nl_frame_args(cell, pbc, batch, N)
    _require_cuda(pos)
    L = _capi.lib()
    pos = pos.detach().double().contiguous()
    dev = pos.device
    frame = torch.as_tensor(batch).to(device=dev, dtype=torch.int64).contiguous()
    invs = np.linalg.inv(cells) if F else np.zeros((0, 3, 3))
    # per-frame atom counts and, for frames with an open direction, the bounding box of the fractional coordinates:
    # one segmented min / max on the device and one read-back
    stats = torch.bincount(frame, minlength=F).double().view(F, 1)
    if N and not pbc_np.all():
        frac = torch.bmm(pos.view(N, 1, 3), torch.as_tensor(invs, device=dev)[frame]).view(N, 3)
        idx = frame.view(N, 1).expand(N, 3)
        fmin = torch.full((F, 3), float("inf"), dtype=torch.float64, device=dev).scatter_reduce(0, idx, frac, "amin")
        fmax = torch.full((F, 3), float("-inf"), dtype=torch.float64, device=dev).scatter_reduce(0, idx, frac, "amax")
        stats = torch.cat([stats, fmin, fmax], 1)
    host = stats.cpu().numpy()
    I3, D9, D3 = C.c_int * (3 * F), C.c_double * (9 * F), C.c_double * (3 * F)
    cols = {k: [] for k in ("pbc", "nb", "sr", "lo", "width")}
    nbins = [0]
    for f in range(F):
        nf = int(host[f, 0])
        lo, width = np.zeros(3), np.ones(3)
        if not pbc_np[f].all() and nf > 0:
            for d in range(3):
                if not pbc_np[f, d]:
                    lo[d], width[d] = host[f, 1 + d], max(host[f, 4 + d] - host[f, 1 + d], 1e-9) * (1 + 1e-9)
        a = _NlArgs(nf, cells[f], invs[f], [bool(v) for v in pbc_np[f]], r_max, lo, width)
        for k in cols:
            cols[k].extend(getattr(a, k))
        nbins.append(a.nbins)
    bin_base = np.cumsum(nbins)
    block_bytes = int(L.nqb_nl_params_bytes())
    blocks = C.create_string_buffer(max(1, F * block_bytes))
    _capi.check(L.nqb_nl_frames_pack(F, D9(*cells.reshape(-1)), D9(*invs.reshape(-1)), I3(*cols["pbc"]),
                                     I3(*cols["nb"]), I3(*cols["sr"]), D3(*cols["lo"]), D3(*cols["width"]),
                                     float(r_max), blocks), "nqb_nl_frames_pack")
    blocks_dev = torch.frombuffer(bytearray(blocks.raw), dtype=torch.uint8).to(dev)
    bin_base_dev = torch.as_tensor(bin_base, dtype=torch.int64).to(dev)
    ty = None
    if edge_type_cutoff is not None:
        ty = _NlTypes(atom_types, edge_type_cutoff, float(r_max), N, dev)
    elif atom_types is not None:
        raise ValueError("atom_types is only read with edge_type_cutoff")
    types, rc2, T = (0, 0, 0) if ty is None else (_ptr(ty.types), _ptr(ty.rc2), ty.T)
    s = _nl_scratch(N, int(bin_base[-1]), dev)
    st = _stream()
    fr = (_ptr(blocks_dev), _ptr(frame), _ptr(bin_base_dev))
    _capi.check(L.nqb_nl_bin_frames(_ptr(pos), N, *fr, _ptr(s["wpos"]), _ptr(s["base"]), _ptr(s["binid"]),
                                    _ptr(s["cidx"]), st), "nqb_nl_bin_frames")
    torch.sort(s["binid"], stable=True, out=(s["sorted_bin"], s["order"]))
    torch.searchsorted(s["sorted_bin"], s["bins"], out=s["bin_start"])
    _capi.check(L.nqb_nl_count_frames(N, *fr, _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["order"]),
                                      _ptr(s["bin_start"]), types, rc2, T, _ptr(s["counts"]), st),
                "nqb_nl_count_frames")
    row_ptr = s["row_ptr"]
    torch.cumsum(s["counts"], 0, out=row_ptr[1:])
    E = int(row_ptr[-1].item())
    edge_index = torch.empty((2, E), dtype=torch.int64, device=dev)
    shifts = torch.empty((E, 3), dtype=torch.float64, device=dev)
    _capi.check(L.nqb_nl_fill_frames(N, E, *fr, _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["base"]), _ptr(s["order"]),
                                     _ptr(s["bin_start"]), _ptr(row_ptr), types, rc2, T, _ptr(edge_index),
                                     _ptr(shifts), st), "nqb_nl_fill_frames")
    out = {"edge_index": edge_index, "edge_cell_shift": shifts, "row_ptr": row_ptr}
    if transpose_perm:
        # frames hold disjoint, increasing atom ranges: the global (neighbour, centre) order is the frames' orders
        out["edge_transpose_perm"] = torch.argsort(edge_index[1] * N + edge_index[0], stable=True)
    return out


def null_edge_shift(cell, r_max: float):
    """Cell shift [3] (integer-valued float64, host) of the null edges of ``NeighborListPlan``: ``k e_d`` along the
    longest lattice vector ``a_d``, ``k = floor(r_max / |a_d|) + 2``, so the edge (i, i, k e_d) is at least
    ``r_max + |a_d|`` long.  Its cutoff envelope and the envelope's derivative are exactly 0 there, and the radial MLP
    has no bias with silu(0) = 0, so such an edge adds exact zeros to the energy, the forces and the virial."""
    import numpy as np

    cell_np = (cell.detach().cpu().double().reshape(3, 3).numpy() if torch.is_tensor(cell)
               else np.asarray(cell, dtype=np.float64).reshape(3, 3))
    lengths = np.linalg.norm(cell_np, axis=1)
    d = int(np.argmax(lengths))
    shift = np.zeros(3)
    shift[d] = np.floor(r_max / lengths[d]) + 2
    return shift


def _nl_check_cell(cell, what: str):
    """``cell`` ([3,3] or [1,3,3]) as a [3, 3] float64 host array; ``ValueError`` for another shape, a non-finite or a
    singular cell."""
    import numpy as np

    c = cell.detach().cpu().double().numpy() if torch.is_tensor(cell) else np.asarray(cell, dtype=np.float64)
    if c.shape not in ((3, 3), (1, 3, 3)):
        raise ValueError(f"{what}: cell must be [3, 3] or [1, 3, 3], got {tuple(c.shape)}")
    c = c.reshape(3, 3)
    if not np.all(np.isfinite(c)):
        raise ValueError(f"{what}: cell is not finite")
    vol = abs(float(np.linalg.det(c)))
    if not vol > 1e-12 * float(np.prod(np.linalg.norm(c, axis=1))):
        raise ValueError(f"{what}: cell is singular")
    return c


def _nl_cell_block(cell, r_max: float, nb, num_atoms: int):
    """Host part of ``NeighborListPlan.set_cell``: checks ``cell`` ([3,3] or [1,3,3], finite, non-singular) and returns
    the ``_NlArgs`` of this cell on the fixed bin grid ``nb`` (inverse as in ``neighbor_list``, search range for this
    cell), its null-edge shift and the packed device parameter block (``nqb_nl_params_pack``, ctypes buffer)."""
    import numpy as np

    c = _nl_check_cell(cell, "set_cell")
    pbc, cell_np, inv_np = _nl_cell(c, True)
    a = _NlArgs(num_atoms, cell_np, inv_np, pbc, r_max, np.zeros(3), np.ones(3), nb=nb)
    pad_shift = null_edge_shift(cell_np, r_max)
    L = _capi.lib()
    block = C.create_string_buffer(int(L.nqb_nl_params_bytes()))
    _capi.check(L.nqb_nl_params_pack(a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, (C.c_double * 3)(*pad_shift), block),
                "nqb_nl_params_pack")
    return a, pad_shift, block


class NeighborListPlan:
    """Device neighbour list of a fixed length ``capacity`` for one cell: positions in, list out, without a host
    synchronisation, so it can be captured in a CUDA graph (``graph.GraphedMDStep``).

    All host work (inverse cell, bin grid, search range, the null-edge shift) and every allocation happen here; the
    cell is fixed for the plan's lifetime unless ``variable_cell``.  The cell must be given and periodic in all three
    directions unless ``open_boundaries`` (below).

    ``variable_cell=True`` (constant-pressure MD): the kernels read the cell-dependent arguments from a parameter
    block in device memory, and ``set_cell(cell)`` replaces them between runs (or graph replays) without touching
    the captured launches.  The bin grid chosen for the construction cell is kept for the plan's lifetime (the
    scratch sizes depend on it); each cell gets the search range it needs on that grid, so any cell gives the exact
    list and a cell far from the first one only costs more or less bin visits.  The null-edge shift follows the cell.

    ``run(pos)`` returns ``edge_index`` [2, capacity], ``edge_cell_shift`` [capacity, 3], ``row_ptr`` [N+1] (the
    padded destination CSR), ``num_edges`` [1] int64 (the true edge count E) and ``overflow`` [1] int32, all on the
    device and all overwritten by the next ``run``.  Row i holds its real edges in the order of ``neighbor_list``,
    then null edges (i, i, ``pad_shift``); each row gets floor or ceil of (capacity - E) / N of them.  When
    E > capacity, ``overflow`` is 1 and every row holds only null edges: the list must not be used.

    ``atom_types`` [N] + ``edge_type_cutoff`` [T, T]: per-edge-type cutoffs as in ``neighbor_list``.  The types are
    fixed for the plan's lifetime (the plan keeps a device copy whose pointer captured graphs hold); the cutoff table
    does not depend on the cell, so ``set_cell`` leaves it alone.

    ``open_boundaries=True`` (molecules in vacuum, slabs): any ``pbc`` is accepted, and ``cell=None`` when no direction
    is periodic (the identity then serves as the cell, as in ``neighbor_list``).  A plan with an open direction reads
    its arguments from a device parameter block (``nqb_nl_params_pack_open``), and ``run`` first finds the bounding box
    of the positions along the open directions on the device (``nqb_nl_bbox``), with the grid ``neighbor_list``
    derives from it on the host: ``nb = min(cap, max(1, floor(perp * width / r_max)))``, cap = round((4 N)^(1/3)).
    The rows are those of ``neighbor_list(pos, cell, pbc)``.  ``plan.cell`` ([3, 3] float64, on the device) is the cell
    the shifts refer to: the caller must give it to the model as ``cell``, since the null edges (i, i, pad_shift)
    only have their length r_max + |a_d| through it; real edges along open directions have shift 0.  The cell must be
    finite and non-singular, and ``variable_cell`` needs all three directions periodic.

    ``batch`` [N] (a batch of independent frames, as in ``neighbor_list(..., batch=)``): ``cell`` [F, 3, 3] or None,
    ``pbc`` a bool, [3] or [F, 3]; ``batch`` is checked once, here, and is fixed for the plan's lifetime, as are the
    frames' atom counts.  Each frame gets its own parameter block (``nqb_nl_frames_pack_capacity``): its bin grid, fixed
    here, with ``cap_f = round((4 N_f)^(1/3))`` bins along its open directions, and its own null-edge shift
    (``pad_shift`` [F, 3]): one shift for all frames could be shorter than r_max in another frame's cell.  ``run`` finds
    the bounding boxes of the frames with an open direction on the device (``nqb_nl_bbox_frames``, one CTA per frame),
    then bins, counts and fills over all frames.  Row i holds the real edges of ``neighbor_list(pos, cell, pbc,
    batch=)`` then null edges (i, i, pad_shift of i's frame); one ``capacity`` and one ``overflow`` flag serve the batch,
    since every row only holds its own frame's edges.  ``plan.cell`` [F, 3, 3] (the identity for a frame open in every
    direction) is the cell the model must be given.  A frame with an open direction needs ``open_boundaries``;
    ``variable_cell`` needs every frame periodic in all three directions, and ``set_cell`` then takes [F, 3, 3]."""

    _fr = None  # the frames of a batched plan (batch=); None for one frame

    def __init__(self, num_atoms: int, cell, pbc, r_max: float, capacity: int, device=None,
                 variable_cell: bool = False, atom_types=None, edge_type_cutoff=None, *,
                 open_boundaries: bool = False, batch=None):
        import numpy as np

        if batch is not None:
            self._init_frames(num_atoms, cell, pbc, r_max, capacity, device, variable_cell, atom_types,
                              edge_type_cutoff, open_boundaries, batch)
            return
        if isinstance(pbc, bool):
            pbc = (pbc,) * 3
        pbc = [bool(b) for b in (pbc.tolist() if torch.is_tensor(pbc) else pbc)]
        if not open_boundaries:
            if cell is None:
                raise ValueError("NeighborListPlan needs a cell")
            if len(pbc) != 3 or not all(pbc):
                raise ValueError("NeighborListPlan needs all three directions periodic unless built with "
                                 "open_boundaries=True")
        else:
            if len(pbc) != 3:
                raise ValueError(f"NeighborListPlan: pbc must be a bool or 3 bools, got {pbc}")
            if cell is None and any(pbc):
                raise ValueError("NeighborListPlan: a periodic direction needs a cell")
            if variable_cell and not all(pbc):
                raise ValueError("NeighborListPlan: variable_cell needs all three directions periodic")
            if cell is not None:
                _nl_check_cell(cell, "NeighborListPlan")
        if int(num_atoms) < 1 or int(capacity) < 0:
            raise ValueError("NeighborListPlan needs num_atoms >= 1 and capacity >= 0")
        self.num_atoms, self.capacity, self.r_max = int(num_atoms), int(capacity), float(r_max)
        pbc, cell_np, inv_np = _nl_cell(cell, pbc)
        self.pad_shift = null_edge_shift(cell_np, r_max)
        self._pad_shift_c = (C.c_double * 3)(*self.pad_shift)
        dev = torch.device(device) if device is not None else (
            cell.device if torch.is_tensor(cell) and cell.is_cuda else torch.device("cuda"))
        self.device = dev
        self._a = _NlArgs(self.num_atoms, cell_np, inv_np, pbc, r_max, np.zeros(3), np.ones(3))
        self._open = not all(pbc)
        if open_boundaries:
            self.cell = torch.from_numpy(cell_np.copy()).to(dev)
        if self._open:
            # scratch grid: cap bins along every open direction; nqb_nl_bbox picks at most that many per run
            cap = _nl_bin_cap(self.num_atoms)
            nb = [n if p else cap for n, p in zip(self._a.nb, pbc)]
            self._a = _NlArgs(self.num_atoms, cell_np, inv_np, pbc, r_max, np.zeros(3), np.ones(3), nb=nb)
            L = _capi.lib()
            block = C.create_string_buffer(int(L.nqb_nl_params_bytes()))
            a = self._a
            _capi.check(L.nqb_nl_params_pack_open(a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max, self._pad_shift_c, cap,
                                                  (C.c_double * 3)(*_nl_perp(inv_np)), block),
                        "nqb_nl_params_pack_open")
            open_block = torch.frombuffer(bytearray(block.raw), dtype=torch.uint8).to(dev)
            self._bbox_work = torch.zeros((8,), dtype=torch.int64, device=dev)  # left zero by every nqb_nl_bbox
        self._ty = None
        if edge_type_cutoff is not None:
            self._ty = _NlTypes(atom_types, edge_type_cutoff, self.r_max, self.num_atoms, dev)
        elif atom_types is not None:
            raise ValueError("NeighborListPlan: atom_types is only read with edge_type_cutoff")
        self._s = _nl_scratch(self.num_atoms, self._a.nbins, dev)
        N, cap = self.num_atoms, self.capacity
        self.edge_index = torch.empty((2, cap), dtype=torch.int64, device=dev)
        self.edge_cell_shift = torch.empty((cap, 3), dtype=torch.float64, device=dev)
        self.row_ptr = torch.empty((N + 1,), dtype=torch.int64, device=dev)
        self.num_edges = torch.empty((1,), dtype=torch.int64, device=dev)
        self.overflow = torch.empty((1,), dtype=torch.int32, device=dev)
        self.variable_cell = bool(variable_cell)
        self._params_dev = None
        if self.variable_cell:
            self.nbins = tuple(self._a.nb)
            nbytes = int(_capi.lib().nqb_nl_params_bytes())
            self._params_dev = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
            self._params_host = torch.empty((nbytes,), dtype=torch.uint8).pin_memory()
            self._params_event: Optional[torch.cuda.Event] = None
            self.set_cell(cell)
        elif self._open:
            self._params_dev = open_block

    def _init_frames(self, num_atoms, cell, pbc, r_max, capacity, device, variable_cell, atom_types, edge_type_cutoff,
                     open_boundaries, batch) -> None:
        import numpy as np

        N = int(num_atoms)
        if N < 1 or int(capacity) < 0:
            raise ValueError("NeighborListPlan needs num_atoms >= 1 and capacity >= 0")
        F, pbc_np, cells = _nl_frame_args(cell, pbc, batch, N)
        open_f = ~pbc_np.all(axis=1)
        if open_f.any() and not open_boundaries:
            raise ValueError("NeighborListPlan: a frame with an open direction needs open_boundaries=True")
        if variable_cell and open_f.any():
            raise ValueError("NeighborListPlan: variable_cell needs every frame periodic in all three directions")
        for f in range(F):
            _nl_check_cell(cells[f], "NeighborListPlan")
        self.num_atoms, self.capacity, self.r_max = N, int(capacity), float(r_max)
        self.num_frames = F
        frame = torch.as_tensor(batch).view(-1).to(torch.int64)
        counts = torch.bincount(frame.cpu(), minlength=F).numpy()
        dev = torch.device(device) if device is not None else (
            frame.device if frame.is_cuda else torch.device("cuda"))
        self.device = dev
        invs = np.linalg.inv(cells)
        self._counts = [int(n) for n in counts]
        self._pbc = [[bool(v) for v in pbc_np[f]] for f in range(F)]
        # the bin grid of every frame, fixed here: cap_f bins along open directions (nqb_nl_bbox_frames picks at most
        # that many per run); the frames' ranges of one global bin range start at bin_base
        self._caps = [_nl_bin_cap(n) for n in self._counts]
        self._nbins = []
        for f in range(F):
            a = _NlArgs(self._counts[f], cells[f], invs[f], self._pbc[f], r_max, np.zeros(3), np.ones(3))
            self._nbins.append([n if p else self._caps[f] for n, p in zip(a.nb, self._pbc[f])])
        block = self._pack_frames(cells, invs)
        self._fr = {
            "frame": frame.to(dev).contiguous().clone(),
            "bin_base": torch.as_tensor(np.cumsum([0] + [int(np.prod(nb)) for nb in self._nbins]),
                                        dtype=torch.int64).to(dev),
            "atom_ptr": torch.as_tensor(np.cumsum([0] + self._counts), dtype=torch.int64).to(dev),
        }
        self._open = bool(open_f.any())
        self.cell = torch.from_numpy(cells.copy()).to(dev)
        self._ty = None
        if edge_type_cutoff is not None:
            self._ty = _NlTypes(atom_types, edge_type_cutoff, self.r_max, N, dev)
        elif atom_types is not None:
            raise ValueError("NeighborListPlan: atom_types is only read with edge_type_cutoff")
        self._s = _nl_scratch(N, int(self._fr["bin_base"][-1]), dev)
        cap = self.capacity
        self.edge_index = torch.empty((2, cap), dtype=torch.int64, device=dev)
        self.edge_cell_shift = torch.empty((cap, 3), dtype=torch.float64, device=dev)
        self.row_ptr = torch.empty((N + 1,), dtype=torch.int64, device=dev)
        self.num_edges = torch.empty((1,), dtype=torch.int64, device=dev)
        self.overflow = torch.empty((1,), dtype=torch.int32, device=dev)
        self.variable_cell = bool(variable_cell)
        self._params_dev = torch.frombuffer(bytearray(block.raw), dtype=torch.uint8).to(dev)
        if self.variable_cell:
            self._params_host = torch.empty((len(block),), dtype=torch.uint8).pin_memory()
            self._params_event: Optional[torch.cuda.Event] = None
            self.cell_error = torch.zeros((F,), dtype=torch.int32, device=dev)

    def _pack_frames(self, cells, invs):
        """The frames' device parameter blocks (``nqb_nl_frames_pack_capacity``, ctypes buffer) for ``cells`` on the
        plan's bin grids, each frame with the search range its cell needs and its own null-edge shift."""
        import numpy as np

        F = self.num_frames
        cols = {k: [] for k in ("pbc", "nb", "sr", "lo", "width")}
        pad, perp = [], []
        for f in range(F):
            a = _NlArgs(self._counts[f], cells[f], invs[f], self._pbc[f], self.r_max, np.zeros(3), np.ones(3),
                        nb=self._nbins[f])
            for k in cols:
                cols[k].extend(getattr(a, k))
            pad.extend(null_edge_shift(cells[f], self.r_max))
            perp.extend(_nl_perp(invs[f]))
        self.pad_shift = np.asarray(pad, dtype=np.float64).reshape(F, 3)
        I3, D9, D3 = C.c_int * (3 * F), C.c_double * (9 * F), C.c_double * (3 * F)
        L = _capi.lib()
        block = C.create_string_buffer(F * int(L.nqb_nl_params_bytes()))
        _capi.check(L.nqb_nl_frames_pack_capacity(F, D9(*cells.reshape(-1)), D9(*invs.reshape(-1)), I3(*cols["pbc"]),
                                                  I3(*cols["nb"]), I3(*cols["sr"]), D3(*cols["lo"]),
                                                  D3(*cols["width"]), self.r_max, D3(*pad), (C.c_int * F)(*self._caps),
                                                  D3(*perp), block), "nqb_nl_frames_pack_capacity")
        return block

    def set_cell(self, cell) -> None:
        """Make the following ``run`` calls (and replays of graphs that captured them) use ``cell`` ([3,3] or
        [1,3,3], rows = lattice vectors).  A host call, not captured: it computes the inverse (as ``neighbor_list``
        does), the search range on the plan's bin grid and the null-edge shift of this cell, packs them and copies the
        block to the device asynchronously on the current stream, after the previous copy out of the staging block
        has finished.  A CUDA ``cell`` costs one device-to-host read.  After ``set_cell(c)``, ``run(pos)`` holds the
        rows of ``neighbor_list(pos, c)`` bit for bit.  Raises ``ValueError`` for a wrong shape, a non-finite or
        singular cell and on a plan built without ``variable_cell``."""
        if not self.variable_cell:
            raise ValueError("NeighborListPlan.set_cell needs a plan built with variable_cell=True")
        if self._fr is not None:
            self._set_cells(cell)
            return
        a, pad_shift, block = _nl_cell_block(cell, self.r_max, self.nbins, self.num_atoms)
        if self._params_event is not None:
            self._params_event.synchronize()
        C.memmove(self._params_host.data_ptr(), block, len(block))
        with torch.cuda.device(self.device):
            self._params_dev.copy_(self._params_host, non_blocking=True)
            self._params_event = torch.cuda.Event()
            self._params_event.record()
        self._a, self.pad_shift = a, pad_shift

    def _set_cells(self, cell) -> None:
        """``set_cell`` of a batched plan: cells [F, 3, 3], each finite and non-singular; every frame's inverse,
        search range on its fixed grid and null-edge shift, one pack of all blocks and one asynchronous copy from
        pinned staging."""
        import numpy as np

        c = cell.detach().cpu().double().numpy() if torch.is_tensor(cell) else np.asarray(cell, dtype=np.float64)
        if c.shape != (self.num_frames, 3, 3):
            raise ValueError(f"set_cell: cell must be [{self.num_frames}, 3, 3], got {tuple(c.shape)}")
        cells = np.stack([_nl_check_cell(c[f], "set_cell") for f in range(self.num_frames)])
        block = self._pack_frames(cells, np.linalg.inv(cells))
        if self._params_event is not None:
            self._params_event.synchronize()
        C.memmove(self._params_host.data_ptr(), block, len(block))
        with torch.cuda.device(self.device):
            self._params_dev.copy_(self._params_host, non_blocking=True)
            self._params_event = torch.cuda.Event()
            self._params_event.record()

    def set_cell_device(self, cells: torch.Tensor) -> torch.Tensor:
        """``set_cell`` of a batched variable-cell plan from device cells [F, 3, 3] (float64, on the plan's device),
        packed on the device (``nqb_nl_frames_set_cells``, one thread per frame): a stream-ordered launch with no host
        synchronisation, so it can be captured together with ``run`` and the cells can move inside a CUDA graph.
        Each frame's cell, inverse, search range on its fixed grid and null-edge shift are those of the host pack (the
        inverse to a few ulp); the host copy ``pad_shift`` is not updated.  A frame whose cell is non-finite or
        singular keeps its previous parameters and gets ``cell_error[f] = 1``; ``cell_error`` [F] int32 is returned,
        and only the caller clears it.  ``ValueError`` on a plan without ``batch`` and ``variable_cell``, or for cells
        of another shape, dtype or device."""
        if self._fr is None or not self.variable_cell:
            raise ValueError("NeighborListPlan.set_cell_device needs a plan built with batch= and variable_cell=True")
        if (not torch.is_tensor(cells) or tuple(cells.shape) != (self.num_frames, 3, 3)
                or cells.dtype != torch.float64 or not cells.is_cuda
                or (self.device.index is not None and cells.device.index != self.device.index)):
            raise ValueError(f"set_cell_device: cells must be float64 [{self.num_frames}, 3, 3] on {self.device}")
        cells = cells.contiguous()
        _capi.check(_capi.lib().nqb_nl_frames_set_cells(self.num_frames, _ptr(cells), _ptr(self._params_dev),
                                                        _ptr(self.cell_error), _stream()), "nqb_nl_frames_set_cells")
        return self.cell_error

    def _run_frames(self, pos: torch.Tensor) -> None:
        L = _capi.lib()
        s, ty, fr = self._s, self._ty, self._fr
        N, st = self.num_atoms, _stream()
        blocks = (_ptr(self._params_dev), _ptr(fr["frame"]), _ptr(fr["bin_base"]))
        types, rc2, T = (0, 0, 0) if ty is None else (_ptr(ty.types), _ptr(ty.rc2), ty.T)
        if self._open:
            _capi.check(L.nqb_nl_bbox_frames(_ptr(pos), self.num_frames, _ptr(fr["atom_ptr"]), _ptr(self._params_dev),
                                             st), "nqb_nl_bbox_frames")
        _capi.check(L.nqb_nl_bin_frames(_ptr(pos), N, *blocks, _ptr(s["wpos"]), _ptr(s["base"]), _ptr(s["binid"]),
                                        _ptr(s["cidx"]), st), "nqb_nl_bin_frames")
        torch.sort(s["binid"], stable=True, out=(s["sorted_bin"], s["order"]))
        torch.searchsorted(s["sorted_bin"], s["bins"], out=s["bin_start"])
        _capi.check(L.nqb_nl_count_frames(N, *blocks, _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["order"]),
                                          _ptr(s["bin_start"]), types, rc2, T, _ptr(s["counts"]), st),
                    "nqb_nl_count_frames")
        torch.cumsum(s["counts"], 0, out=s["row_ptr"][1:])
        _capi.check(L.nqb_nl_pad(N, self.capacity, _ptr(s["row_ptr"]), _ptr(self.row_ptr), _ptr(self.num_edges),
                                 _ptr(self.overflow), st), "nqb_nl_pad")
        _capi.check(L.nqb_nl_fill_capacity_frames(N, self.capacity, *blocks, _ptr(s["wpos"]), _ptr(s["cidx"]),
                                                  _ptr(s["base"]), _ptr(s["order"]), _ptr(s["bin_start"]),
                                                  _ptr(self.row_ptr), _ptr(self.overflow), types, rc2, T,
                                                  _ptr(self.edge_index), _ptr(self.edge_cell_shift), st),
                    "nqb_nl_fill_capacity_frames")

    def run(self, pos: torch.Tensor) -> Dict[str, torch.Tensor]:
        _require_cuda(pos)
        if tuple(pos.shape) != (self.num_atoms, 3):
            raise ValueError(f"NeighborListPlan: pos must be [{self.num_atoms}, 3], got {tuple(pos.shape)}")
        pos = pos.detach().double().contiguous()
        if self._fr is not None:
            self._run_frames(pos)
            for t in (self.edge_index, self.edge_cell_shift, self.row_ptr, self.num_edges, self.overflow):
                torch.autograd.graph.increment_version(t)
            return {"edge_index": self.edge_index, "edge_cell_shift": self.edge_cell_shift, "row_ptr": self.row_ptr,
                    "num_edges": self.num_edges, "overflow": self.overflow}
        L = _capi.lib()
        a, s, ty = self._a, self._s, self._ty
        if self._open:
            _capi.check(L.nqb_nl_bbox(_ptr(pos), self.num_atoms, _ptr(self._params_dev), _ptr(self._bbox_work),
                                      _stream()), "nqb_nl_bbox")
        if ty is None:
            _nl_rows(pos, a, s, self._params_dev)
        else:
            _nl_rows(pos, a, s, self._params_dev, ty)
        st = _stream()
        _capi.check(L.nqb_nl_pad(self.num_atoms, self.capacity, _ptr(s["row_ptr"]), _ptr(self.row_ptr),
                                 _ptr(self.num_edges), _ptr(self.overflow), st), "nqb_nl_pad")
        if ty is not None and self._params_dev is not None:
            _capi.check(L.nqb_nl_fill_capacity_dp_typed(self.num_atoms, self.capacity, _ptr(self._params_dev),
                                                        _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["base"]),
                                                        _ptr(s["order"]), _ptr(s["bin_start"]), _ptr(self.row_ptr),
                                                        _ptr(self.overflow), _ptr(ty.types), _ptr(ty.rc2), ty.T,
                                                        _ptr(self.edge_index), _ptr(self.edge_cell_shift), st),
                        "nqb_nl_fill_capacity_dp_typed")
        elif ty is not None:
            _capi.check(L.nqb_nl_fill_capacity_typed(self.num_atoms, self.capacity, a.cell, a.inv, a.pbc, a.nb, a.sr,
                                                     a.r_max, _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["base"]),
                                                     _ptr(s["order"]), _ptr(s["bin_start"]), _ptr(self.row_ptr),
                                                     _ptr(self.overflow), self._pad_shift_c, _ptr(ty.types),
                                                     _ptr(ty.rc2), ty.T, _ptr(self.edge_index),
                                                     _ptr(self.edge_cell_shift), st),
                        "nqb_nl_fill_capacity_typed")
        elif self._params_dev is not None:
            _capi.check(L.nqb_nl_fill_capacity_dp(self.num_atoms, self.capacity, _ptr(self._params_dev),
                                                  _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["base"]), _ptr(s["order"]),
                                                  _ptr(s["bin_start"]), _ptr(self.row_ptr), _ptr(self.overflow),
                                                  _ptr(self.edge_index), _ptr(self.edge_cell_shift), st),
                        "nqb_nl_fill_capacity_dp")
        else:
            _capi.check(L.nqb_nl_fill_capacity(self.num_atoms, self.capacity, a.cell, a.inv, a.pbc, a.nb, a.sr, a.r_max,
                                               _ptr(s["wpos"]), _ptr(s["cidx"]), _ptr(s["base"]), _ptr(s["order"]),
                                               _ptr(s["bin_start"]), _ptr(self.row_ptr), _ptr(self.overflow),
                                               self._pad_shift_c, _ptr(self.edge_index), _ptr(self.edge_cell_shift),
                                               st),
                        "nqb_nl_fill_capacity")
        # the kernels write through raw pointers: bump the version counters so that the CSRs cached against these
        # buffers (csr_cache, src_csr_cache) are rebuilt for the new list
        for t in (self.edge_index, self.edge_cell_shift, self.row_ptr, self.num_edges, self.overflow):
            torch.autograd.graph.increment_version(t)
        return {"edge_index": self.edge_index, "edge_cell_shift": self.edge_cell_shift, "row_ptr": self.row_ptr,
                "num_edges": self.num_edges, "overflow": self.overflow}
