"""Write contracts of every kernel (include/nqb.h), checked with guarded buffers (tests/kernel_contracts.py).

Each output lives in a flat allocation with NaN sentinels before it, after it and between its rows; its body holds a
poison NaN where the kernel promises to write every element, a random finite base where it accumulates, and the data
for inputs (which are guarded too, so that reading past an input shows as NaN in an output).  References are float64:
the CPU oracle or torch.  The TP tolerances are those of test_tp_scatter_gpu.py; the others are per element.
"""
import math

import pytest
import torch

import kernel_contracts as kc
from kernel_contracts import Guarded, assert_elementwise
from nequip_b200 import _capi
from nequip_b200 import data as D
from nequip_b200 import known_signatures as ks
from nequip_b200 import ops
from nequip_b200.codegen import GenOptions, TPGenerator, TPSignature
from nequip_b200.irreps import Irreps, mul_ir_to_ir_mul
from oracle import irreps as OI
from oracle import model as omodel
from oracle import sh as osh
from oracle import tp as otp

pytestmark = pytest.mark.gpu

F32, F64 = torch.float32, torch.float64
DT = {F32: 0, F64: 1}
P = ops._ptr


def _L():
    return _capi.lib()


def _st():
    return ops._stream()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _data(t, dtype=None, ld=None):
    """A guarded input holding ``t``."""
    t = t if dtype is None else t.to(dtype)
    return Guarded(t.shape[0], t.shape[1], t.dtype, ld=ld, body=t)


# ---------------------------------------------------------------------------------------------------------------
# a. nqb_gemm_grouped
# ---------------------------------------------------------------------------------------------------------------
def _gemm_ref(A, B, scale=1.0, rs=None):
    r = A.double() @ B.double() * scale
    return r if rs is None else r * rs.double().unsqueeze(1)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("M,K,N", kc.GEMM_SHAPES, ids=lambda v: str(v))
def test_gemm_shapes_store_and_accumulate(M, K, N):
    """Plain store into a poisoned C (fully overwritten) and accumulation onto a random base, with A strided
    (lda = K + 8: NaN sentinels in columns [K, lda) and in the rows past M)."""
    A, B = kc.gemm_operands(M, K, N, seed=M * 7 + K * 3 + N)
    ga = _data(A, ld=K + 8)
    # plain store
    gc = Guarded(M, N, F32)
    # one problem: the even split, or the weighted one when a ragged last N-tile makes the tile costs differ
    gg = ops.GroupedGemm([ops.GemmProblem(0, K + 8, 0, N, B, scale=0.37)], "cuda")
    gg.run(ga.view, gc.view, M)
    torch.cuda.synchronize()
    ga.check_guards("A")
    gc.check_guards("C")
    ref = _gemm_ref(A, B, 0.37)
    assert_elementwise(gc.view, ref, kc.gemm_bound(A, B, 0.37, ref=ref), f"C = A @ B {(M, K, N)}")
    # accumulate onto a random base, C strided
    gb = Guarded(M, N, F32, ld=N + 4, body="random", generator=torch.Generator().manual_seed(M + N))
    base = gb.initial.double()
    gg2 = ops.GroupedGemm([ops.GemmProblem(0, K + 8, 0, N + 4, B, accumulate=True)], "cuda")
    gg2.run(ga.view, gb.view, M)
    torch.cuda.synchronize()
    gb.check_guards("C (accumulate)")
    ref2 = base + _gemm_ref(A, B)
    assert_elementwise(gb.view, ref2, kc.gemm_bound(A, B, ref=ref2), f"C += A @ B {(M, K, N)}")


def test_gemm_shapes_include_launches_smaller_and_larger_than_the_device():
    nwork = [-(-M // 128) * -(-N // 128) for M, _K, N in kc.GEMM_SHAPES]
    assert min(nwork) < _sms() < max(nwork)


@pytest.mark.timeout(300)
def test_gemm_weighted_split_mixing_resident_and_streamed():
    """Problems whose costs differ by >= 1.3x get the cost-weighted split; one is resident (K <= 128), one streamed."""
    M = 1000
    g = torch.Generator().manual_seed(1)
    A = torch.randn(M, 644, generator=g)
    B1, B2 = torch.randn(64, 128, generator=g), torch.randn(644, 260, generator=g)
    ga = _data(A)
    gc = Guarded(M, 388, F32)
    gg = ops.GroupedGemm([ops.GemmProblem(0, 644, 0, 388, B1), ops.GemmProblem(0, 644, 128, 388, B2)], "cuda")
    assert gg.tile_ctas is not None and gg.sched_ctas <= _sms()
    gg.run(ga.view, gc.view, M)
    torch.cuda.synchronize()
    ga.check_guards("A")
    gc.check_guards("C")
    ref = torch.cat([_gemm_ref(A[:, :64], B1), _gemm_ref(A, B2)], 1)
    bound = torch.cat([kc.gemm_bound(A[:, :64], B1), kc.gemm_bound(A, B2)], 1) + 2.0 ** -23 * ref.abs()
    assert_elementwise(gc.view, ref, bound, "weighted split")


@pytest.mark.timeout(300)
def test_gemm_more_n_tiles_than_sms_and_cta_moving_from_resident_to_streamed():
    """T > #SMs: CTA b owns N-tiles b, b + G, ...; the launch holds a resident (K = 128) and a streamed (K = 324)
    problem of 68 tiles each, so the CTAs that own two tiles move from the first to the second."""
    M, T = 129, 68
    g = torch.Generator().manual_seed(2)
    A = torch.randn(M, 324, generator=g)
    B1, B2 = torch.randn(128, T * 128, generator=g), torch.randn(324, T * 128 - 4, generator=g)
    ldc = 2 * T * 128
    ga = _data(A)
    gc = Guarded(M, ldc - 4, F32, ld=ldc)
    gg = ops.GroupedGemm([ops.GemmProblem(0, 324, 0, ldc, B1), ops.GemmProblem(0, 324, T * 128, ldc, B2)], "cuda")
    assert gg.ntiles_total > _sms() and gg.tile_ctas is None
    gg.run(ga.view, gc.view, M)
    torch.cuda.synchronize()
    ga.check_guards("A")
    gc.check_guards("C")
    ref = torch.cat([_gemm_ref(A[:, :128], B1), _gemm_ref(A, B2)], 1)
    bound = torch.cat([kc.gemm_bound(A[:, :128], B1), kc.gemm_bound(A, B2)], 1) + 2.0 ** -23 * ref.abs()
    assert_elementwise(gc.view, ref, bound, "T > SMs, resident then streamed")
    # one wide problem: 134 N-tiles with a ragged last one
    N = 133 * 128 + 60
    B = torch.randn(36, N, generator=g)
    A2 = torch.randn(65, 36, generator=g)
    ga2, gc2 = _data(A2), Guarded(65, N, F32)
    gg2 = ops.GroupedGemm([ops.GemmProblem(0, 36, 0, N, B)], "cuda")
    assert gg2.ntiles_total > _sms()
    gg2.run(ga2.view, gc2.view, 65)
    torch.cuda.synchronize()
    gc2.check_guards("C")
    ref2 = _gemm_ref(A2, B)
    assert_elementwise(gc2.view, ref2, kc.gemm_bound(A2, B, ref=ref2), "134 N-tiles")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("K", [36, 324])
def test_gemm_offsets_and_column_slice_of_wider_c(K):
    """Nonzero a_off / c_off: A's data sits between poisoned columns of a wider buffer, C is a column slice of a
    wider poisoned buffer whose other columns must stay bitwise untouched."""
    M, N, a_off, c_off = 300, 132, 8, 12
    lda, ldc = a_off + K + 12, c_off + N + 20
    g = torch.Generator().manual_seed(K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    Afull = torch.full((M, lda), float("nan"))
    Afull[:, a_off:a_off + K] = A
    ga = Guarded(M, lda, F32, body=Afull)
    gc = Guarded(M, ldc, F32)
    ops.GroupedGemm([ops.GemmProblem(a_off, lda, c_off, ldc, B)], "cuda").run(ga.view, gc.view, M)
    torch.cuda.synchronize()
    ga.check_guards("A")
    gc.check_guards("C")
    C = gc.view.cpu()
    assert bool(kc.is_poison(C[:, :c_off]).all()) and bool(kc.is_poison(C[:, c_off + N:]).all())
    ref = _gemm_ref(A, B)
    assert_elementwise(C[:, c_off:c_off + N], ref, kc.gemm_bound(A, B, ref=ref), "C slice")


@pytest.mark.timeout(300)
def test_gemm_two_atomic_problems_into_the_same_columns():
    M, N = 777, 260
    g = torch.Generator().manual_seed(3)
    A = torch.randn(M, 64 + 132, generator=g)
    B1, B2 = torch.randn(64, N, generator=g), torch.randn(132, N, generator=g)
    ga = _data(A)
    gc = Guarded(M, N, F32, body="random", generator=g)
    base = gc.initial.double()
    gg = ops.GroupedGemm([ops.GemmProblem(0, 196, 0, N, B1, atomic=True),
                          ops.GemmProblem(64, 196, 0, N, B2, atomic=True, scale=-0.5)], "cuda")
    gg.run(ga.view, gc.view, M)
    torch.cuda.synchronize()
    gc.check_guards("C")
    ref = base + _gemm_ref(A[:, :64], B1) + _gemm_ref(A[:, 64:], B2, -0.5)
    bound = kc.gemm_bound(A[:, :64], B1) + kc.gemm_bound(A[:, 64:], B2, 0.5) + 2.0 ** -22 * ref.abs()
    assert_elementwise(gc.view, ref, bound, "two atomic writers")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("K", [64, 324])
def test_gemm_row_scale_and_skipped_zero_rows(K):
    """Row scales that are non-binary, negative and zero: with skip_zero_rows a zero-scale row stays bitwise poisoned
    (plain store) or bitwise equal to its base (accumulate); without it the row gets rowscale * (A @ B)."""
    M, N = 1031, 132
    g = torch.Generator().manual_seed(K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    rs = torch.randn(3, M, generator=g)
    rs[:, ::3] = 0.0
    rs[1, 1::7] = -2.5
    ga, grs = _data(A), _data(rs)
    # C columns [0, N): store, skip zero rows; [N, 2N): store; [2N, 3N): accumulate onto a base, skip zero rows
    base = torch.randn(M, N, generator=g)
    body = kc.poison_value(F32).expand(M, 3 * N).clone()
    body[:, 2 * N:] = base
    gc = Guarded(M, 3 * N, F32, body=body)
    probs = [ops.GemmProblem(0, K, 0, 3 * N, B, rs_off=0, skip_zero_rows=True),
             ops.GemmProblem(0, K, N, 3 * N, B, rs_off=1),
             ops.GemmProblem(0, K, 2 * N, 3 * N, B, rs_off=2, skip_zero_rows=True, accumulate=True)]
    ops.GroupedGemm(probs, "cuda").run(ga.view, gc.view, M, rowscale=grs.view)
    torch.cuda.synchronize()
    ga.check_guards("A")
    grs.check_guards("rowscale")
    gc.check_guards("C")
    C = gc.view.cpu()
    z0 = rs[0] == 0
    assert bool(kc.is_poison(C[z0, :N]).all()), "skip_zero_rows: a zero-scale row was written"
    r0 = _gemm_ref(A, B, rs=rs[0])
    assert_elementwise(C[~z0, :N], r0[~z0], kc.gemm_bound(A, B, rowscale=rs[0], ref=r0)[~z0], "rowscale + skip")
    r1 = _gemm_ref(A, B, rs=rs[1])
    assert_elementwise(C[:, N:2 * N], r1, kc.gemm_bound(A, B, rowscale=rs[1], ref=r1), "rowscale")
    z2 = rs[2] == 0
    assert torch.equal(C[z2, 2 * N:].view(torch.int32), base[z2].view(torch.int32))
    r2 = base.double() + _gemm_ref(A, B, rs=rs[2])
    assert_elementwise(C[:, 2 * N:], r2, kc.gemm_bound(A, B, rowscale=rs[2], ref=r2), "rowscale + skip, accumulate")


def test_gemm_m0_writes_nothing():
    g = torch.Generator().manual_seed(4)
    B = torch.randn(132, 60, generator=g)
    ga, gc = Guarded(0, 132, F32), Guarded(0, 60, F32)
    gg = ops.GroupedGemm([ops.GemmProblem(0, 132, 0, 60, B)], "cuda")
    gg.run(ga.view, gc.view, 0)
    # a real C, M = 0: untouched
    gc2 = Guarded(5, 60, F32)
    gg.run(_data(torch.randn(5, 132)).view, gc2.view, 0)
    torch.cuda.synchronize()
    gc.check_guards("C")
    gc2.check_guards("C")
    assert bool(kc.is_poison(gc2.view.cpu()).all())


def test_gemm_rejects_misaligned_bases():
    """The kernel stages A with 16-byte copies: a base that is not 16-byte aligned is an error, and nothing runs."""
    g = torch.Generator().manual_seed(5)
    B = torch.randn(32, 4, generator=g)
    gg = ops.GroupedGemm([ops.GemmProblem(0, 32, 0, 4, B)], "cuda")
    ga, gc = Guarded(9, 32, F32, body=torch.randn(9, 32)), Guarded(8, 8, F32)
    L = _L()
    for a_ptr, c_ptr in ((ga.view.data_ptr() + 4, gc.view.data_ptr()), (ga.view.data_ptr(), gc.view.data_ptr() + 8)):
        rc = L.nqb_gemm_grouped(P(gg.descs), gg.ndesc, gg.ntiles_total, None, 0, a_ptr, P(gg.prepared), c_ptr, None, 0,
                                8, _st())
        assert rc != 0 and b"16-byte aligned" in L.nqb_last_error()
    torch.cuda.synchronize()
    gc.check_guards("C")
    assert bool(kc.is_poison(gc.view.cpu()).all())


# ---------------------------------------------------------------------------------------------------------------
# b. nqb_tp_scatter_fwd / bwd and the deterministic backward
# ---------------------------------------------------------------------------------------------------------------
TOL = {F32: 1e-5, F64: 1e-10}


def _ir_str(irr):
    return "+".join(f"{m}x{ir.l}{'e' if ir.p == 1 else 'o'}" for m, ir in Irreps(irr))


def _unread(sig):
    return [i for i in range(len(sig.irreps_in1)) if i not in {p.i1 for p in sig.paths}]


def _unwritten_out_sig():
    try:
        sig = TPSignature(Irreps("8x0e+8x1o"), Irreps("1x0e+1x1o"), Irreps("8x0e+8x1o+8x2e"),
                          [(0, 0, 0), (1, 1, 0), (0, 1, 1)])
    except Exception:
        return None
    return sig if len(sig.written_outs) < len(sig.irreps_out) else None


def _tp_sigs():
    unread = [s for s in ks.all_known() if _unread(s)]
    assert len(unread) == 5
    sigs = {
        "register_l2f32": ks.nequip_layer_signatures(2, 32, 4)[1],
        "ring_l2f64": ks.nequip_layer_signatures(2, 64, 4)[1],
        "preset_M": ks.preset_layer_signatures("M")[1],
    }
    for s in unread:
        sigs["unread_" + "_".join(str(i) for i in _unread(s)) + f"_d{s.d_in}"] = s
    sigs["unwritten_out"] = _unwritten_out_sig()
    return sigs


TP_SIGS = _tp_sigs()


def _csr(dst, N):
    """(row_ptr, perm or None) of the destination CSR, on the host."""
    srt, perm = torch.sort(dst, stable=True)
    row_ptr = torch.searchsorted(srt, torch.arange(N + 1))
    return row_ptr, (None if bool((perm == torch.arange(dst.numel())).all()) else perm)


def _tp_oracle(sig, x, y, w, dst, src, gout, N):
    """float64 CPU oracle: out, grad_x, per-edge grad_x, grad_y, grad_w (mul_ir)."""
    ins = [(a, b, c, "uvu", True) for a, b, c in sig.instructions]
    xe = x[src].clone().requires_grad_(True)
    yo, wo = y.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ef = otp.tensor_product_uvu(xe, yo, wo, _ir_str(sig.irreps_in1), _ir_str(sig.irreps_in2),
                                _ir_str(sig.irreps_out), ins)
    out = otp.scatter_sum(ef, dst, N)
    if dst.numel() == 0:
        z = torch.zeros
        return out.detach(), z(N, sig.d_in, dtype=F64), z(0, sig.d_in, dtype=F64), y.clone(), w.clone()
    gxe, gy, gw = torch.autograd.grad(out, [xe, yo, wo], gout)
    gx = otp.scatter_sum(gxe, src, N)
    return out.detach(), gx, gxe, gy, gw


def _graph(kind, N, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "unsorted":
        E = 301
        dst, src = torch.randint(0, N, (E,), generator=g), torch.randint(0, N, (E,), generator=g)
    elif kind == "isolated_ends":  # nodes 0 and N-1 receive no edge; sorted
        E = 97
        dst = torch.sort(torch.randint(1, N - 1, (E,), generator=g)).values
        src = torch.randint(0, N, (E,), generator=g)
    elif kind == "single_node":
        dst = src = torch.zeros(5, dtype=torch.long)
    elif kind == "no_edges":
        dst = src = torch.zeros(0, dtype=torch.long)
    elif kind == "ring_degrees":  # around the ring capacity (RING_CAP = 256 edges staged per node)
        degs = torch.tensor([255, 0, 256, 257, 512, 513, 1])
        dst = torch.repeat_interleave(torch.arange(degs.numel()), degs)
        src = torch.randint(0, degs.numel(), (dst.numel(),), generator=g)
    else:
        raise ValueError(kind)
    return dst, src


GRAPHS = {"unsorted": 23, "isolated_ends": 40, "single_node": 1, "no_edges": 6}


def _tp_case(sig, dtype, layout, kind, N, seed):
    L, st = _L(), _st()
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, GenOptions(layout=layout))
    dst, src = _graph(kind, N, seed)
    E = dst.numel()
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(N, sig.d_in, generator=g, dtype=F64)
    y = torch.randn(E, sig.s_dim, generator=g, dtype=F64)
    w = torch.randn(E, sig.weight_numel, generator=g, dtype=F64)
    gout = torch.randn(N, sig.d_out, generator=g, dtype=F64)
    out_o, gx_o, gxe_o, gy_o, gw_o = _tp_oracle(sig, x, y, w, dst, src, gout, N)
    out_irr = sig.irreps_out.simplify()
    if layout == "ir_mul":
        to_in = lambda t: mul_ir_to_ir_mul(t, sig.irreps_in1)  # noqa: E731
        x_k, gout_k = to_in(x), mul_ir_to_ir_mul(gout, out_irr)
        out_o, gx_o, gxe_o = mul_ir_to_ir_mul(out_o, out_irr), to_in(gx_o), to_in(gxe_o)
    else:
        x_k, gout_k = x, gout
    tol = TOL[dtype]
    gtol = tol * (10 if dtype == F32 else 1)
    row_ptr, perm = _csr(dst, N)
    ins = {"x": _data(x_k, dtype), "y": _data(y, dtype), "w": _data(w, dtype), "gout": _data(gout_k, dtype),
           "row_ptr": _data(row_ptr.view(-1, 1)), "src": _data(src.view(-1, 1))}
    if perm is not None:
        ins["perm"] = _data(perm.view(-1, 1))
    pp = P(ins["perm"].view) if perm is not None else 0
    dt = DT[dtype]

    def close(got, ref, what, t):
        # atol relative to the largest reference element: nodes of degree 513 sum that many fp32 products
        a = t * max(1.0, float(ref.abs().max()) if ref.numel() else 1.0)
        torch.testing.assert_close(got.cpu().double(), ref, atol=a, rtol=t, msg=lambda m: f"{kind} {what}: {m}")

    # forward: out fully written (isolated nodes and E = 0 included)
    go = Guarded(N, sig.d_out, dtype)
    _capi.check(L.nqb_tp_scatter_fwd(plan.handle, dt, P(ins["x"].view), P(ins["y"].view), P(ins["w"].view),
                                     P(ins["row_ptr"].view), pp, P(ins["src"].view), N, E, P(go.view), st))
    torch.cuda.synchronize()
    go.check_guards("out")
    close(go.view, out_o, "out", tol)

    def bwd(det, want_x, gxg, gyg, gwg):
        _capi.check(L.nqb_tp_scatter_bwd(plan.handle, dt, P(ins["x"].view), P(ins["y"].view), P(ins["w"].view),
                                         P(ins["row_ptr"].view), pp, P(ins["src"].view), P(ins["gout"].view), N, E,
                                         P(gxg.view) if want_x else 0, P(gyg.view), P(gwg.view), det, st))
        torch.cuda.synchronize()
        for nm, b in (("grad_x", gxg), ("grad_y", gyg), ("grad_w", gwg)):
            if b is not None:
                b.check_guards(nm)

    # default backward: grad_x / grad_y accumulate onto a random base, grad_w fully written
    rg = torch.Generator().manual_seed(seed + 2)
    gx, gy = Guarded(N, sig.d_in, dtype, body="random", generator=rg), Guarded(E, sig.s_dim, dtype, body="random",
                                                                                generator=rg)
    gw = Guarded(E, sig.weight_numel, dtype)
    bwd(0, True, gx, gy, gw)
    close(gx.view, gx.initial.double() + gx_o, "grad_x (onto base)", gtol)
    close(gy.view, gy.initial.double() + gy_o, "grad_y (onto base)", gtol)
    close(gw.view, gw_o, "grad_w", gtol)
    # grad_x = NULL: grad_y and grad_w as with it
    gy2 = Guarded(E, sig.s_dim, dtype, body=gy.initial)
    gw2 = Guarded(E, sig.weight_numel, dtype)
    bwd(0, False, None, gy2, gw2)
    assert torch.equal(gw2.view.cpu(), gw.view.cpu()), "grad_w differs without grad_x"
    close(gy2.view, gy2.initial.double() + gy_o, "grad_y (grad_x = NULL)", gtol)
    if E == 0:
        assert torch.equal(gx.view.cpu(), gx.initial) and torch.equal(gy.view.cpu(), gy.initial)
        return

    # deterministic backward: the per-edge grad_x buffer is poisoned and must be fully written (zeros in unread
    # chunks), the grad_Y slices start zeroed; the segmented sum is checked against the oracle
    ns = int(L.nqb_tp_scatter_gy_slices(plan.handle, dt))
    assert ns > 0
    perm_t = torch.sort(src, stable=True).indices
    seg = torch.searchsorted(src[perm_t], torch.arange(N + 1))
    gperm, gseg = _data(perm_t.view(-1, 1)), _data(seg.view(-1, 1))
    runs = []
    for _ in range(2):
        gxe = Guarded(E, sig.d_in, dtype)
        gys = Guarded(ns * E, sig.s_dim, dtype, body=torch.zeros(ns * E, sig.s_dim, dtype=dtype))
        gwd = Guarded(E, sig.weight_numel, dtype)
        bwd(1, True, gxe, gys, gwd)
        gxs = Guarded(N, sig.d_in, dtype)
        _capi.check(L.nqb_segment_sum(dt, P(gxe.view), sig.d_in, P(gperm.view), P(gseg.view), N, P(gxs.view), st))
        torch.cuda.synchronize()
        gxs.check_guards("segment_sum out")
        gperm.check_guards("perm")
        runs.append([b.view.cpu() for b in (gxe, gys, gwd, gxs)])
    gxe_k, gys_k, gwd_k, gxs_k = runs[0]
    close(gxe_k, gxe_o, "per-edge grad_x (deterministic)", gtol)
    for i1 in _unread(sig):
        off, dim = sig.irreps_in1.offsets()[i1], sig.irreps_in1[i1][0] * sig.irreps_in1[i1][1].dim
        assert bool((gxe_k[:, off:off + dim] == 0).all()), f"unread chunk {i1}: per-edge grad_x not zero"
    gy_det = gys_k.view(ns, E, sig.s_dim).double().sum(0)
    close(gy_det, gy_o, "grad_y (deterministic)", gtol)
    close(gwd_k, gw_o, "grad_w (deterministic)", gtol)
    close(gxs_k, gx_o, "grad_x = segment_sum (deterministic)", gtol)
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "deterministic backward is not repeatable"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", list(TP_SIGS))
def test_tp_scatter_write_contracts(name, dtype, layout):
    sig = TP_SIGS[name]
    if sig is None:
        pytest.skip("TPSignature rejects an irreps_out entry that no instruction writes")
    for i, (kind, N) in enumerate(GRAPHS.items()):
        _tp_case(sig, dtype, layout, kind, N, seed=17 * i + len(name))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_tp_scatter_degrees_around_the_ring_capacity(dtype, layout):
    sig = TP_SIGS["ring_l2f64"]
    assert TPGenerator(sig, GenOptions(layout=layout)).use_ring or layout == "mul_ir"
    _tp_case(sig, dtype, layout, "ring_degrees", 7, seed=5)


# ---------------------------------------------------------------------------------------------------------------
# c. deterministic energy and forces of a model whose last layer has unread input chunks
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_deterministic_forces_match_oracle_with_nan_filled_allocator():
    from nequip_b200.nn.model import NequIPEnergyModel

    torch.backends.cuda.matmul.allow_tf32 = False
    sysd = D.make_system("li3po4", 5, r_max=5.0, seed=0)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=5.0, type_names=meta["type_names"], l_max=2, num_layers=4, num_features=64,
                              radial_mlp_depth=1, radial_mlp_width=128, avg_num_neighbors=meta["avg_num_neighbors"],
                              strict_fast_path=True).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    assert _unread(ks.nequip_layer_signatures(2, 64, 4)[-1])
    dev = D.to_device(sysd, "cuda")
    # what the caching allocator hands out next is NaN unless a kernel writes it
    junk = torch.empty(1 << 29, dtype=F32, device="cuda")
    junk.fill_(float("nan"))
    del junk
    prev = ops._DETERMINISTIC
    ops.set_deterministic(True)
    try:
        outs = []
        for _ in range(2):
            o = model(dev)
            outs.append((o["total_energy"].detach().cpu(), o["forces"].detach().cpu()))
    finally:
        ops.set_deterministic(prev)
    e_ref, ea_ref, f_ref = omodel.energy_and_forces(model.state_dict(), model.config, sysd, F32)
    e, f = outs[0]
    assert bool(torch.isfinite(f).all()), "deterministic forces hold NaN"
    assert abs(float(e) - float(e_ref)) <= 1e-5 * float(ea_ref.abs().sum()), (float(e), float(e_ref))
    ferr = float((f - f_ref).abs().max()) / float(f_ref.abs().max())
    assert ferr <= 1e-5, ferr
    # the energy is bitwise repeatable; the forces are not, to the last bit: the edge-embedding backward scatters
    # grad_pos with float64 atomics, which the deterministic mode does not cover
    assert torch.equal(outs[0][0], outs[1][0])
    assert float((outs[0][1] - outs[1][1]).abs().max()) <= 1e-12 * float(f_ref.abs().max())


# ---------------------------------------------------------------------------------------------------------------
# d. nqb_tp_fused_fwd
# ---------------------------------------------------------------------------------------------------------------
FUSED_DEGS = [0, 1, 63, 64, 65, 127, 128, 129]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("K", [8, 16, 40, 64, 120, 128])
def test_tp_fused_write_contracts(K):
    sig = ks.nequip_layer_signatures(2, 64, 4)[1]
    opts = GenOptions(layout="ir_mul")
    assert TPGenerator(sig, opts).fused_layout() is not None
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, opts)
    g = torch.Generator().manual_seed(K)
    W2 = (torch.rand(K, sig.weight_numel, generator=g) * 2 - 1) * math.sqrt(3)
    a2 = math.sqrt(2) / math.sqrt(K)
    fw = ops.FusedTPWeights(plan, W2.cuda(), a2, "cuda")
    graphs = [("degrees", torch.repeat_interleave(torch.arange(len(FUSED_DEGS)), torch.tensor(FUSED_DEGS))),
              ("no_edges", torch.zeros(0, dtype=torch.long))]
    if K == 64:
        degs = torch.randint(0, 7, (3001,), generator=g)
        graphs.append(("3001_nodes", torch.repeat_interleave(torch.arange(3001), degs)))
    for name, dst in graphs:
        N = {"degrees": len(FUSED_DEGS), "no_edges": 5, "3001_nodes": 3001}[name]
        E = dst.numel()
        src = torch.randint(0, N, (E,), generator=g)
        x = torch.randn(N, sig.d_in, generator=g, dtype=F64)
        y = torch.randn(E, sig.s_dim, generator=g, dtype=F64)
        h = torch.randn(E, K, generator=g).float()
        gx, gy = _data(mul_ir_to_ir_mul(x, sig.irreps_in1), F32), _data(y, F32)
        gh = Guarded(E, K, F32, ld=K + 8, body=h)
        row_ptr, perm = _csr(dst, N)
        assert perm is None
        grp, gsrc = _data(row_ptr.view(-1, 1)), _data(src.view(-1, 1))
        gout = Guarded(N, sig.d_out, F32)
        gwo = Guarded(E, sig.weight_numel, F32)
        _capi.check(_L().nqb_tp_fused_fwd(plan.handle, P(gx.view), P(gy.view), P(gh.view), K + 8, K, P(fw.prepared),
                                          P(grp.view), P(gsrc.view), N, E, P(gout.view), P(gwo.view),
                                          P(fw.cta0_dev), int(fw.nctas), _st()))
        torch.cuda.synchronize()
        for nm, b in (("x", gx), ("y", gy), ("h", gh), ("out", gout), ("w_out", gwo)):
            b.check_guards(f"{name}: {nm}")
        W2s = W2.double() * a2
        w_ref = h.double() @ W2s
        assert_elementwise(gwo.view, w_ref, 2 * kc.gemm_bound(h, W2s, ref=w_ref), f"{name}: w_out")
        out_o, *_ = _tp_oracle(sig, x, y, w_ref, dst, src, torch.zeros(N, sig.d_out, dtype=F64), N)
        out_o = mul_ir_to_ir_mul(out_o, sig.irreps_out.simplify())
        bound = 3e-6 * max(float(out_o.abs().max()), 1e-30)
        assert_elementwise(gout.view, out_o, bound, f"{name}: out")


def test_tp_fused_rejects_misaligned_h():
    sig = ks.nequip_layer_signatures(2, 64, 4)[1]
    opts = GenOptions(layout="ir_mul")
    plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, opts)
    fw = ops.FusedTPWeights(plan, torch.randn(8, sig.weight_numel, device="cuda"), 1.0, "cuda")
    gx, gy = Guarded(2, sig.d_in, F32, body=torch.zeros(2, sig.d_in)), Guarded(2, sig.s_dim, F32,
                                                                                body=torch.zeros(2, sig.s_dim))
    gh = Guarded(3, 12, F32, body=torch.zeros(3, 12))
    rp, src = torch.tensor([0, 1, 2], device="cuda"), torch.tensor([0, 1], device="cuda")
    gout = Guarded(2, sig.d_out, F32)
    L = _L()
    rc = L.nqb_tp_fused_fwd(plan.handle, P(gx.view), P(gy.view), gh.view.data_ptr() + 4, 12, 8, P(fw.prepared), P(rp),
                            P(src), 2, 2, P(gout.view), 0, P(fw.cta0_dev), int(fw.nctas), _st())
    assert rc != 0 and b"16-byte aligned" in L.nqb_last_error()
    torch.cuda.synchronize()
    gout.check_guards("out")
    assert bool(kc.is_poison(gout.view.cpu()).all())


# ---------------------------------------------------------------------------------------------------------------
# e. small kernels
# ---------------------------------------------------------------------------------------------------------------
GATE = ("16x0e+8x0o", "8x0e+8x0o", "4x1o+4x1e+8x2e")


@pytest.mark.parametrize("layout", ["mul_ir", "ir_mul"])
@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
def test_gate_write_contracts(dtype, layout):
    sc, ga, gd = GATE
    tabs = ops.GateTables(sc, ga, gd, layout, "cuda")
    N = 257
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, tabs.d_in, generator=g, dtype=F64) * 3
    if dtype == F32:
        x[::5, :] = 100.0
        x[1::5, :] = -100.0
    gout = torch.randn(N, tabs.d_out, generator=g, dtype=F64)
    x, gout = x.to(dtype).double(), gout.to(dtype).double()  # the kernel sees exactly the reference's inputs
    in_irr, out_irr = Irreps(sc) + Irreps(ga) + Irreps(gd), Irreps(sc) + Irreps(gd)
    xo = x.clone().requires_grad_(True)
    out_o = omodel.gate(xo, OI.parse(sc), OI.parse(ga), OI.parse(gd))
    (gx_o,) = torch.autograd.grad(out_o, xo, gout)
    out_o = out_o.detach()
    if layout == "ir_mul":
        x_k, gout_k = mul_ir_to_ir_mul(x, in_irr), mul_ir_to_ir_mul(gout, out_irr)
        out_o, gx_o = mul_ir_to_ir_mul(out_o, out_irr), mul_ir_to_ir_mul(gx_o, in_irr)
    else:
        x_k, gout_k = x, gout
    gxin, ggo = _data(x_k, dtype), _data(gout_k, dtype)
    go, ggx = Guarded(N, tabs.d_out, dtype), Guarded(N, tabs.d_in, dtype)
    L, st, dt = _L(), _st(), DT[dtype]
    _capi.check(L.nqb_gate_fwd(dt, P(gxin.view), N, tabs.d_in, tabs.d_out, P(tabs.src), P(tabs.gate), P(tabs.kind),
                               P(go.view), st))
    _capi.check(L.nqb_gate_bwd(dt, P(gxin.view), P(ggo.view), N, tabs.d_in, tabs.d_out, P(tabs.tab), P(ggx.view), st))
    torch.cuda.synchronize()
    go.check_guards("out")
    ggx.check_guards("grad_x")
    t = 1e-6 if dtype == F32 else 1e-13
    assert_elementwise(go.view, out_o, t * (1 + out_o.abs()), "gate out")
    assert_elementwise(ggx.view, gx_o, t * (1 + gx_o.abs()) * 4, "gate grad_x")


def _edges(N, E, seed):
    g = torch.Generator().manual_seed(seed)
    pos = torch.rand(N, 3, generator=g, dtype=F64) * 6.0
    i = torch.randint(0, N, (E,), generator=g)
    j = (i + 1 + torch.randint(0, N - 1, (E,), generator=g)) % N
    return pos, torch.stack([i, j])


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("E", [1, 255, 256, 257])
def test_sh_and_edge_embed_write_contracts(E, dtype):
    L, st, dt = _L(), _st(), DT[dtype]
    N, lmax, nb, r_max, p = 30, 3, 8, 5.0, 6.0
    S = (lmax + 1) ** 2
    pos, ei = _edges(N, E, seed=E)
    g = torch.Generator().manual_seed(E + 1)
    gy = torch.randn(E, S, generator=g, dtype=F64).to(dtype).double()
    gemb = torch.randn(E, nb, generator=g, dtype=F64).to(dtype).double()
    t = 2e-6 if dtype == F32 else 1e-12
    # nqb_sh_fwd / bwd
    vec = pos[ei[1]] - pos[ei[0]]
    vo = vec.clone().requires_grad_(True)
    y_o = osh.spherical_harmonics(lmax, vo)
    (gv_o,) = torch.autograd.grad(y_o, vo, gy)
    gvec_in, gyv = _data(vec), _data(gy, dtype)
    gys, ggv = Guarded(E, S, dtype), Guarded(E, 3, F64)
    _capi.check(L.nqb_sh_fwd(lmax, P(gvec_in.view), E, dt, P(gys.view), st))
    _capi.check(L.nqb_sh_bwd(lmax, P(gvec_in.view), E, dt, P(gyv.view), P(ggv.view), st))
    torch.cuda.synchronize()
    gys.check_guards("sh y")
    ggv.check_guards("sh grad_vec")
    assert_elementwise(gys.view, y_o.detach(), t * (1 + y_o.detach().abs()), "sh y")
    assert_elementwise(ggv.view, gv_o, 10 * t * (1 + gv_o.abs()), "sh grad_vec")
    # nqb_edge_embed_fwd / bwd; E = 257 with a triclinic cell and integer shifts in -1..1 (the kernel's cell branch)
    cell = shift = None
    if E == 257:
        cell = torch.tensor([[3.1, 0.0, 0.0], [0.9, 2.8, 0.0], [-0.6, 0.7, 3.3]], dtype=F64)
        shift = torch.randint(-1, 2, (E, 3), generator=g).to(F64)
    pf = 2 * math.pi / r_max ** 2
    po = pos.clone().requires_grad_(True)
    vec_o, ye_o, emb_o = omodel.edge_embed(po, ei, cell, shift, lmax, nb, r_max, p, dtype)
    (gp_o,) = torch.autograd.grad([ye_o, emb_o], [po], [gy.to(dtype), gemb.to(dtype)])
    gpos, gei, ggy, gge = _data(pos), _data(ei), _data(gy, dtype), _data(gemb, dtype)
    gsh, gcell = (None, None) if cell is None else (_data(shift), _data(cell))
    gv, gye, gem = Guarded(E, 3, F64), Guarded(E, S, dtype), Guarded(E, nb, dtype)
    _capi.check(L.nqb_edge_embed_fwd(lmax, nb, r_max, p, pf, P(gpos.view), P(gei.view),
                                     0 if gsh is None else P(gsh.view), 0 if gcell is None else P(gcell.view), N, E,
                                     dt, P(gv.view), P(gye.view), P(gem.view), st))
    gp = Guarded(N, 3, F64, body="random", generator=g)
    gvo = Guarded(E, 3, F64)
    _capi.check(L.nqb_edge_embed_bwd(lmax, nb, r_max, p, pf, P(gv.view), P(gei.view), N, E, dt, P(ggy.view),
                                     P(gge.view), P(gp.view), P(gvo.view), st))
    torch.cuda.synchronize()
    for nm, b in (("vec", gv), ("y", gye), ("emb", gem), ("grad_pos", gp), ("grad_vec", gvo), ("pos", gpos)):
        b.check_guards(f"edge_embed {nm}")
    if cell is not None:
        gsh.check_guards("edge_embed shift")
        gcell.check_guards("edge_embed cell")
        r = vec_o.detach().norm(dim=1)
        assert int((shift != 0).any(1).sum()) > E // 2 and int((r < r_max).sum()) > E // 4
    assert_elementwise(gv.view, vec_o.detach(), 1e-13 * (1 + vec_o.detach().abs()), "edge vec")
    assert_elementwise(gye.view, ye_o.detach().double(), t * (1 + ye_o.detach().double().abs()), "edge y")
    assert_elementwise(gem.view, emb_o.detach().double(), t * (1 + emb_o.detach().double().abs()), "edge emb")
    scale = float(gp_o.abs().max())
    gt = (2e-5 if dtype == F32 else 1e-10) * scale
    assert_elementwise(gp.view, gp.initial + gp_o, gt + 1e-5 * gp_o.abs() + 2.0 ** -50 * gp.initial.abs(),
                       "grad_pos (onto base)")
    # grad_vec: the per-edge gradient, whose scatter is grad_pos
    gvec_k = gvo.view.cpu()
    gpos_from_vec = torch.zeros(N, 3, dtype=F64).index_add_(0, ei[1], gvec_k).index_add_(0, ei[0], -gvec_k)
    assert_elementwise(gpos_from_vec, gp_o, gt + 1e-5 * gp_o.abs(), "grad_vec scattered")


@pytest.mark.parametrize("case", ["gaps", "no_edges", "all_in_one"])
def test_csr_from_sorted_writes_every_entry(case):
    N = 12
    keys = {"gaps": torch.tensor([2, 2, 3, 7, 7, 7, 9]), "no_edges": torch.zeros(0, dtype=torch.long),
            "all_in_one": torch.full((5,), 4)}[case]
    E = keys.numel()
    gk = _data(keys.view(-1, 1)) if E else Guarded(0, 1, torch.int64)
    grp = Guarded(N + 1, 1, torch.int64)
    _capi.check(_L().nqb_csr_from_sorted(P(gk.view), E, N, P(grp.view), _st()))
    torch.cuda.synchronize()
    grp.check_guards("row_ptr")
    ref = torch.searchsorted(keys, torch.arange(N + 1))
    assert torch.equal(grp.view.cpu().view(-1), ref)


@pytest.mark.parametrize("dtype", [F32, F64], ids=["f32", "f64"])
@pytest.mark.parametrize("D", [1, 63, 64, 65, 129, 257])
def test_segment_sum_write_contracts(D, dtype):
    g = torch.Generator().manual_seed(D)
    N = 9
    cnt = torch.tensor([0, 3, 0, 1, 5, 0, 2, 7, 0])
    R = int(cnt.sum())
    rows = torch.randn(R, D, generator=g, dtype=F64)
    perm = torch.randperm(R, generator=g)
    seg = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(cnt, 0)])
    gr, gpm, gsg = _data(rows, dtype), _data(perm.view(-1, 1)), _data(seg.view(-1, 1))
    go = Guarded(N, D, dtype)
    _capi.check(_L().nqb_segment_sum(DT[dtype], P(gr.view), D, P(gpm.view), P(gsg.view), N, P(go.view), _st()))
    torch.cuda.synchronize()
    go.check_guards("out")
    rd = rows.to(dtype).double()
    ref = torch.stack([rd[perm[seg[n]:seg[n + 1]]].sum(0) for n in range(N)])
    eps = 2.0 ** -23 if dtype == F32 else 2.0 ** -52
    bound = 8 * eps * torch.stack([rd[perm[seg[n]:seg[n + 1]]].abs().sum(0) for n in range(N)])
    assert_elementwise(go.view, ref, bound, "segment_sum")
    assert bool((go.view.cpu()[cnt == 0] == 0).all())


@pytest.mark.parametrize("E", [1, 31, 32, 33, 4099])
def test_hidden_layer_guard_bands(E):
    g = torch.Generator().manual_seed(E)
    emb = torch.rand(E, 8, generator=g) * 2 - 0.5
    w1s = (torch.rand(8, 128, generator=g) * 2 - 1) * 0.6
    gh = torch.randn(E, 128, generator=g)
    e_r = emb.double().requires_grad_(True)
    h_ref = torch.nn.functional.silu(e_r @ w1s.double())
    (ge_ref,) = torch.autograd.grad(h_ref, e_r, gh.double())
    ge_, gw_, ggh = _data(emb), _data(w1s), _data(gh)
    gho, geo = Guarded(E, 128, F32), Guarded(E, 8, F32)
    ops.mlp_hidden_fwd(ge_.view, gw_.view, gho.view)
    ops.mlp_hidden_bwd(ge_.view, gw_.view, ggh.view, geo.view)
    torch.cuda.synchronize()
    gho.check_guards("h")
    geo.check_guards("grad_emb")
    torch.testing.assert_close(gho.view.cpu().double(), h_ref.detach(), atol=2e-6, rtol=2e-6)
    torch.testing.assert_close(geo.view.cpu().double(), ge_ref, atol=2e-5, rtol=2e-5)
