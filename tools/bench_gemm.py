#!/usr/bin/env python
"""Time the grouped 3xTF32 GEMM on the dense shapes of the Li3PO4 workload vs cuBLAS fp32.

``--against PATH`` compares with a second build of the runtime library (for example the parent commit's
``libnqb.so`` built into a directory of its own): for every case both libraries run the same descriptors and
buffers alternately, every round's time is printed, and the outputs of the plain, row-scaled, accumulate,
``silu_save`` and ``silu_grad`` problems must be bit-identical.  The first line names the GPU, its power limit and
its maximum SM clock."""
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nequip_b200 import _capi, ops  # noqa: E402

MODES = {"plain": {}, "row_scaled": {"rs_off": 0}, "accumulate": {"accumulate": True}, "silu_save": {"act": "silu_save"},
         "silu_grad": {"act": "silu_grad"}}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    dev = torch.cuda.current_device()
    rows = [r.split(", ") for r in q.stdout.strip().splitlines()] if q.returncode == 0 else []
    row = next((r for r in rows if r and r[0] == str(dev)), None)
    return {"kind": "gpu", "name": torch.cuda.get_device_name(dev),
            "power_limit": row[2] if row else "not read", "max_sm_clock": row[3] if row else "not read"}


def timeit(fn, reps=8, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def load_other(path):
    """A second build of the runtime library, with the GEMM entry points typed like the first one's."""
    L = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    for name in ("nqb_gemm_prepare", "nqb_gemm_grouped", "nqb_gemm_grouped_act"):
        fn = getattr(L, name)
        fn.restype, fn.argtypes = _capi.SIGNATURES[name]
    return L


def run_other(L, gg, a, c, M, rowscale=None, aux=None):
    """``GroupedGemm.run`` on the other library: the same descriptors, prepared weights and buffers."""
    p = ops._ptr
    head = (p(gg.descs), gg.ndesc, gg.ntiles_total, p(gg.tile_ctas), int(gg.sched_ctas), p(a), p(gg.prepared), p(c),
            p(rowscale), int(rowscale.shape[-1]) if rowscale is not None else 0, int(M))
    if gg.act:
        rc = L.nqb_gemm_grouped_act(*head, p(c if aux is None else aux), ops._stream())
    else:
        rc = L.nqb_gemm_grouped(*head, ops._stream())
    if rc != 0:
        raise RuntimeError(f"--against library: GEMM launch failed (rc={rc})")


def compare_modes(L, name, A, B, M, K, N, g):
    """Both libraries on the same inputs, once per store mode: full-output bit equality."""
    out = {}
    rowscale = torch.randn(1, M, device="cuda", generator=g)
    rowscale[0, ::7] = 0.0
    for mode, kw in MODES.items():
        gg = ops.GroupedGemm([ops.GemmProblem(0, K, 0, N, B, **kw)], "cuda")
        prep = torch.empty_like(gg.prepared)
        rc = L.nqb_gemm_prepare(ops._ptr(B), B.shape[1], K, N, 0, 1.0, ops._ptr(prep), ops._stream())
        if rc != 0 or not torch.equal(prep, gg.prepared):
            raise AssertionError(f"{name}: the two libraries prepare different weights")
        del prep
        rs = rowscale if "rs_off" in kw else None
        c0 = torch.randn(M, N, device="cuda", generator=g)  # what "accumulate" adds to
        x0 = torch.randn(M, N, device="cuda", generator=g) if "act" in kw else None  # silu_grad reads it
        res = []
        for other in (False, True):
            c, x = c0.clone(), (x0.clone() if x0 is not None else None)
            if other:
                run_other(L, gg, A, c, M, rs, x)
            else:
                gg.run(A, c, M, rowscale=rs, aux=x)
            torch.cuda.synchronize()
            res.append((c, x))
        same = torch.equal(res[0][0], res[1][0]) and (x0 is None or torch.equal(res[0][1], res[1][1]))
        if not same:
            raise AssertionError(f"{name} / {mode}: outputs of the two libraries differ")
        out[mode] = same
        del res, c0, x0
    return out


def main():
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--cases", default="")
    ap.add_argument("--no-cublas", action="store_true")
    ap.add_argument("--against", default="", metavar="PATH", help="a second libnqb.so to alternate with and compare to")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if args.against and args.rounds < 5:
        ap.error("--against: at least 5 rounds")
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(gpu_info()), flush=True)
    other = load_other(args.against) if args.against else None
    E, Nat = int(588616 * args.scale), int(10648 * args.scale)
    g = torch.Generator(device="cuda").manual_seed(0)
    for (name, M, K, N) in [("mlp_fwd_L2", E, 128, 1728), ("mlp_bwd_L2", E, 1728, 128), ("mlp_fwd_L1", E, 128, 960),
                            ("mlp_fwd_L0", E, 128, 192), ("lin2_2e", Nat * 5, 384, 64), ("lin_sq", Nat, 1088, 1408)]:
        if args.cases and name not in args.cases.split(","):
            continue
        A = torch.randn(M, K, device="cuda", generator=g)
        B = torch.randn(K, N, device="cuda", generator=g)
        C = torch.empty(M, N, device="cuda")
        gg = ops.GroupedGemm([ops.GemmProblem(0, K, 0, N, B)], "cuda")
        ms = timeit(lambda: gg.run(A, C, M))
        ref = A[:4096].double() @ B.double()
        err = float((C[:4096].double() - ref).abs().max() / ref.abs().max())
        ms_t = 0.0 if args.no_cublas else timeit(lambda: torch.mm(A, B, out=C), reps=3, warm=1)
        line = {"case": name, "M": M, "K": K, "N": N, "ms": round(ms, 4), "cublas_fp32_ms": round(ms_t, 4),
                "TFLOPs_fp32_equiv": round(2.0 * M * K * N / ms / 1e9, 1),
                "io_GBps": round((M * K + M * N) * 4 / ms / 1e6, 1), "rel_err": err}
        if other is not None:
            new_ms, old_ms = [], []
            for _ in range(args.rounds):  # A B A B ...: 20 launches of each library a round
                new_ms.append(round(timeit(lambda: gg.run(A, C, M), reps=20, warm=1), 4))
                old_ms.append(round(timeit(lambda: run_other(other, gg, A, C, M), reps=20, warm=1), 4))
            line.update({"ms_rounds": new_ms, "against_ms_rounds": old_ms,
                         "speedup_worst_round": round(min(o / n for o, n in zip(old_ms, new_ms)), 3),
                         "bit_identical": compare_modes(other, name, A, B, M, K, N, g)})
        print(json.dumps(line), flush=True)
        del A, B, C
    return 0


if __name__ == "__main__":
    sys.exit(main())
