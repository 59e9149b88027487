#!/usr/bin/env python
"""Time the grouped 3xTF32 GEMM on the dense shapes of the Li3PO4 workload vs cuBLAS fp32."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nequip_b200 import ops  # noqa: E402


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


def main():
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--cases", default="")
    ap.add_argument("--no-cublas", action="store_true")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
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
        print(json.dumps({"case": name, "M": M, "K": K, "N": N, "ms": round(ms, 4), "cublas_fp32_ms": round(ms_t, 4),
                          "TFLOPs_fp32_equiv": round(2.0 * M * K * N / ms / 1e9, 1),
                          "io_GBps": round((M * K + M * N) * 4 / ms / 1e6, 1), "rel_err": err}), flush=True)
        del A, B, C


if __name__ == "__main__":
    main()
