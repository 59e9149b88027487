#!/usr/bin/env python
"""Time generator variants (GenOptions) of the fused TP kernels on one workload's layer signatures.
`--build-only` compiles every variant (CPU box); on the GPU box the prebuilt libraries are timed."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nequip_b200 import build  # noqa: E402
from nequip_b200.codegen import GenOptions  # noqa: E402
from nequip_b200.known_signatures import nequip_layer_signatures  # noqa: E402

VARIANTS = {
    "irmul": GenOptions(layout="ir_mul"),
    "irmul_nobwdring": GenOptions(layout="ir_mul", bwd_ring=False),
    "irmul_b16": GenOptions(layout="ir_mul", acc_cap_bwd=16),
    "irmul_b32": GenOptions(layout="ir_mul", acc_cap_bwd=32),
    "irmul_st6": GenOptions(layout="ir_mul", ring_stages=6),
    "irmul_noring": GenOptions(layout="ir_mul", fwd_ring=False, bwd_ring=False),
    "irmul_noring_split": GenOptions(layout="ir_mul", fwd_ring=False, bwd_ring=False, split_groups=True),
    "irmul_noring_split_a16": GenOptions(layout="ir_mul", fwd_ring=False, bwd_ring=False, split_groups=True, acc_cap=16, acc_cap_bwd=16),
    "irmul_noring_split_a64": GenOptions(layout="ir_mul", fwd_ring=False, bwd_ring=False, split_groups=True, acc_cap=64, acc_cap_bwd=64),
    "irmul_ring_a16": GenOptions(layout="ir_mul", acc_cap=16, acc_cap_bwd=16),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="2,64,4")
    ap.add_argument("--layers", default="1,2,3")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--variants", default=",".join(VARIANTS))
    args = ap.parse_args()
    lm, nf, nl = map(int, args.cfg.split(","))
    sigs = nequip_layer_signatures(lm, nf, nl)
    layers = [int(x) for x in args.layers.split(",")]
    names = args.variants.split(",")
    todo = [(sigs[li], VARIANTS[v]) for li in layers for v in names]
    build.ensure_specs(todo)
    if args.build_only:
        print("built", len(todo))
        return
    from bench import H100_HBM_GBS, build_system, tp_algorithmic_bytes
    from nequip_b200 import ops

    peak = H100_HBM_GBS
    wl = {(2, 64): "li3po4_10k_l2_f64", (2, 32): "water_1k_l2_f32", (3, 32): "asi_50k_l3_f32"}[(lm, nf)]
    sysd, meta, mk = build_system(wl, seed=0)
    dev = torch.device("cuda")
    N, E = sysd["pos"].shape[0], sysd["edge_index"].shape[1]
    ei = sysd["edge_index"].to(dev)
    csr = ops.build_csr(ei[0].contiguous(), N)
    src = ei[1].contiguous()
    L = ops._capi.lib()
    g = torch.Generator(device=dev).manual_seed(0)

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

    for li in layers:
        sig = sigs[li]
        x = torch.randn(N, sig.d_in, device=dev, generator=g)
        y = torch.randn(E, sig.s_dim, device=dev, generator=g)
        w = torch.randn(E, sig.weight_numel, device=dev, generator=g)
        gout = torch.randn(N, sig.d_out, device=dev, generator=g)
        out = torch.empty(N, sig.d_out, device=dev)
        gx, gy, gw = torch.zeros_like(x), torch.zeros_like(y), torch.empty_like(w)
        st = torch.cuda.current_stream().cuda_stream
        ref_out = None
        for v in names:
            plan = ops.TPPlan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, VARIANTS[v])

            def fwd():
                ops._capi.check(L.nqb_tp_scatter_fwd(plan.handle, 0, x.data_ptr(), y.data_ptr(), w.data_ptr(), csr.row_ptr.data_ptr(),
                                                     0, src.data_ptr(), N, E, out.data_ptr(), st), "fwd")

            def bwd():
                ops._capi.check(L.nqb_tp_scatter_bwd(plan.handle, 0, x.data_ptr(), y.data_ptr(), w.data_ptr(), csr.row_ptr.data_ptr(),
                                                     0, src.data_ptr(), gout.data_ptr(), N, E, gx.data_ptr(), gy.data_ptr(),
                                                     gw.data_ptr(), 0, st), "bwd")

            tf, tb = timeit(fwd), timeit(bwd)
            if ref_out is None:
                ref_out = out.clone()
            dev_max = float((out - ref_out).abs().max())
            af, ab = tp_algorithmic_bytes(sig, N, E), tp_algorithmic_bytes(sig, N, E, backward=True)
            print(json.dumps({"layer": li, "variant": v, "fwd_ms": round(tf, 4), "fwd_frac": round(af / tf / 1e6 / peak, 3),
                              "bwd_ms": round(tb, 4), "bwd_frac": round(ab / tb / 1e6 / peak, 3), "dev_vs_first": dev_max}), flush=True)
        del x, y, w, gout, out, gx, gy, gw


if __name__ == "__main__":
    main()
