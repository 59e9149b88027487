#!/usr/bin/env python
"""Per-kernel timings (CUDA events) of the hot-path kernels for one workload: TP fwd/bwd per layer,
radial MLP fwd/bwd per layer, edge embedding.  Prints one JSON line per kernel."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench import H100_HBM_GBS, WORKLOADS, build_system, tp_algorithmic_bytes, R_MAX  # noqa: E402
from nequip_b200 import ops  # noqa: E402
from nequip_b200 import data as D  # noqa: E402
from nequip_b200.nn.model import NequIPEnergyModel, ScalarLinearLayer  # noqa: E402


def timeit(fn, reps=10, warm=3):
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
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="li3po4_10k_l2_f64")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-mlp", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda")
    peak, src = H100_HBM_GBS, "H100 SXM data sheet (HBM3)"
    sysd, meta, mk = build_system(args.workload, seed=0)
    N, E = sysd["pos"].shape[0], sysd["edge_index"].shape[1]
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], parity=True,
                              avg_num_neighbors=meta["avg_num_neighbors"], **mk).to(dev)
    ei = sysd["edge_index"].to(dev)
    csr = ops.build_csr(ei[0].contiguous(), N)
    src_idx = ei[1].contiguous()
    g = torch.Generator(device=dev).manual_seed(0)
    for li, layer in enumerate(model.layers):
        tps = layer.conv.tp_scatter
        sig = tps._plan.sig
        x = torch.randn(N, sig.d_in, device=dev, generator=g)
        y = torch.randn(E, sig.s_dim, device=dev, generator=g)
        w = torch.randn(E, sig.weight_numel, device=dev, generator=g)
        with torch.no_grad():
            ms = timeit(lambda: ops.tp_scatter(tps._plan, x, y, w, ei[0], src_idx, csr=csr), args.reps)
        alg = tp_algorithmic_bytes(sig, N, E)
        print(json.dumps({"kernel": "tp_fwd", "layer": li, "W": sig.weight_numel, "ms": round(ms, 4),
                          "alg_GB": round(alg / 1e9, 3), "GBps": round(alg / ms / 1e6, 1), "frac_hbm": round(alg / ms / 1e6 / peak, 3),
                          "fma_per_edge_ch": sig.fma_count()}))
        L = ops._capi.lib()
        gout = torch.randn(N, sig.d_out, device=dev, generator=g)
        for want_gx in ([False] if li == 0 else [True]):
            gx = torch.zeros_like(x) if want_gx else None
            gy = torch.zeros_like(y)
            gw = torch.empty_like(w)

            def bwd():
                ops._capi.check(L.nqb_tp_scatter_bwd(tps._plan.handle, 0, x.data_ptr(), y.data_ptr(), w.data_ptr(),
                                                     csr.row_ptr.data_ptr(), 0, src_idx.data_ptr(), gout.data_ptr(), N, E,
                                                     0 if gx is None else gx.data_ptr(), gy.data_ptr(), gw.data_ptr(), 0,
                                                     torch.cuda.current_stream().cuda_stream), "bwd")

            ms = timeit(bwd, args.reps)
            algb = tp_algorithmic_bytes(sig, N, E, backward=True)
            print(json.dumps({"kernel": "tp_bwd", "layer": li, "want_gx": want_gx, "ms": round(ms, 4),
                              "alg_GB": round(algb / 1e9, 3), "GBps": round(algb / ms / 1e6, 1),
                              "frac_hbm": round(algb / ms / 1e6 / peak, 3)}))
        del gout, gy, gw, gx
        if not args.skip_mlp:
            lins = [m for m in layer.conv.edge_mlp.mlp if isinstance(m, ScalarLinearLayer)]
            from nequip_b200.nn import dense

            if len(lins) == 2 and dense.RadialMLPGemm.supported(lins[0], lins[1], torch.float32):
                mlp = dense.RadialMLPGemm(lins[0], lins[1], dev)
                emb = torch.rand(E, 8, device=dev, generator=g)
                with torch.no_grad():
                    ms = timeit(lambda: mlp(emb), args.reps)
                    ref = torch.nn.functional.silu(emb.double() @ (lins[0].weight.double() * lins[0].alpha.double())) @ (
                        lins[1].weight.double() * lins[1].alpha.double())
                    out = mlp(emb)
                    err = float((out.double() - ref).abs().max() / ref.abs().max())
                    del ref, out
                W = sig.weight_numel
                flops = 2.0 * E * 128 * W
                print(json.dumps({"kernel": "mlp_fwd (hidden + grouped GEMM)", "layer": li, "W": W, "ms": round(ms, 4),
                                  "out_GB": round(E * W * 4 / 1e9, 3), "GBps_out": round(E * W * 4 / ms / 1e6, 1),
                                  "TFLOPs_fp32_equiv": round(flops / ms / 1e9, 1), "rel_err": err}))
                gemb = None
                # torch reference timing (cuBLAS fp32 SIMT)
                with torch.no_grad():
                    W1 = lins[0].weight * lins[0].alpha
                    W2 = lins[1].weight * lins[1].alpha
                    ms = timeit(lambda: torch.mm(torch.nn.functional.silu(torch.mm(emb, W1)), W2), max(3, args.reps // 3))
                print(json.dumps({"kernel": "mlp_fwd_torch_cublas_fp32", "layer": li, "ms": round(ms, 4)}))
                del emb, gemb
        del x, y, w
    pos = sysd["pos"].to(dev)
    sh, cell = sysd["edge_cell_shift"].to(dev), sysd["cell"].to(dev)
    with torch.no_grad():
        ms = timeit(lambda: ops.edge_embed(pos, ei, sh, cell, lmax=mk["l_max"], num_bessel=8, r_max=R_MAX, prefactor=1.0), args.reps)
    print(json.dumps({"kernel": "edge_embed_fwd", "ms": round(ms, 4), "E": E}))


if __name__ == "__main__":
    main()
