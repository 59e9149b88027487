#!/usr/bin/env python
"""Time the per-atom dense blocks (linear_1, linear_2, self-connection) of one interaction layer of the
Li3PO4 bench model on the grouped GEMM, forward and backward, and print their problem lists."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nequip_b200.irreps import build_tp_instructions  # noqa: E402
from nequip_b200.nn import dense  # noqa: E402
from nequip_b200.nn.model import Linear, SelfConnection, layer_irreps  # noqa: E402


def timeit(fn, reps=20, warm=3):
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
    N, T = 10648, 3
    dev = "cuda"
    layers = layer_irreps(2, 64, 4, True)
    for li, (fin, fe, fout, _) in enumerate(layers):
        mid, _ins = build_tp_instructions(fin, fe, fout)
        lin1 = Linear(fin, fin, "ir_mul").to(dev)
        lin2 = Linear(mid.simplify(), fout, "ir_mul").to(dev)
        sc = SelfConnection(fin, T, fout, "ir_mul").to(dev)
        tt = torch.randn(T, T, device=dev)
        types = torch.randint(0, T, (N,), device=dev)
        blocks = {"lin1": dense.IrrepsLinearGemm(lin1, dev), "lin2": dense.IrrepsLinearGemm(lin2, dev),
                  "sc": dense.SelfConnectionGemm(sc, tt, dev)}
        for name, blk in blocks.items():
            x = torch.randn(N, blk.d_in, device=dev)
            out = torch.zeros(N, blk.d_out, device=dev)
            gx = torch.zeros(N, blk.d_in, device=dev)
            rs = torch.nn.functional.one_hot(types, T).float().t().contiguous() if name == "sc" else None
            f = timeit(lambda: blk.fwd.run(x, out, N, rs))
            b = timeit(lambda: blk.bwd.run(out, gx, N, rs))
            flops = 2.0 * N * sum(p.B.shape[0] * p.B.shape[1] for p in blk.fwd.problems)
            print(json.dumps({"layer": li, "block": name, "d_in": blk.d_in, "d_out": blk.d_out,
                              "problems": len(blk.fwd.problems), "ntiles": blk.fwd.ntiles_total,
                              "fwd_ms": round(f, 4), "bwd_ms": round(b, 4), "gflop": round(flops / 1e9, 2)}), flush=True)


if __name__ == "__main__":
    main()
