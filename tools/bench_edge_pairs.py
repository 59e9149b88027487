"""Radial-MLP forward with and without the reverse-edge pair map, on bench.py's default frame and model.

Per layer: the per-edge forward (k_hidden_fwd + k_gemm3x over E rows) against the pair-shared one
(k_hidden_fwd on the slots + the paired k_gemm3x over U rows, each row stored to both edges of its slot), alternated
over ROUNDS rounds of LAUNCHES launches, with the two [E, W] outputs checked bitwise equal.  Then the pair-map
kernels (ops.edge_pairs) alone.  One JSON line per measurement, with the card's name, power limit and max SM clock
read in the same process.  Whole steps are compared with bench.py against the parent commit.

    python tools/bench_edge_pairs.py [--out FILE.jsonl]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nequip_b200 import data as D  # noqa: E402
from nequip_b200 import ops  # noqa: E402
from nequip_b200.nn.model import NequIPEnergyModel  # noqa: E402

ROUNDS, LAUNCHES = 5, 20
R_MAX = 5.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def timed(fn, n=LAUNCHES):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    dev = torch.device("cuda")
    gpu = card()
    sysd = D.make_system("li3po4", 22, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], l_max=2, num_layers=4, num_features=64,
                              parity=True, radial_mlp_depth=1, radial_mlp_width=128,
                              avg_num_neighbors=meta["avg_num_neighbors"], strict_fast_path=True).to(dev)
    for p in model.parameters():
        p.requires_grad_(False)
    d = D.to_device(sysd, dev)
    model(d)  # prepares every layer's tensor-core blocks
    torch.cuda.synchronize()
    ei, E, N = d["edge_index"], d["edge_index"].shape[1], d["pos"].shape[0]
    _v, _y, emb = ops.edge_embed(d["pos"], ei, d["edge_cell_shift"], d["cell"], lmax=2, num_bessel=8, r_max=R_MAX,
                                 prefactor=2 * math.pi / R_MAX ** 2)
    csr = ops.csr_cache.get(ei[0], N)
    pairs = ops.edge_pairs(ei, d["edge_cell_shift"], emb, csr)
    U = int(pairs[1].item())
    lines = []

    def emit(rec):
        rec.update(gpu=gpu, E=E, U=U)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for li, layer in enumerate(model.layers):
        mlp = layer.conv._tc_cache[1]["mlp"]
        h = torch.empty((E, 128), device=dev)
        w_edge = torch.empty((E, mlp.W), device=dev)
        hp = torch.empty((E, 128), device=dev)
        w_pair = torch.empty((E, mlp.W), device=dev)

        def per_edge():
            ops.mlp_hidden_fwd(emb, mlp.w1s, h, None)
            mlp.fwd.run(h, w_edge, E)

        def shared():
            ops.mlp_hidden_fwd_rows(emb, mlp.w1s, pairs, hp)
            mlp.fwd.run_pairs(hp, w_pair, pairs)

        per_edge(), shared()
        torch.cuda.synchronize()
        assert torch.equal(w_edge, w_pair), f"layer {li}: w differs"
        a, b = [], []
        for _ in range(ROUNDS):
            a.append(timed(per_edge))
            b.append(timed(shared))
        emit(dict(what="radial_mlp_fwd", layer=li, W=mlp.W, per_edge_ms=a, pair_shared_ms=b, w_bitwise_equal=True))

    t = [timed(lambda: ops.edge_pairs(ei, d["edge_cell_shift"], emb, csr)) for _ in range(ROUNDS)]
    emit(dict(what="edge_pairs", ms=t))

    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
