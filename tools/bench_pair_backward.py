"""Radial-MLP backward per edge and on the slots of the reverse-edge pair map, on bench.py's default frame and model.

Per layer: the per-edge backward (the transposed k_gemm3x over E rows + k_hidden_bwd) against the slot backward (the
gathered-sum k_gemm3x over U slots, each A row the sum of the slot's two edge-weight gradients, + k_hidden_bwd on the
slots), alternated over ROUNDS rounds of LAUNCHES launches.  The deviation reported is max |slot - per-edge| of
grad_emb summed over the two edges of each slot, over max |per-edge|.  One JSON line per layer, with the card's name,
power limit and max SM clock read in the same process.  Whole steps are compared with bench.py against the parent
commit.

    python tools/bench_pair_backward.py [--out FILE.jsonl]
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
    rep, par = pairs[0][:U, 0], pairs[0][:U, 1]
    has_par = par >= 0
    lines = []

    def emit(rec):
        rec.update(gpu=gpu, E=E, U=U)
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    g = torch.Generator(device=dev).manual_seed(0)
    for li, layer in enumerate(model.layers):
        mlp = layer.conv._tc_cache[1]["mlp"]
        gw = torch.randn((E, mlp.W), device=dev, generator=g)  # > the 50 MB L2 from W = 192 on
        gh_e, gemb_e = torch.empty((E, 128), device=dev), torch.empty_like(emb)
        gh_s, gemb_s = torch.empty((E, 128), device=dev), torch.empty_like(emb)

        def per_edge():
            mlp.bwd.run(gw, gh_e, E)
            ops.mlp_hidden_bwd(emb, mlp.w1s, gh_e, gemb_e)

        def slots():
            mlp.bwd.run_pair_sum(gw, gh_s, pairs)
            ops.mlp_hidden_bwd_rows(emb, mlp.w1s, gh_s, pairs, gemb_s)

        per_edge(), slots()
        torch.cuda.synchronize()
        want = gemb_e[rep].double()
        want[has_par] += gemb_e[par[has_par]].double()
        dev_rel = float((gemb_s[rep].double() - want).abs().max()) / float(gemb_e.abs().max())
        partners_zero = bool((gemb_s[par[has_par]] == 0).all())
        a, b = [], []
        for _ in range(ROUNDS):
            a.append(timed(per_edge))
            b.append(timed(slots))
        emit(dict(what="radial_mlp_bwd", layer=li, W=mlp.W, per_edge_ms=a, slot_ms=b,
                  slot_sum_max_dev_over_max=dev_rel, partner_rows_zero=partners_zero))
        del gw

    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
