#!/usr/bin/env python
"""Radial MLPs of any depth on the project's kernels, timed on the GPU.

``--mode layer``: one radial MLP at the edge count of the 10 648-atom Li3PO4 frame, forward + grad_emb (the inference
step's use: frozen weights, gradient w.r.t. the edge embedding only):
  A: the layer's torch formulation (``conv.edge_mlp``: torch.mm + SiLU, autograd backward);
  B: ``RadialMLPGemm`` (k_hidden_fwd/bwd for an [8, 128] first layer, k_gemm3x with the SiLU epilogue otherwise);
  B_gemm_first (width 128 only): ``RadialMLPGemm`` with the first layer on k_gemm3x as well.
Arms alternate A, B, A, B ... in one process; B's output and gradient are compared with A's.

``--mode step``: a whole MD step (energy + forces) of the tutorial model (l_max 1, 4 layers, 32 features, radial 2x64)
and of a radial 2x128 model, on the 1 000-atom water box and the 10 648-atom Li3PO4 frame: eager
(``ops.neighbor_list`` + ``model(d)``) and ``GraphedMDStep`` on the frozen frame.  ``--root`` imports the package from
another tree, so that two versions can be timed alternately by a driver script.  ``strict_fast_path`` is left off, so a
version without the depth >= 2 path runs its torch fallback; ``radial_on_gemm`` says which path each layer took.

The first line names the GPU, its power limit and its maximum SM clock.

    python tools/bench_radial_mlp.py --mode layer|step [--reps 5] [--iters 20] [--root DIR] [--tag NAME] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--mode", choices=["layer", "step"], required=True)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--tag", default="")
ap.add_argument("--out", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

from nequip_b200 import data as D  # noqa: E402
from nequip_b200.nn.model import NequIPEnergyModel  # noqa: E402

R_MAX = 5.0
SINK = []


def emit(line):
    line = dict(line, tag=args.tag) if args.tag else line
    print(json.dumps(line), flush=True)
    SINK.append(line)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    dev = torch.cuda.current_device()
    rows = [r.split(", ") for r in q.stdout.strip().splitlines()] if q.returncode == 0 else []
    row = next((r for r in rows if r and r[0] == str(dev)), None)
    return {"kind": "gpu", "name": torch.cuda.get_device_name(dev),
            "power_limit": row[2] if row else "not read", "max_sm_clock": row[3] if row else "not read"}


def make(kind, n_side, depth, width, l_max, features):
    sysd = D.make_system(kind, n_side, r_max=R_MAX, seed=0)
    meta = sysd.pop("_meta")
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
                              parity=True, l_max=l_max, num_layers=4, num_features=features, radial_mlp_depth=depth,
                              radial_mlp_width=width).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    return model, sysd


def cuda_ms(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def layer_mode():
    from nequip_b200.nn import dense
    from nequip_b200.nn.model import ScalarLinearLayer

    class GemmFirst(dense.RadialMLPGemm):
        """The same MLP with an [8, 128] first layer on k_gemm3x instead of k_hidden_fwd/bwd."""

        @staticmethod
        def uses_hidden_kernel(first):
            return False

    E = None
    for depth in (1, 2, 3):
        for width in (64, 128):
            model, sysd = make("li3po4", 22, depth, width, 2, 64)
            E = int(sysd["edge_index"].shape[1])
            conv = model.layers[1].conv
            lins = [m for m in conv.edge_mlp.mlp if isinstance(m, ScalarLinearLayer)]
            W = lins[-1].weight.shape[1]
            g = torch.Generator(device="cuda").manual_seed(depth * 1000 + width)
            emb = torch.rand(E, 8, device="cuda", generator=g).requires_grad_(True)
            gw = torch.randn(E, W, device="cuda", generator=g)
            arms = {"A_torch": conv.edge_mlp,
                    "B": dense.RadialMLPGemm(lins[0], lins[-1], "cuda", middle=lins[1:-1])}
            if width == 128:
                arms["B_gemm_first"] = GemmFirst(lins[0], lins[-1], "cuda", middle=lins[1:-1])

            def step(mlp):
                out = mlp(emb)
                (ge,) = torch.autograd.grad(out, emb, gw)
                return out, ge

            res = {k: tuple(t.detach() for t in step(m)) for k, m in arms.items()}
            o_ref, g_ref = (t.double() for t in res["A_torch"])
            dev = {k: [float((o.double() - o_ref).abs().max() / o_ref.abs().max()),
                       float((ge.double() - g_ref).abs().max() / g_ref.abs().max())] for k, (o, ge) in res.items()}
            del res, o_ref, g_ref
            ms = {k: [] for k in arms}
            for _ in range(args.reps):
                for k, m in arms.items():
                    ms[k].append(round(cuda_ms(lambda: step(m), args.iters), 4))
            emit({"kind": "radial_layer", "E": E, "num_bessels": 8, "depth": depth, "width": width, "W": W,
                  "ms_fwd_plus_grad_emb": ms, "best_ms": {k: min(v) for k, v in ms.items()},
                  "speedup_B_over_A": round(min(ms["A_torch"]) / min(ms["B"]), 3),
                  "max_rel_dev_vs_torch_out_grad": dev})
            del arms, emb, gw, model
            torch.cuda.empty_cache()


def step_mode():
    from nequip_b200 import ops
    from nequip_b200.graph import GraphedMDStep

    for name, (depth, width) in (("tutorial_l1_r2x64", (2, 64)), ("l1_r2x128", (2, 128))):
        for kind, n_side in (("water", 10), ("li3po4", 22)):
            model, sysd = make(kind, n_side, depth, width, 1, 32)
            dev = D.to_device({k: sysd[k] for k in ("pos", "atom_types", "cell")}, "cuda")
            pos = dev["pos"]

            def eager():
                nl = ops.neighbor_list(pos, dev["cell"], True, R_MAX)
                return model(dict(dev, pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"]))

            ref = eager()
            g = GraphedMDStep(model, dev)
            out = g(pos)
            on_gemm = [l.conv._tc_cache is not None and l.conv._tc_cache[1] is not None
                       and l.conv._tc_cache[1]["mlp"] is not None for l in model.layers]
            fused = [bool(l.conv._fused_choice) for l in model.layers]
            de = abs(float(out["total_energy"]) - float(ref["total_energy"])) / abs(float(ref["total_energy"]))
            df = float((out["forces"] - ref["forces"]).abs().max() / ref["forces"].abs().max())
            ms = {"eager": [], "graph": []}
            for _ in range(args.reps):
                for arm, fn in (("eager", eager), ("graph", lambda: g(pos))):
                    for _w in range(3):
                        fn()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _i in range(args.iters):
                        fn()["forces"].cpu()
                    ms[arm].append(round((time.perf_counter() - t0) * 1e3 / args.iters, 4))
            emit({"kind": "md_step", "model": name, "system": f"{kind}_{n_side}", "atoms": int(pos.shape[0]),
                  "edges": int(sysd["edge_index"].shape[1]), "ms_per_step": ms,
                  "best_ms": {k: min(v) for k, v in ms.items()}, "radial_on_gemm": on_gemm, "fused_choice": fused,
                  "graph_vs_eager_rel_energy": de, "graph_vs_eager_rel_force": df,
                  "energy": float(ref["total_energy"])})
            del g, model, dev
            torch.cuda.empty_cache()


if __name__ == "__main__":
    if not torch.cuda.is_available():
        raise SystemExit("bench_radial_mlp.py times GPU kernels and needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    emit(gpu_info())
    layer_mode() if args.mode == "layer" else step_mode()
    if args.out:
        with open(args.out, "a") as f:
            for line in SINK:
                f.write(json.dumps(line) + "\n")
