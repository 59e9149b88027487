#!/usr/bin/env python
"""Throughput of the reference's named architectures S/M/L/XL on the bench's Li3PO4-like box.

Per preset (frozen weights, ``strict_fast_path``, float32, ir_mul): the CUDA-graph energy + forces step in atom-steps/s,
the per-layer TP kernel times (forward, and backward with grad_x where the layer needs it), and the timed step's forces
against the same model and weights on the float64 kernels.  Prints one JSON line per result and the GPU's name and
power limit first.

``--tp-only`` times just the TP kernels of the M / L / XL middle layers through ``ops.get_plan``, ``ops.tp_scatter``
and ``nqb_tp_scatter_bwd``; with ``--tree DIR`` it imports ``nequip_b200`` from another checkout instead, so that two
versions of the kernels can be timed alternately in one session.  Each line names the timed tree by ``--label`` or,
by default, by its git commit.

When the float64 model does not fit on the timed frame (XL), the force check runs on the largest smaller box of the
same structure that fits; ``f64_check_atoms`` says which.

    python tools/bench_presets.py [--presets S,M,L,XL] [--n-side 22] [--steps 20] [--warmup 5]
    python tools/bench_presets.py --tp-only [--tree DIR] [--label NAME] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# middle-layer signatures (feature_irreps_in, irreps_edge_attr, conv_irreps_out) of the presets; written out so that
# checkouts without the preset table can build them too (checked against nequip_b200.known_signatures when present)
MIDDLE = {
    "M": ("128x0e+64x1o+32x2e", "1x0e+1x1o+1x2e", "224x0e+64x1o+32x2e"),
    "L": ("128x0e+64x1o+32x2e+32x3o", "1x0e+1x1o+1x2e+1x3o", "256x0e+64x1o+32x2e+32x3o"),
    "XL": ("320x0e+96x1o+64x2e+32x3o+32x4e", "1x0e+1x1o+1x2e+1x3o+1x4e", "544x0e+96x1o+64x2e+32x3o+32x4e"),
}
R_MAX = 5.0


def emit(line, sink):
    print(json.dumps(line), flush=True)
    sink.append(line)


def gpu_info():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    dev = torch.cuda.current_device()
    rows = [r.split(", ") for r in q.stdout.strip().splitlines()] if q.returncode == 0 else []
    row = next((r for r in rows if r and r[0] == str(dev)), None)
    return {"kind": "gpu", "name": torch.cuda.get_device_name(dev),
            "power_limit": row[2] if row else "not read", "max_sm_clock": row[3] if row else "not read"}


def timeit(fn, reps, warm=3):
    import torch

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


def time_tp(sig, plan, N, E, want_gx, reps, seed=0):
    """(forward ms, backward ms) of one TP signature on a random graph with the bench's node / edge counts."""
    import torch

    from nequip_b200 import ops

    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    dst = torch.sort(torch.randint(0, N, (E,), device=dev, generator=g)).values
    src = torch.randint(0, N, (E,), device=dev, generator=g)
    csr = ops.build_csr(dst, N)
    x = torch.randn(N, sig.d_in, device=dev, generator=g)
    y = torch.randn(E, sig.s_dim, device=dev, generator=g)
    w = torch.randn(E, sig.weight_numel, device=dev, generator=g)
    gout = torch.randn(N, sig.d_out, device=dev, generator=g)
    gx = torch.zeros_like(x) if want_gx else None
    gy, gw = torch.zeros_like(y), torch.empty_like(w)
    L = ops._capi.lib()
    with torch.no_grad():
        fwd = timeit(lambda: ops.tp_scatter(plan, x, y, w, dst, src, csr=csr), reps)

    def bwd():
        ops._capi.check(L.nqb_tp_scatter_bwd(plan.handle, 0, x.data_ptr(), y.data_ptr(), w.data_ptr(),
                                             csr.row_ptr.data_ptr(), 0, src.data_ptr(), gout.data_ptr(), N, E,
                                             0 if gx is None else gx.data_ptr(), gy.data_ptr(), gw.data_ptr(), 0,
                                             torch.cuda.current_stream().cuda_stream), "nqb_tp_scatter_bwd")

    return fwd, timeit(bwd, reps)


def tree_label(args) -> str:
    """What was timed: ``--label``, else the checkout's commit (with "+changes" when its working tree differs)."""
    if args.label:
        return args.label
    tree = os.path.abspath(args.tree) if args.tree else ROOT
    try:
        rev = subprocess.run(["git", "-C", tree, "rev-parse", "--short", "HEAD"], capture_output=True, text=True)
        dirty = subprocess.run(["git", "-C", tree, "status", "--porcelain", "--untracked-files=no"],
                               capture_output=True, text=True)
    except OSError:
        return "unknown commit"
    if rev.returncode != 0:
        return "unknown commit"
    return rev.stdout.strip() + ("+changes" if dirty.stdout.strip() else "")


def f64_check(name, meta, state, dev, f32, n_side):
    """max|F32 - F64| / max|F64| of the same model and weights on the float64 kernels.  ``f32`` are the forces of the
    timed step; when the float64 model does not fit on that frame, smaller boxes of the same structure are tried
    (float32 forces from an eager step there).  Returns (value, atoms of the checked frame)."""
    import warnings

    import torch

    from nequip_b200 import data as D
    from nequip_b200.nn.model import NequIPEnergyModel

    def forces(dtype, frame):
        m = NequIPEnergyModel.from_preset(name, r_max=R_MAX, type_names=meta["type_names"],
                                          avg_num_neighbors=meta["avg_num_neighbors"], model_dtype=dtype,
                                          strict_fast_path=(dtype == torch.float32)).cuda()
        m.load_state_dict({k: v.to(dtype) if v.is_floating_point() else v for k, v in state.items()})
        for p in m.parameters():
            p.requires_grad_(False)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # float64 runs the torch dense blocks, by design
            return m(frame)["forces"].detach().clone()

    ns = n_side
    while ns >= 6:
        try:
            if ns != n_side:
                sysd = D.make_system("li3po4", ns, r_max=R_MAX, seed=0)
                sysd.pop("_meta")
                dev = D.to_device(sysd, "cuda")
                f32 = forces(torch.float32, dev)
            f64 = forces(torch.float64, dev)
            return float((f32.double() - f64).abs().max()) / float(f64.abs().max()), int(dev["pos"].shape[0])
        except torch.cuda.OutOfMemoryError:
            torch.cuda.empty_cache()
            ns -= 4
    return "not measured (the float64 model does not fit)", None


def tp_only(args, sink):
    from nequip_b200 import known_signatures as ks
    from nequip_b200 import ops
    from nequip_b200.codegen import GenOptions

    N, E = 10648, 588616  # the bench frame (Li3PO4-like, 22^3 atoms, r_max 5)
    for name, (fin, fe, fout) in MIDDLE.items():
        sig = ks.make_signature(fin, fe, fout)
        if hasattr(ks, "preset_layer_signatures"):
            assert sig.canonical() == ks.preset_layer_signatures(name)[1].canonical(), name
        plan = ops.get_plan(sig.irreps_in1, sig.irreps_in2, sig.irreps_out, sig.instructions, GenOptions(layout="ir_mul"))
        fwd, bwd = time_tp(sig, plan, N, E, True, args.reps)
        emit({"kind": "tp_middle", "tree": tree_label(args), "preset": name, "W": sig.weight_numel, "N": N, "E": E,
              "tp_fwd_ms": round(fwd, 4), "tp_bwd_ms": round(bwd, 4)}, sink)


def presets(args, sink):
    import torch

    from nequip_b200 import data as D
    from nequip_b200.graph import GraphedEnergyForces
    from nequip_b200.nn.model import NequIPEnergyModel

    for name in args.presets.split(","):
        n_side = args.n_side
        while True:
            try:
                sysd = D.make_system("li3po4", n_side, r_max=R_MAX, seed=0)
                meta = sysd.pop("_meta")
                N, E = sysd["pos"].shape[0], sysd["edge_index"].shape[1]
                model = NequIPEnergyModel.from_preset(name, r_max=R_MAX, type_names=meta["type_names"],
                                                      avg_num_neighbors=meta["avg_num_neighbors"],
                                                      strict_fast_path=True).cuda()
                for p in model.parameters():
                    p.requires_grad_(False)
                dev = D.to_device(sysd, "cuda")
                model(dev)  # first call: per-layer fused/unfused choice, kernel libraries
                graphed = GraphedEnergyForces(model, dev)
                for _ in range(args.warmup):
                    graphed.replay()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    out = graphed.replay()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.steps
                graphed.check_sorted()
                f32 = out["forces"].clone()
                break
            except torch.cuda.OutOfMemoryError:
                model = graphed = dev = out = None
                torch.cuda.empty_cache()
                n_side -= 2
        peak_gb = torch.cuda.max_memory_allocated() / 1e9
        del graphed, out
        torch.cuda.empty_cache()
        check, check_atoms = f64_check(name, meta, model.state_dict(), dev, f32, n_side)
        torch.cuda.empty_cache()
        emit({"kind": "step", "preset": name, "atoms": N, "edges": E, "n_side": n_side, "ms_per_step": round(ms, 3),
              "atom_steps_per_s": round(N / ms * 1e3, 1), "peak_mem_GB": round(peak_gb, 1),
              "max_dF_rel_vs_f64_kernels": check, "f64_check_atoms": check_atoms,
              "cuda_graph": True, "dtype": "f32"}, sink)
        for li, layer in enumerate(model.layers):
            plan = layer.conv.tp_scatter._plan
            fwd, bwd = time_tp(plan.sig, plan, N, E, li != 0, args.reps, seed=li)
            emit({"kind": "tp_layer", "preset": name, "layer": li, "W": plan.sig.weight_numel,
                  "tp_fwd_ms": round(fwd, 4), "tp_bwd_ms": round(bwd, 4), "bwd_grad_x": li != 0}, sink)
        del model, dev
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", default="S,M,L,XL")
    ap.add_argument("--n-side", type=int, default=22)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tp-only", action="store_true")
    ap.add_argument("--tree", default=None, help="import nequip_b200 from this checkout")
    ap.add_argument("--label", default=None, help="name of the timed tree in the output (default: its git commit)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree) if args.tree else ROOT)
    import torch

    torch.backends.cuda.matmul.allow_tf32 = False
    sink = []
    emit(dict(gpu_info(), time=time.strftime("%Y-%m-%dT%H:%M:%S")), sink)
    if args.tp_only:
        tp_only(args, sink)
    else:
        presets(args, sink)
    if args.out:
        with open(args.out, "a") as f:
            for line in sink:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
