"""The device relaxation on the GPU: the cell packed into a batched neighbour-list plan on the device
(``NeighborListPlan.set_cell_device``) against the host pack and ``ops.neighbor_list``, the nqb_relax kernels' write
contracts and one step against the float64 oracle (tests/relax_oracle.py), and ``GraphedRelax`` against a host loop
of the eager model and the oracle, plus its bookkeeping: frozen frames, block sizes, early stop, zero-step frames,
max_steps, failure and re-capture.

Under ``ops.set_deterministic(True)`` a float64 model's graphed forces agree with its eager forces to 1e-12 max|F|
(tests/test_md_trajectory_gpu.py).  A FIRE step moves a DOF by at most dtmax^2 |g| (before the maxstep clip, which
only shrinks it), so over n steps two runs from one structure differ by about n * dtmax^2 * 1e-12 max|F| times the
growth the model's Hessian allows per step; ``POS_TOL`` = 1e-8 Angstrom leaves three orders of magnitude for that
growth over 30 steps."""
import ctypes
import math

import numpy as np
import pytest
import torch

import relax_oracle as ro
from kernel_contracts import guarded
from nequip_b200 import _capi, ops
from nequip_b200.relax import GraphedRelax
from test_md_trajectory_gpu import _system

pytestmark = pytest.mark.gpu

R_MAX = 5.0
POS_TOL = 1e-8
N_STEPS = 30


@pytest.fixture(autouse=True)
def _deterministic():
    prev = ops.deterministic()
    ops.set_deterministic(True)
    yield
    ops.set_deterministic(prev)


# ------------------------------------------------------------------------------------------------------------------
# set_cell_device
# ------------------------------------------------------------------------------------------------------------------
# NlBlock (csrc/nqb_nl.cu): byte offsets of the fields the cell determines
_DBL = {"cell": (0, 9), "inv": (72, 9), "diag": (144, 3), "pad_shift": (264, 3), "perp": (304, 3)}
_INT = {"orthorhombic": (168, 1), "sr": (196, 3), "nb": (184, 3)}
_CELLS = {
    "triclinic": [[6.1, 0.0, 0.0], [1.3, 5.7, 0.0], [-0.8, 1.1, 6.6]],
    "left_handed": [[0.0, 6.2, 0.0], [6.0, 0.0, 0.0], [0.4, 0.3, 6.4]],
    "sheared": [[6.0, 0.0, 0.0], [4.9, 5.5, 0.0], [0.0, 0.0, 6.3]],
    "sub_r_max": [[3.1, 0.0, 0.0], [0.2, 2.9, 0.0], [0.1, 0.3, 3.4]],
    "orthorhombic": [[6.0, 0.0, 0.0], [0.0, 7.0, 0.0], [0.0, 0.0, 5.5]],
    "tied_lengths": [[6.0, 0.0, 0.0], [0.0, 6.0, 0.0], [0.0, 0.0, 6.0]],
}


def _fields(block: torch.Tensor, F: int):
    raw = block.cpu().view(F, -1)
    out = {}
    for k, (o, n) in _DBL.items():
        out[k] = raw[:, o:o + 8 * n].contiguous().view(torch.float64).view(F, n)
    for k, (o, n) in _INT.items():
        out[k] = raw[:, o:o + 4 * n].contiguous().view(torch.int32).view(F, n)
    return out, raw


def _plan(cells0, counts, typed=False, capacity=None):
    F = len(counts)
    batch = torch.repeat_interleave(torch.arange(F), torch.tensor(counts)).cuda()
    N = sum(counts)
    kw = {}
    if typed:
        g = torch.Generator().manual_seed(1)
        kw = dict(atom_types=torch.randint(0, 2, (N,), generator=g).cuda(),
                  edge_type_cutoff=torch.tensor([[3.0, 4.5], [4.0, 5.0]], dtype=torch.float64))
    cap = capacity or 200 * N
    return ops.NeighborListPlan(N, torch.tensor(cells0, dtype=torch.float64), True, R_MAX, cap, device="cuda",
                                variable_cell=True, batch=batch, **kw), batch, kw


def test_set_cell_device_block_equals_host_pack():
    assert int(_capi.lib().nqb_nl_params_bytes()) == 336
    names = list(_CELLS)
    F = len(names)
    counts = [40] * F
    start = np.stack([np.diag([7.0, 7.5, 8.0])] * F)
    plan, _, _ = _plan(start, counts)
    new = torch.tensor(np.stack([_CELLS[n] for n in names]), dtype=torch.float64)
    plan.set_cell(new)
    torch.cuda.synchronize()
    host, host_raw = _fields(plan._params_dev.clone(), F)
    plan.set_cell(torch.tensor(start))
    torch.cuda.synchronize()
    err = plan.set_cell_device(new.cuda())
    dev, dev_raw = _fields(plan._params_dev.clone(), F)
    assert int(err.sum()) == 0
    for k in _INT:
        assert torch.equal(dev[k], host[k]), k
    for k in ("cell", "diag"):
        assert torch.equal(dev[k], host[k]), k
    for k in ("inv", "perp"):
        scale = host[k].abs().amax(dim=1, keepdim=True)
        assert ((dev[k] - host[k]).abs() <= 8 * 2.0 ** -52 * scale).all(), k
    assert torch.equal(dev["pad_shift"], host["pad_shift"])
    # every other byte is the host pack's
    mask = torch.ones(dev_raw.shape[1], dtype=torch.bool)
    for o, n in [_DBL["inv"], _DBL["perp"]]:
        mask[o:o + 8 * n] = False
    assert torch.equal(dev_raw[:, mask], host_raw[:, mask])


@pytest.mark.parametrize("typed", [False, True], ids=["untyped", "typed"])
def test_set_cell_device_rows_equal_neighbor_list(typed):
    names = ["triclinic", "left_handed", "sheared", "sub_r_max"]
    counts = [30, 25, 35, 12]
    g = torch.Generator().manual_seed(7)
    cells = torch.tensor(np.stack([_CELLS[n] for n in names]), dtype=torch.float64)
    frac = torch.rand(sum(counts), 3, generator=g, dtype=torch.float64)
    batch_h = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    pos = torch.einsum("ni,nij->nj", frac, cells[batch_h]).cuda()
    plan, batch, kw = _plan(np.stack([np.diag([7.0, 7.5, 8.0])] * len(counts)), counts, typed)
    plan.set_cell_device(cells.cuda())
    out = plan.run(pos)
    assert int(out["overflow"]) == 0
    ref = ops.neighbor_list(pos, cells.cuda(), True, R_MAX, batch=batch, **kw)
    E = int(out["num_edges"])
    assert E == ref["edge_index"].shape[1]
    rp = out["row_ptr"].cpu()
    real = torch.cat([torch.arange(int(rp[i]), int(rp[i]) + int((ref["edge_index"][0] == i).sum()))
                      for i in range(pos.shape[0])]).cuda()
    assert torch.equal(out["edge_index"][:, real], ref["edge_index"])
    assert torch.equal(out["edge_cell_shift"][real], ref["edge_cell_shift"])


def test_set_cell_device_invalid_cell_sets_the_flag_and_keeps_the_block():
    counts = [10, 10, 10]
    plan, _, _ = _plan(np.stack([np.diag([7.0, 7.5, 8.0])] * 3), counts)
    before = plan._params_dev.clone()
    cells = torch.tensor(np.stack([_CELLS["triclinic"]] * 3), dtype=torch.float64)
    cells[0, 2] = cells[0, 0] + cells[0, 1]  # singular
    cells[2, 1, 1] = float("nan")
    err = plan.set_cell_device(cells.cuda())
    assert err.cpu().tolist() == [1, 0, 1]
    after = plan._params_dev.view(3, -1).cpu()
    assert torch.equal(after[0], before.view(3, -1)[0].cpu()) and torch.equal(after[2], before.view(3, -1)[2].cpu())
    assert not torch.equal(after[1], before.view(3, -1)[1].cpu())


def test_set_cell_device_captured_follows_the_cells():
    counts = [20, 30]
    plan, batch, _ = _plan(np.stack([np.diag([7.0, 7.5, 8.0])] * 2), counts)
    cells = torch.tensor(np.stack([_CELLS["triclinic"], _CELLS["sheared"]]), dtype=torch.float64).cuda()
    g = torch.Generator().manual_seed(3)
    frac = torch.rand(50, 3, generator=g, dtype=torch.float64).cuda()
    buf_cells, buf_pos = cells.clone(), torch.zeros(50, 3, dtype=torch.float64, device="cuda")
    bh = batch

    def step():
        buf_pos.copy_(torch.einsum("ni,nij->nj", frac, buf_cells[bh]))
        plan.set_cell_device(buf_cells)
        return plan.run(buf_pos)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for scale in (1.0, 0.93, 1.07):
        buf_cells.copy_(cells * scale)
        graph.replay()
        ref = ops.neighbor_list(buf_pos, buf_cells, True, R_MAX, batch=bh)
        assert int(out["num_edges"]) == ref["edge_index"].shape[1]
        assert int(out["overflow"]) == 0


# ------------------------------------------------------------------------------------------------------------------
# kernels against one oracle step
# ------------------------------------------------------------------------------------------------------------------
def _kernel_cases():
    named = [("batch_empty", [5, 0, 37]), ("cta_edges", [255, 256, 257]), ("above_64_ctas", [16385, 3])]
    cases = []
    for name, counts in named:
        driver = min(64, -(-max(counts) // 256))
        for nblk in sorted({1, 2, driver}):
            cases.append(pytest.param(counts, nblk, id=f"{name}-nblk{nblk}"))
    return cases


@pytest.mark.parametrize("counts,nblk", _kernel_cases())
@pytest.mark.parametrize("has_cell", [False, True], ids=["positions", "frechet"])
def test_kernels_match_one_oracle_step_and_write_only_their_outputs(counts, nblk, has_cell):
    rng = np.random.default_rng(len(counts) + nblk)
    F, N = len(counts), sum(counts)
    ptr = [0] + np.cumsum(counts).tolist()
    p = 0.01 if has_cell else 0.0
    frames, forces0, forces1, virials = [], [], [], []
    for f, n in enumerate(counts):
        C0 = np.diag([8.0, 9.0, 10.0]) + 0.3 * rng.standard_normal((3, 3))
        fr = ro.Frame(rng.random((n, 3)) @ C0, C0, has_cell, fmax=1e-9, p=p)
        fr.Q = 0.02 * rng.standard_normal((3, 3)) if has_cell else fr.Q
        fr.v = 0.1 * rng.standard_normal((n + 3 * has_cell, 3))
        fr.dt, fr.a, fr.Nsteps = 0.1 + 0.05 * f, 0.08, 3 + 4 * (f % 2)
        f0, f1 = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
        w0, w1 = rng.standard_normal((3, 3)), rng.standard_normal((3, 3))
        fr.evaluate(0.0, f0, w0 + w0.T)
        frames.append(fr)
        forces1.append(f1)
        virials.append(w1 + w1.T)
    if F > 1:  # one frame mixes, one resets
        frames[-1].v = -frames[-1].g.copy()
    cat = lambda xs: torch.tensor(np.concatenate(xs) if xs else np.zeros((0, 3)), dtype=torch.float64)  # noqa
    cu = dict(device="cuda")
    s = cat([fr.s for fr in frames])
    d_pos, c_pos = guarded(N, 3, torch.float64, body=cat([fr.positions() for fr in frames]), **cu)
    d_s, c_s = guarded(N, 3, torch.float64, body=s, **cu)
    d_vel, c_vel = guarded(N, 3, torch.float64, body=cat([fr.v[:len(fr.s)] for fr in frames]), **cu)
    d_g, c_g = guarded(N, 3, torch.float64, body=cat([fr.g[:len(fr.s)] for fr in frames]), **cu)
    d_part, c_part = guarded(F * nblk, 4, torch.float64, **cu)
    t3 = lambda xs: torch.tensor(np.stack(xs).reshape(F, 9), dtype=torch.float64)  # noqa
    d_Q, c_Q = guarded(F, 9, torch.float64, body=t3([fr.Q for fr in frames]), **cu)
    vc = [fr.v[len(fr.s):] if has_cell else np.zeros((3, 3)) for fr in frames]
    d_vc, c_vc = guarded(F, 9, torch.float64, body=t3(vc), **cu)
    gc = [fr.g[len(fr.s):] if has_cell else np.zeros((3, 3)) for fr in frames]
    d_gc, c_gc = guarded(F, 9, torch.float64, body=t3(gc), **cu)
    d_Fd, c_Fd = guarded(F, 9, torch.float64, body=t3([fr.Fd() for fr in frames]), **cu)
    d_cell, c_cell = guarded(F, 9, torch.float64, body=t3([fr.cell() for fr in frames]), **cu)
    d_fs, c_fs = guarded(F, 2, torch.float64, body=torch.tensor([[fr.dt, fr.a] for fr in frames], dtype=torch.float64), **cu)
    ist = torch.tensor([[fr.Nsteps, 0, int(fr.converged), 0, 7] for fr in frames], dtype=torch.int64)
    steps = [7 if fr.converged else 8 for fr in frames]
    d_is, c_is = guarded(F, 5, torch.int64, body=ist, **cu)
    d_coef, c_coef = guarded(F, 4, torch.float64, **cu)
    C0 = t3([fr.C0 for fr in frames]).cuda()
    cfac = torch.tensor([fr.c for fr in frames], dtype=torch.float64).cuda()
    # the partial sums of the current state (what the previous step's gforce left)
    aptr = torch.tensor(ptr, dtype=torch.int64).cuda()
    P, L, st = ops._ptr, _capi.lib(), ops._stream()
    f_cur = cat([fr.g[:len(fr.s)] @ np.linalg.inv(fr.Fd()) for fr in frames]).cuda()
    _capi.check(L.nqb_relax_gforce(F, nblk, P(aptr), int(has_cell), P(d_Fd), P(f_cur), P(d_vel), P(d_g), P(d_part),
                                   st))
    fire = (ctypes.c_double * 7)(0.2, 1.0, 1.1, 0.5, 0.1, 0.99, 5)
    _capi.check(L.nqb_relax_fire(F, nblk, P(d_part), fire, int(has_cell), P(cfac), P(C0), P(d_gc), P(d_Q), P(d_vc),
                                 P(d_Fd), P(d_cell), P(d_fs), P(d_is), P(d_coef), st))
    _capi.check(L.nqb_relax_move(F, nblk, P(aptr), P(d_coef), int(has_cell), P(d_Fd), P(d_g), P(d_vel),
                                 P(d_s) if has_cell else 0, P(d_pos), st))
    # oracle step, then the new forces at the new structure
    for fr, f1, w1 in zip(frames, forces1, virials):
        fr.step()
        fr.evaluate(1.5, f1, w1)
    f_new = cat(forces1).cuda()
    _capi.check(L.nqb_relax_gforce(F, nblk, P(aptr), int(has_cell), P(d_Fd), P(f_new), P(d_vel), P(d_g), P(d_part),
                                   st))
    vir = torch.tensor(np.stack(virials), dtype=torch.float64).cuda()
    e = torch.full((F,), 1.5, dtype=torch.float64, device="cuda")
    zero64, zero32 = torch.zeros(1, dtype=torch.int64, **cu), torch.zeros(1, dtype=torch.int32, **cu)
    one32 = torch.ones(1, dtype=torch.int32, **cu)
    step = torch.zeros(1, dtype=torch.int64, **cu)
    d_log, c_log = guarded(2 * F, 4, torch.float64, **cu)
    flags = torch.tensor([0, 0, -1, 0], dtype=torch.int64, **cu)
    _capi.check(L.nqb_relax_finish(F, nblk, P(d_part), int(has_cell), p, P(cfac), P(d_Q), P(d_Fd), P(d_cell),
                                   P(vir), P(e), 1e-9, 1e6, P(d_gc), P(d_is), P(zero64), P(zero32), P(one32), 2,
                                   P(step), P(d_log), P(flags), st))
    torch.cuda.synchronize()
    for c in (c_pos, c_s, c_vel, c_g, c_part, c_Q, c_vc, c_gc, c_Fd, c_cell, c_fs, c_is, c_coef, c_log):
        c()

    def close(got, ref, what):
        ref = torch.as_tensor(np.asarray(ref), dtype=torch.float64)
        got = got.cpu().reshape(ref.shape)
        tol = 1e-14 * max(1.0, float(ref.abs().max()) if ref.numel() else 1.0)
        assert not torch.isnan(got).any(), what
        if ref.numel():
            err = (got - ref).abs()
            assert float(err.max()) <= tol, (what, float(err.max()), tol, torch.nonzero(err > tol)[:5].tolist())

    close(d_pos, np.concatenate([fr.positions() for fr in frames]), "pos")
    close(d_vel, np.concatenate([fr.v[:len(fr.s)] for fr in frames]), "vel")
    close(d_g, np.concatenate([fr.g[:len(fr.s)] for fr in frames]), "g")
    close(d_fs, [[fr.dt, fr.a] for fr in frames], "dt, a")
    assert d_is.cpu()[:, 0].tolist() == [fr.Nsteps for fr in frames]
    assert d_is.cpu()[:, 4].tolist() == steps
    assert d_is.cpu()[:, 2].tolist() == [int(fr.converged) for fr in frames]
    if has_cell:
        close(d_s, np.concatenate([fr.s for fr in frames]), "s")
        close(d_Q, np.stack([fr.Q for fr in frames]), "Q")
        close(d_cell, np.stack([fr.cell() for fr in frames]), "cell")
        close(d_gc, np.stack([fr.g[len(fr.s):] for fr in frames]), "gcell")
        close(d_vc, np.stack([fr.v[len(fr.s):] for fr in frames]), "vcell")
    log = d_log.view(2, F, 4).cpu()[0]
    close(log, [fr.log for fr in frames], "log")
    assert int(step) == 1


# ------------------------------------------------------------------------------------------------------------------
# GraphedRelax against a host loop
# ------------------------------------------------------------------------------------------------------------------
def _as_batch(ex):
    if "batch" in ex:
        return ex
    N = ex["pos"].shape[0]
    b = dict(ex, batch=torch.zeros(N, dtype=torch.int64, device="cuda"),
             num_atoms=torch.tensor([N], device="cuda"))
    if "cell" in ex:
        b["cell"] = ex["cell"].reshape(1, 3, 3)
    b["pbc"] = torch.as_tensor(ex.get("pbc", "cell" in ex)).reshape(-1).expand(3).reshape(1, 3)
    return b


def _eager(model, ex, pos, cell, stress):
    kw = {"batch": ex["batch"]}
    if model.per_edge_type_cutoff is not None:
        kw.update(atom_types=ex["atom_types"], edge_type_cutoff=model.per_edge_type_cutoff)
    nl = ops.neighbor_list(pos, cell, ex["pbc"], R_MAX, **kw)
    d = {"pos": pos, "atom_types": ex["atom_types"], "batch": ex["batch"], "num_atoms": ex["num_atoms"],
         "edge_index": nl["edge_index"], "edge_cell_shift": nl["edge_cell_shift"]}
    if cell is not None:
        d["cell"] = cell
    out = model(d, compute_stress=True) if stress else model(d)
    vir = out["virial"].detach().double().cpu().numpy() if stress else None
    return (out["total_energy"].detach().double().view(-1).cpu().numpy(), out["forces"].detach().double().cpu().numpy(),
            vir)


def _host_relax(model, ex, n, filt, p=0.0, fmax=0.05):
    """The oracle frames after n steps of the host loop (eager list + model + oracle FIRE)."""
    counts = ex["num_atoms"].cpu().tolist()
    ptr = [0] + np.cumsum(counts).tolist()
    pos = ex["pos"].double().cpu().numpy()
    _, pbc, cells = ops._nl_frame_args(ex.get("cell"), ex["pbc"].cpu(), ex["batch"].cpu(), len(pos))
    frames = [ro.Frame(pos[ptr[f]:ptr[f + 1]], cells[f], filt, fmax=fmax, p=p) for f in range(len(counts))]
    has_cell = ex.get("cell") is not None
    for it in range(n + 1):
        P = torch.tensor(np.concatenate([fr.positions() for fr in frames]), device="cuda")
        C = torch.tensor(np.stack([fr.cell() for fr in frames]), device="cuda") if has_cell else None
        e, forces, vir = _eager(model, ex, P, C, filt)
        for f, fr in enumerate(frames):
            fr.evaluate(float(e[f]), forces[ptr[f]:ptr[f + 1]], vir[f] if filt else None)
        if it < n:
            for fr in frames:
                fr.step()
    return frames


RELAX_CASES = [("water", None, 0.0), ("slab", None, 0.0), ("molecule", None, 0.0), ("mixed_batch", None, 0.0),
               ("water", "frechet", 0.0), ("water", "frechet", 0.02), ("li3po4_zbl_table", "frechet", 0.0),
               ("li3po4_zbl_table", "frechet", 0.01)]


@pytest.mark.parametrize("kind,filt,p", RELAX_CASES, ids=[f"{k}-{f or 'positions'}-p{p}" for k, f, p in RELAX_CASES])
def test_graphed_relax_matches_the_host_loop(kind, filt, p):
    ex, model = _system(kind)[:2]
    ex = _as_batch(ex)
    if kind == "mixed_batch":
        ex["pos"] = ex["pos"].double()
    kw = {} if filt is None else dict(cell_filter=filt, scalar_pressure=p)
    r = GraphedRelax(model, ex, fmax=1e-6, **kw)
    res = r.run(N_STEPS, block=7)
    frames = _host_relax(model, ex, N_STEPS, filt is not None, p, fmax=1e-6)
    ref_pos = np.concatenate([fr.positions() for fr in frames])
    assert np.abs(res["pos"].numpy() - ref_pos).max() <= POS_TOL
    if filt is not None:
        ref_cell = np.stack([fr.cell() for fr in frames])
        assert np.abs(res["cell"].numpy() - ref_cell).max() <= POS_TOL
    assert res["steps"].tolist() == [fr.steps for fr in frames]
    last = res["log"]
    ref_log = np.array([fr.log for fr in frames])
    for j, name in enumerate(("e_pot", "enthalpy", "fmax", "volume")):
        scale = max(1.0, float(np.abs(ref_log[:, j]).max()))
        assert np.abs(last[name][-1].numpy() - ref_log[:, j]).max() <= 1e-7 * scale, name
    assert r.host_reads == math.ceil(N_STEPS / 7) + r.recaptures  # a rolled-back block is read twice


# ------------------------------------------------------------------------------------------------------------------
# bookkeeping
# ------------------------------------------------------------------------------------------------------------------
def test_frames_converge_at_different_steps_and_stay_frozen():
    ex, model = _system("mixed_batch")[:2]
    ex["pos"] = ex["pos"].double()
    r = GraphedRelax(model, ex, fmax=0.02)
    seen = {}
    for _ in range(12):
        res = r.run(10, block=10)
        for f in range(r.num_frames):
            a, b = r._atom_ptr[f].item(), r._atom_ptr[f + 1].item()
            if bool(res["converged"][f]) and f not in seen:
                seen[f] = res["pos"][a:b].clone()
            elif f in seen:
                assert torch.equal(res["pos"][a:b], seen[f])
        if bool(res["converged"].all()):
            break
    assert len(set(res["steps"].tolist())) > 1  # different steps to converge


def test_block_sizes_agree_and_run_stops_within_a_block():
    ex, model = _system("molecule")[:2]
    ex = _as_batch(ex)
    out = {}
    for block in (1, 7, 50):
        r = GraphedRelax(model, ex, fmax=0.05)
        out[block] = r.run(1000, block=block)
        res = out[block]
        assert bool(res["converged"].all())
        n = res["log"]["fmax"].shape[0]
        assert n - block < int(res["steps"].max()) <= n
    for block in (7, 50):
        assert torch.equal(out[block]["steps"], out[1]["steps"])
        assert (out[block]["pos"] - out[1]["pos"]).abs().max() <= POS_TOL * 10


def test_zero_steps_max_steps_and_failure():
    ex, model = _system("molecule")[:2]
    ex = _as_batch(ex)
    r = GraphedRelax(model, ex, fmax=1e6)
    res = r.run(20)
    assert bool(res["converged"].all()) and res["steps"].tolist() == [0] and r.host_reads == 0
    r = GraphedRelax(model, ex, fmax=1e-9)
    res = r.run(5, block=2)
    assert not bool(res["converged"].any()) and res["steps"].tolist() == [5]
    r = GraphedRelax(model, ex, fmax=1e-9, fail_force=1e-6)
    res = r.run(5)
    assert bool(res["failed"].all()) and res["steps"].tolist() == [0]


def test_recapture_from_half_capacity_matches_a_large_capacity_run():
    ex, model = _system("water")[:2]
    ex = _as_batch(ex)
    e0 = ops.neighbor_list(ex["pos"], ex["cell"], True, R_MAX, batch=ex["batch"])["edge_index"].shape[1]
    kw = dict(fmax=1e-6, cell_filter="frechet", scalar_pressure=0.05)  # the pressure compresses the cell
    small = GraphedRelax(model, ex, capacity=e0 // 2, **kw)
    a = small.run(20, block=5)
    big = GraphedRelax(model, ex, capacity=4 * e0, **kw)
    b = big.run(20, block=5)
    assert small.recaptures >= 1 and big.recaptures == 0
    assert float(a["log"]["volume"][-1, 0]) < float(a["log"]["volume"][0, 0])
    assert (a["pos"] - b["pos"]).abs().max() <= POS_TOL
    assert torch.equal(a["steps"], b["steps"])
