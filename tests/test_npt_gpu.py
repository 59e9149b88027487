"""``GraphedNPT`` and the nqb_npt kernels on the GPU: every kernel against one step of the float64 oracle
(tests/npt_oracle.py) with its write contract, float64 trajectories against a host loop of the oracle around
``ops.neighbor_list`` and the eager model with stress, a float32 model, frame independence, blocks and the log ring,
rollback, NPH energy drift and time reversal, and the error flag.

As in tests/test_md_trajectory_gpu.py, under ``ops.set_deterministic(True)`` a float64 model's graphed forces agree
with its eager forces to F64_AGREE max|F|, and its virial (a sum over the same edge forces) to F64_AGREE max|virial|.
``_bounds`` carries that agreement through n steps of the NPT update to first order, with the same factor 10 of slack
for the growth of a difference through the forces; nothing in it is fitted.  The largest error / bound seen on an H100
is in each docstring."""
import math

import numpy as np
import pytest
import torch

import md_oracle as mo
import npt_oracle as no
from batched_oracle import concat_frames
from cell_frames import cell_frame
from kernel_contracts import guarded
from nequip_b200 import _capi, ops
from nequip_b200.npt import GPA, LOG_FIELDS, GraphedNPT
from test_batched_md_step_gpu import _mixed_frames
from test_batched_md_step_gpu import _model as _model_any
from test_md_run_gpu import F_AGREE, R_MAX, _case
from test_md_trajectory_gpu import _system

pytestmark = pytest.mark.gpu

F64_AGREE = 1e-12
DT_FS = 0.5
LI3PO4_MASSES = [6.94, 30.974, 15.999]


@pytest.fixture(autouse=True)
def _deterministic():
    prev = ops.deterministic()
    ops.set_deterministic(True)
    yield
    ops.set_deterministic(prev)


# ------------------------------------------------------------------------------------------------------------------
# kernels against one oracle step
# ------------------------------------------------------------------------------------------------------------------
def _kernel_cases():
    cases = []
    for name, counts in (("cta_edges", [255, 256, 257]), ("above_64_ctas", [16385, 3])):
        driver = min(64, -(-max(counts) // 256))
        for nblk in sorted({1, 2, driver}):
            for M, Mp in ((0, 0), (1, 3), (3, 1), (3, 3)):
                cases.append(pytest.param(counts, nblk, M, Mp, id=f"{name}-nblk{nblk}-t{M}p{Mp}"))
    return cases


@pytest.mark.parametrize("counts,nblk,M,Mp", _kernel_cases())
def test_kernels_match_one_oracle_step_and_write_only_their_outputs(counts, nblk, M, Mp):
    """pre, move, kick (new forces), post (new virial), scale and log against one oracle step, tloop = ploop = 2, on a
    state with every barostat and chain variable non-zero; each output within 1e-14 of its magnitude, and no kernel
    writes outside its buffers."""
    rng = np.random.default_rng(sum(counts) + nblk + 10 * M + Mp)
    F, N = len(counts), sum(counts)
    C0 = torch.tensor(np.stack([np.diag([20.0, 21.0, 22.0]) + rng.standard_normal((3, 3)) for _ in counts]))
    prm = no.Params(counts, C0, [300.0 + 50 * f for f in range(F)], [0.01 * (f - 1) for f in range(F)],
                    [40.0 * mo.FS] * F, [300.0 * mo.FS + f for f in range(F)], M, Mp, 2, 2)
    t = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
    mass = t(rng.uniform(1.0, 30.0, N))
    w0 = rng.standard_normal((F, 3, 3))
    st = no.State(t(rng.standard_normal((N, 3)) * 10), t(rng.standard_normal((N, 3)) * 0.05),
                  t(rng.standard_normal((N, 3))), mass, t(w0 + w0.transpose(0, 2, 1)) * 5, prm)
    for f in range(F):
        st.eps[f], st.veps[f] = 0.01 * rng.standard_normal(), 0.02 * rng.standard_normal()
        st.K2[f] *= 1.0 + 1e-3 * f  # the tracked K2 need not be the recomputed one
        for xs in (st.xi[f], st.vxi[f], st.eta[f], st.veta[f]):
            xs[:] = (0.1 * rng.standard_normal(len(xs))).tolist()
    st.cell = prm.C0 * t([math.exp(e) for e in st.eps]).view(F, 1, 1)
    f1 = t(rng.standard_normal((N, 3)))
    w1 = rng.standard_normal((F, 3, 3))
    vir1 = t(w1 + w1.transpose(0, 2, 1)) * 5
    e1 = t(rng.standard_normal(F))
    cu = dict(device="cuda")
    d_pos, c_pos = guarded(N, 3, torch.float64, body=st.pos, **cu)
    d_vel, c_vel = guarded(N, 3, torch.float64, body=st.vel, **cu)
    d_frc, c_frc = guarded(N, 3, torch.float64, body=st.forces, **cu)
    d_st, c_st = guarded(F, no.MAX_CHAIN * 4 + 3, torch.float64, body=st.rows(), **cu)
    d_vir, c_vir = guarded(F, 9, torch.float64, body=st.vir.reshape(F, 9), **cu)
    d_cell, c_cell = guarded(F, 9, torch.float64, body=st.cell.reshape(F, 9), **cu)
    d_coef, c_coef = guarded(F, 7, torch.float64, **cu)
    d_err, c_err = guarded(F, 1, torch.int32, body=torch.zeros(F, 1, dtype=torch.int32), **cu)
    d_work, c_work = guarded(F, no.MAX_CHAIN * 4 + 3, torch.float64, **cu)
    d_part, c_part = guarded(F * nblk, 1, torch.float64, **cu)
    d_log, c_log = guarded(2 * F, 6, torch.float64, **cu)
    dprm, dC0, aptr = prm.table().cuda(), prm.C0.reshape(F, 9).cuda(), torch.tensor(prm.ptr).cuda()
    dmass, df1, dvir1, de1 = mass.cuda(), f1.cuda(), vir1.reshape(F, 9).cuda(), e1.cuda()
    zero64, zero32 = torch.zeros(1, dtype=torch.int64, **cu), torch.zeros(1, dtype=torch.int32, **cu)
    one32 = torch.ones(1, dtype=torch.int32, **cu)
    step = torch.zeros(1, dtype=torch.int64, **cu)
    flags = torch.tensor([0, 0, -1, 0], dtype=torch.int64, **cu)
    P, L, s = ops._ptr, _capi.lib(), ops._stream()
    dt = DT_FS * mo.FS
    _capi.check(L.nqb_npt_pre(F, M, Mp, 2, 2, dt, P(dprm), P(dC0), P(d_vir), P(d_st), P(d_cell), P(d_coef), P(d_err),
                              P(d_work), s))
    _capi.check(L.nqb_npt_move(F, nblk, P(aptr), P(dmass), P(d_frc), P(d_coef), P(d_pos), P(d_vel), s))
    _capi.check(L.nqb_npt_kick(F, nblk, P(aptr), P(dmass), P(df1), P(d_coef), P(d_vel), P(d_frc), P(d_part), s))
    _capi.check(L.nqb_npt_post(F, nblk, M, Mp, 2, 2, dt, P(dprm), P(d_part), P(dvir1), P(d_st), P(d_vir), P(d_coef),
                               P(d_err), P(d_work), s))
    _capi.check(L.nqb_npt_scale(F, nblk, P(aptr), P(d_coef), P(d_vel), s))
    _capi.check(L.nqb_npt_log(F, M, Mp, P(de1), P(dprm), P(d_st), P(d_vir), P(zero64), P(zero32), P(one32), 2,
                              P(step), P(d_log), P(flags), s))
    torch.cuda.synchronize()
    for c in (c_pos, c_vel, c_frc, c_st, c_vir, c_cell, c_coef, c_err, c_work, c_part, c_log):
        c()
    no.step(st, prm, dt, lambda pos, cell: (e1, f1, vir1))

    def close(got, ref, what):
        ref = ref.double().cpu()
        got = got.cpu().reshape(ref.shape)
        assert not torch.isnan(got).any(), what
        err = (got - ref).abs()
        tol = 1e-14 * max(1.0, float(ref.abs().max()))
        assert float(err.max()) <= tol, (what, float(err.max()), tol, torch.nonzero(err > tol)[:5].tolist())

    close(d_pos, st.pos, "pos")
    close(d_vel, st.vel, "vel")
    close(d_frc, f1, "forces")
    close(d_st, st.rows(), "state")
    close(d_vir, st.vir.reshape(F, 9), "virial")
    close(d_cell, st.cell.reshape(F, 9), "cell")
    close(d_log.view(2, F, 6)[0], no.log_row(st, prm), "log")
    assert int(d_err.sum()) == 0 and int(step) == 1 and flags.cpu().tolist() == [0, 0, -1, 0]


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int64) if t.dtype == torch.float64 else t


@pytest.mark.parametrize("nblk", [1, 2])
def test_frozen_frames_keep_their_state_and_atoms(nblk):
    """The frozen paths of the kernels, on guarded buffers: frame 0 enters with err set, frame 2 with a NaN v_eps (pre
    finds a non-finite update), frame 1 gets a NaN virial from the model (post finds it), frame 3 is an ordinary frame.
    pre gives frames 0 and 2 the coefficients {1, 1, 0, 1, 0, 0, 1} and leaves their state rows and cells bitwise as
    they were; move, kick and scale leave their atoms untouched and kick writes 0 into their partial sums; post flags
    frame 1, sets its final scale to 1 and leaves its state row (as pre left it) and its virial unchanged, so scale
    leaves its velocities as kick left them; frame 3 takes the step."""
    rng = np.random.default_rng(nblk)
    counts = [5, 300, 7, 9]
    F, N = len(counts), sum(counts)
    C0 = torch.tensor(np.stack([np.diag([12.0, 13.0, 14.0]) + 0.3 * rng.standard_normal((3, 3)) for _ in counts]))
    prm = no.Params(counts, C0, 300.0, 0.01, 40.0 * mo.FS, 300.0 * mo.FS, 3, 3, 2, 2)
    t = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
    mass = t(rng.uniform(1.0, 30.0, N))
    w0 = rng.standard_normal((F, 3, 3))
    st = no.State(t(rng.standard_normal((N, 3)) * 5), t(rng.standard_normal((N, 3)) * 0.05),
                  t(rng.standard_normal((N, 3))), mass, t(w0 + w0.transpose(0, 2, 1)), prm)
    for f in range(F):
        st.veps[f] = 0.01 * (f + 1)
    st.veps[2] = float("nan")
    rows0 = st.rows()
    cu = dict(device="cuda")
    d_pos, c_pos = guarded(N, 3, torch.float64, body=st.pos, **cu)
    d_vel, c_vel = guarded(N, 3, torch.float64, body=st.vel, **cu)
    d_frc, c_frc = guarded(N, 3, torch.float64, body=st.forces, **cu)
    d_st, c_st = guarded(F, no.MAX_CHAIN * 4 + 3, torch.float64, body=rows0, **cu)
    d_vir, c_vir = guarded(F, 9, torch.float64, body=st.vir.reshape(F, 9), **cu)
    d_cell, c_cell = guarded(F, 9, torch.float64, body=st.cell.reshape(F, 9), **cu)
    d_coef, c_coef = guarded(F, 7, torch.float64, **cu)
    d_err, c_err = guarded(F, 1, torch.int32, body=torch.tensor([[1], [0], [0], [0]], dtype=torch.int32), **cu)
    d_work, c_work = guarded(F, no.MAX_CHAIN * 4 + 3, torch.float64, **cu)
    d_part, c_part = guarded(F * nblk, 1, torch.float64, **cu)
    dprm, dC0, aptr = prm.table().cuda(), prm.C0.reshape(F, 9).cuda(), torch.tensor(prm.ptr).cuda()
    dmass = mass.cuda()
    f1 = torch.randn(N, 3, generator=torch.Generator().manual_seed(nblk), dtype=torch.float64).cuda()
    vir1 = torch.randn(F, 9, generator=torch.Generator().manual_seed(9), dtype=torch.float64).cuda()
    vir1[1, 4] = float("nan")
    P, L, s_ = ops._ptr, _capi.lib(), ops._stream()
    dt = DT_FS * mo.FS
    ptr = prm.ptr
    at = lambda x, f: x[ptr[f]:ptr[f + 1]]  # noqa: E731
    pos0, vel0, frc0, cell0, vir0 = (d_pos.clone(), d_vel.clone(), d_frc.clone(), d_cell.clone(), d_vir.clone())
    _capi.check(L.nqb_npt_pre(F, 3, 3, 2, 2, dt, P(dprm), P(dC0), P(d_vir), P(d_st), P(d_cell), P(d_coef), P(d_err),
                              P(d_work), s_))
    torch.cuda.synchronize()
    frozen = torch.tensor([1, 1, 0, 1, 0, 0, 1], dtype=torch.float64)
    for f in (0, 2):
        assert torch.equal(d_coef[f].cpu(), frozen), f
        assert torch.equal(_bits(d_st[f]), _bits(rows0[f])) and torch.equal(d_cell[f], cell0[f]), f
    assert d_err.view(-1).cpu().tolist() == [1, 0, 1, 0]
    assert float(d_coef[1, 5]) == 1.0 and float(d_coef[3, 5]) == 1.0
    st_pre = d_st.clone()
    _capi.check(L.nqb_npt_move(F, nblk, P(aptr), P(dmass), P(d_frc), P(d_coef), P(d_pos), P(d_vel), s_))
    _capi.check(L.nqb_npt_kick(F, nblk, P(aptr), P(dmass), P(f1), P(d_coef), P(d_vel), P(d_frc), P(d_part), s_))
    torch.cuda.synchronize()
    vel_kick = d_vel.clone()
    _capi.check(L.nqb_npt_post(F, nblk, 3, 3, 2, 2, dt, P(dprm), P(d_part), P(vir1), P(d_st), P(d_vir), P(d_coef),
                               P(d_err), P(d_work), s_))
    _capi.check(L.nqb_npt_scale(F, nblk, P(aptr), P(d_coef), P(d_vel), s_))
    torch.cuda.synchronize()
    for c in (c_pos, c_vel, c_frc, c_st, c_vir, c_cell, c_coef, c_err, c_work, c_part):
        c()
    assert d_err.view(-1).cpu().tolist() == [1, 1, 1, 0]
    part = d_part.view(F, nblk).cpu()
    for f in (0, 2):
        for x, x0 in ((d_pos, pos0), (d_vel, vel0), (d_frc, frc0)):
            assert torch.equal(at(x, f), at(x0, f)), f
        assert torch.equal(part[f], torch.zeros(nblk, dtype=torch.float64))
        assert torch.equal(_bits(d_st[f]), _bits(rows0[f])) and torch.equal(d_vir[f], vir0[f])
        assert torch.equal(d_cell[f], cell0[f])
    assert float(d_coef[1, 6]) == 1.0
    assert torch.equal(d_st[1], st_pre[1]) and torch.equal(d_vir[1], vir0[1])
    assert torch.equal(at(d_vel, 1), at(vel_kick, 1)) and torch.equal(at(d_frc, 1), at(f1, 1))
    assert not torch.equal(at(d_pos, 1), at(pos0, 1)) and bool(torch.isfinite(d_pos).all())
    assert torch.equal(d_vir[3], vir1[3]) and not torch.equal(d_st[3], st_pre[3])
    assert bool(torch.isfinite(d_st[3]).all()) and not torch.equal(d_cell[3], cell0[3])


# ------------------------------------------------------------------------------------------------------------------
# systems, the host loop and the bound
# ------------------------------------------------------------------------------------------------------------------
def _as_batch(ex):
    if "batch" in ex:
        return ex
    N = ex["pos"].shape[0]
    return dict(ex, batch=torch.zeros(N, dtype=torch.int64, device="cuda"), num_atoms=torch.tensor([N], device="cuda"),
                cell=ex["cell"].reshape(1, 3, 3), pbc=torch.ones(1, 3, dtype=torch.bool))


def _npt_system(kind, dtype=torch.float64):
    """(batched example on cuda, model, masses, {temperature, pressure, tdamp_fs, pdamp_fs})."""
    bath = dict(temperature=300.0, pressure=1.0 * GPA, tdamp_fs=50.0, pdamp_fs=200.0)
    if kind in ("water", "li3po4_zbl_table"):
        ex, model, masses = _system(kind)[:3]
        if dtype == torch.float32:
            ex, meta = _case(kind)
            model = _model_any(meta["type_names"], torch.float32, meta["avg_num_neighbors"])
        return _as_batch(ex), model, masses, bath
    names = ["Li", "P", "O"]
    if kind == "left_handed":
        d = cell_frame("li3po4", 3, "left", seed=3, outside=True)
        meta = d.pop("_meta")
        ex = {k: d[k].cuda() for k in ("pos", "atom_types", "cell")}
        return _as_batch(ex), _model_any(names, torch.float64, meta["avg_num_neighbors"]), LI3PO4_MASSES, bath
    # periodic frames of different sizes: cubic, tilted, left-handed, small, one atom
    frames, pbcs = _mixed_frames()
    keep = [0, 1, 3, 4, 7]
    b = concat_frames([frames[k] for k in keep], [pbcs[k] for k in keep])
    ann = b["edge_index"].shape[1] / b["pos"].shape[0]
    ex = {k: b[k].cuda() for k in ("pos", "atom_types", "cell", "batch", "num_atoms", "pbc")}
    bath = dict(temperature=[300.0, 450.0, 200.0, 600.0, 350.0], pressure=[0.0, 2 * GPA, -0.5 * GPA, 5 * GPA, GPA],
                tdamp_fs=[50.0, 30.0, 80.0, 40.0, 60.0], pdamp_fs=[200.0, 150.0, 400.0, 250.0, 300.0])
    return ex, _model_any(names, torch.float64, ann), LI3PO4_MASSES, bath


def _eager(model, ex, pos, cell):
    """(E_pot [F], forces [N, 3], virial [F, 3, 3]) of ``ops.neighbor_list`` and the eager model with stress."""
    kw = {"batch": ex["batch"]}
    if model.per_edge_type_cutoff is not None:
        kw.update(atom_types=ex["atom_types"], edge_type_cutoff=model.per_edge_type_cutoff)
    cell = cell.to("cuda", torch.float64).reshape(-1, 3, 3)
    nl = ops.neighbor_list(pos, cell, ex["pbc"], R_MAX, **kw)
    d = {"pos": pos, "atom_types": ex["atom_types"], "batch": ex["batch"], "num_atoms": ex["num_atoms"],
         "edge_index": nl["edge_index"], "edge_cell_shift": nl["edge_cell_shift"], "cell": cell}
    out = model(d, compute_stress=True)
    return (out["total_energy"].detach().double().view(-1), out["forces"].detach().double(),
            out["virial"].detach().double().reshape(-1, 3, 3).cpu())


def _start(system, tchain=3, pchain=3, capacity=None, seed=7, **over):
    ex, model, masses, bath = system
    bath = dict(bath, **over)
    m = GraphedNPT(model, ex, masses, DT_FS, bath["temperature"], bath["pressure"], tdamp_fs=bath["tdamp_fs"],
                   pdamp_fs=bath["pdamp_fs"], tchain=tchain, pchain=pchain, capacity=capacity, seed=seed)
    counts = ex["num_atoms"].cpu().tolist()
    prm = no.Params(counts, ex["cell"].cpu(), bath["temperature"], bath["pressure"],
                    torch.tensor(bath["tdamp_fs"], dtype=torch.float64) * mo.FS,
                    torch.tensor(bath["pdamp_fs"], dtype=torch.float64) * mo.FS, tchain, pchain)
    e0, f0, v0 = _eager(model, ex, ex["pos"].double(), ex["cell"])
    st = no.State(ex["pos"].double(), m.state["vel"].clone(), f0, m._mass, v0, prm)
    st.e_pot = e0.tolist()
    return m, st, prm


def _host_loop(model, ex, st, prm, n, dt):
    """n oracle steps around the eager list and model: the states after every step and the log rows [n, F, 6]."""
    st = st.clone()
    states, rows = [], []
    for _ in range(n):
        no.step(st, prm, dt, lambda p, c: _eager(model, ex, p, c))
        states.append(st.clone())
        rows.append(no.log_row(st, prm))
    return states, torch.stack(rows)


def _stiffness(model, ex, st0):
    """K_b = max over frames of |d tr(virial) / d eps| at the initial state (central difference of the eager model over
    an affine scaling by e^{+-1e-5}): (eps, v_eps) is an oscillator of frequency sqrt(K_b / W)."""
    h = 1e-5
    tr = []
    for s in (h, -h):
        g = math.exp(s)
        tr.append(_eager(model, ex, st0.pos * g, st0.cell * g)[2].diagonal(dim1=1, dim2=2).sum(1))
    return float(((tr[0] - tr[1]) / (2 * h)).abs().max())


def _virial_gradient(model, ex, st0, h=1e-5, chunk_atoms=30000):
    """G_x = max over frames of sum_i |d tr(virial) / d x_i| (every coordinate of every atom of the frame) at the
    initial state, by central differences of the eager model: the change of tr(virial) that a non-affine position
    difference dx causes is at most G_x dx.  The displaced copies of the batch are evaluated as one larger batch,
    coordinate c of every frame (that has it) displaced in the same copy."""
    counts = ex["num_atoms"].cpu().tolist()
    ptr = [0] + torch.tensor(counts).cumsum(0).tolist()
    F, N = len(counts), st0.pos.shape[0]
    C = 3 * max(counts)
    jobs = [(c, sg) for c in range(C) for sg in (1.0, -1.0)]
    K = max(1, chunk_atoms // N)
    tr = torch.zeros(len(jobs), F, dtype=torch.float64)
    for a in range(0, len(jobs), K):
        part = jobs[a:a + K]
        k = len(part)
        pos = st0.pos.repeat(k, 1)
        for j, (c, sg) in enumerate(part):
            for f in range(F):
                if c < 3 * counts[f]:
                    pos[j * N + ptr[f] + c // 3, c % 3] += sg * h
        big = {"atom_types": ex["atom_types"].repeat(k), "num_atoms": ex["num_atoms"].repeat(k),
               "pbc": ex["pbc"].reshape(F, 3).repeat(k, 1),
               "batch": ex["batch"].repeat(k) + F * torch.arange(k, device="cuda").repeat_interleave(N)}
        vir = _eager(model, big, pos, st0.cell.repeat(k, 1, 1))[2]
        tr[a:a + k] = vir.diagonal(dim1=1, dim2=2).sum(1).reshape(k, F)
    g = (tr[0::2] - tr[1::2]) / (2 * h)  # [C, F]
    mask = torch.arange(C).unsqueeze(1) < 3 * torch.tensor(counts).unsqueeze(0)
    return float((g.abs() * mask).sum(0).max())


def _bounds(n, dt, prm, st0, states, log, agree=F64_AGREE, stiff=0.0, grad=0.0):
    """Bounds after n steps on two trajectories from one state whose forces agree to e = agree max|F| and whose virials
    agree to ew = agree max(max|virial|, N max|F| r_max) (a sum of edge terms rounds with the sum of their sizes), to
    first order with a factor 10 of slack:
      v: n dt e / m_min (forces) + 2 n dt v_max dv_eps (the barostat's friction);   K2: 2 N m_max (v_max + dv) dv;
      tr(virial): 3 ew + grad dx_n + stiff deps, where dx_n = n^2 dt^2 e / m_min + 1e-12 is the non-affine part of
        the position difference (``_virial_gradient``; 0 when not given) and the affine part r deps changes tr(virial)
        by stiff deps (``_stiffness``);
      v_eps: n dt (2 dK2 + dtr) / W_min times the growth e^{omega n dt} of a difference through the oscillators
        it is part of: the cell, sqrt(stiff / W_min) (``_stiffness``; 0 when not given), the barostat chain,
        sqrt(2 W_max v_eps,max^2 / Q'_1,min), and the particle chain, sqrt(2 K2_max / Q_1,min), plus the friction
        rates |v_eta|_max + |v_xi|_max + alpha |v_eps|_max of the linearised equations (a Gronwall bound);
      eps: n dt dv_eps;
      positions: n^2 dt^2 e / m_min + r_max deps;
      v_xi: n dt dK2 / Q_min;   xi: n dt dv_xi;   v_eta: n dt 2 W_max v_eps,max dv_eps / Q'_min;   eta: n dt dv_eta.
    The log follows: E_pot N max|F| dx + max|tr virial| deps; E_kin dK2 / 2; T dK2 / (N_f k_B)_min; V 3 V_max deps;
    pressure (dK2 + dtr) / (3 V_min) + 3 p_max deps; H the sum of its terms' first-order changes.  Every energy also
    carries agree of its largest magnitude and positions and velocities 1e-12 (the update's own rounding).  Returns a
    dict of bounds by state and log field."""
    mass = st0.mass
    N, m_min, m_max = mass.numel(), float(mass.min()), float(mass.max())
    fmax = max(float(s.forces.abs().max()) for s in [st0] + states)
    wmax = max(float(s.vir.abs().max()) for s in [st0] + states)
    vmax = max(float(s.vel.abs().max()) for s in [st0] + states)
    rmax = max(float(s.pos.abs().max()) for s in [st0] + states)
    veps = max(abs(v) for s in states for v in s.veps)
    vxi = max([abs(v) for s in states for r in s.vxi for v in r] + [0.0])
    veta = max([abs(v) for s in states for r in s.veta for v in r] + [0.0])
    # the virial is a sum of edge terms r_ij f_ij with |r_ij| <= r_max: its rounding scales with N max|F| r_max
    e, ew = agree * fmax, agree * max(wmax, N * fmax * R_MAX)
    W_min, W_max = min(prm.W), max(prm.W)
    dv0 = 10 * n * dt * e / m_min + 1e-12
    dK = 2 * N * m_max * (vmax + dv0) * dv0 + agree * max(max(s.K2) for s in states)
    # the oscillators a difference in v_eps grows through: the cell (stiff / W), the barostat chain
    # (d G'_1 / d v_eps * v_eps = 2 W v_eps^2 / Q') and, through K2, the particle chain (2 K2 / Q_1)
    K2max = max(max(s.K2) for s in [st0] + states)
    omega = math.sqrt(stiff / W_min)
    if prm.Qp[0]:
        omega += math.sqrt(2 * W_max * veps * veps / min(r[0] for r in prm.Qp))
    if prm.Q[0]:
        omega += math.sqrt(2 * K2max / min(r[0] for r in prm.Q))
    omega += veta + vxi + 2 * veps  # the friction terms of the linearised equations (Gronwall: their row sum)
    dxn = 10 * n * n * dt * dt * e / m_min + 1e-12
    dtr0 = 3 * ew + grad * dxn  # before the affine part, which the growth through the cell's oscillator covers
    dveps = 10 * n * dt * (2 * dK + dtr0) / W_min * math.exp(omega * n * dt)
    deps = n * dt * dveps
    dtr = dtr0 + stiff * deps
    dv = dv0 + 20 * n * dt * vmax * dveps + 1e-12
    dx = dxn + rmax * deps
    Qs = [q for r in prm.Q for q in r]
    Qps = [q for r in prm.Qp for q in r]
    dvxi = 10 * n * dt * dK / min(Qs) if Qs else 0.0
    dxi = n * dt * dvxi
    dveta = 10 * n * dt * 2 * W_max * veps * dveps / min(Qps) if Qps else 0.0
    deta = n * dt * dveta
    mag = log.abs().amax(dim=(0, 1)).tolist()
    V_max, V_min = max(mag[3], 1e-300), float(log[:, :, 3].min())
    kT, p_max = max(prm.kT), max(abs(p) for p in prm.P)
    de = N * fmax * dx + 3 * wmax * deps + agree * mag[0]
    dh = (de + dK / 2 + W_max * veps * dveps + p_max * 3 * V_max * deps
          + len(Qs) * (max(Qs + [0.0]) * vxi * dvxi + max(prm.Nf) * kT * dxi)
          + len(Qps) * (max(Qps + [0.0]) * veta * dveta + kT * deta) + agree * mag[5])
    return {"pos": dx, "vel": dv, "eps": deps, "v_eps": dveps, "xi": dxi, "v_xi": dvxi, "eta": deta, "v_eta": dveta,
            "e_pot": de, "e_kin": dK / 2 + agree * mag[1], "temperature": dK / min(prm.NfkB) + agree * mag[2],
            "volume": 3 * V_max * deps + agree * mag[3],
            "pressure": (dK + dtr) / (3 * V_min) + 3 * mag[4] * deps + agree * mag[4], "conserved": dh,
            "tr_virial": dtr, "dx_nonaffine": dxn}


def _close(got, want, bound, what):
    got, want = got.detach().double().cpu(), torch.as_tensor(want).detach().double().cpu().reshape(got.shape)
    err = float((got - want).abs().max()) if want.numel() else 0.0
    assert err <= bound, f"{what}: max |err| {err:.3g} > bound {bound:.3g}"
    return err / bound if bound > 0 else 0.0


def _check_state(m, ref: "no.State", b, what):
    """The driver's state against an oracle state, to bounds ``b``; returns the largest error / bound."""
    s = m.state
    F = m.num_frames
    r = [_close(s["pos"], ref.pos, b["pos"], f"{what} pos"), _close(s["vel"], ref.vel, b["vel"], f"{what} vel"),
         _close(s["eps"], torch.tensor(ref.eps, dtype=torch.float64), b["eps"], f"{what} eps"),
         _close(s["v_eps"], torch.tensor(ref.veps, dtype=torch.float64), b["v_eps"], f"{what} v_eps"),
         _close(s["virial"].diagonal(dim1=1, dim2=2).sum(1), ref.vir.diagonal(dim1=1, dim2=2).sum(1), b["tr_virial"],
                f"{what} tr(virial)"),
         _close(s["cell"], ref.cell, 3 * float(ref.cell.abs().max()) * b["eps"] + 1e-13, f"{what} cell")]
    for k, name in (("xi", "xi"), ("vxi", "v_xi"), ("eta", "eta"), ("veta", "v_eta")):
        want = torch.tensor(getattr(ref, k), dtype=torch.float64).reshape(F, -1)
        r.append(_close(s[name], want, b[name], f"{what} {name}"))
    return max(r)


def _check_log(log, want, b, what):
    return max(_close(log[name], want[:, :, j], b[name], f"{what} {name}") for j, name in enumerate(LOG_FIELDS))


# ------------------------------------------------------------------------------------------------------------------
# trajectories against the host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["water", "li3po4_zbl_table", "left_handed", "mixed_batch"])
def test_float64_trajectory_matches_the_host_loop(kind):
    """40 steps of 0.5 fs in blocks of 16 with both chains: F(0) and the virial right after construction against the
    test's own eager call, the state at the end of every block (positions, velocities, eps, v_eps, tr(virial), the
    chains) and every log row against the host loop, to ``_bounds`` with the virial's dependence on the positions
    (``_virial_gradient``) and the growth through the cell's and the chains' oscillators.  The oracle's per-frame
    scalars are Python floats: they are compared as float64 tensors (``torch.tensor`` of a list is float32, which
    rounds a v_eps of 5e-3 by 2e-10)."""
    system = _npt_system(kind)
    ex, model = system[:2]
    m, st0, prm = _start(system)
    _close(m.state["forces"], st0.forces, F64_AGREE * float(st0.forces.abs().max()), f"{kind} F(0)")
    _close(m.state["virial"], st0.vir, F64_AGREE * float(st0.vir.abs().max()) + 1e-300, f"{kind} virial(0)")
    n, block = 40, 16
    ends = []
    log = m.run(n, block=block, on_block=lambda b: ends.append({k: v.clone() for k, v in m.state.items()}))
    states, want = _host_loop(model, ex, st0, prm, n, m.dt)
    stiff, grad = _stiffness(model, ex, st0), _virial_gradient(model, ex, st0)
    worst = 0.0
    for k, got in enumerate(ends):
        s = min(n, (k + 1) * block)
        b = _bounds(s, m.dt, prm, st0, states[:s], want[:s], stiff=stiff, grad=grad)
        worst = max(worst, _close(got["pos"], states[s - 1].pos, b["pos"], f"{kind} pos after {s}"),
                    _close(got["vel"], states[s - 1].vel, b["vel"], f"{kind} vel after {s}"))
        assert int(got["step"]) == s
    b = _bounds(n, m.dt, prm, st0, states, want, stiff=stiff, grad=grad)
    ref = states[-1]
    d_tr = float((m.state["virial"].diagonal(dim1=1, dim2=2).sum(1).cpu() - ref.vir.diagonal(dim1=1, dim2=2).sum(1))
                 .abs().max())
    d_x = float((m.state["pos"] - ref.pos).abs().max())
    d_ve = float((m.state["v_eps"].cpu() - torch.tensor(ref.veps, dtype=torch.float64)).abs().max())
    ratios = {k: _close(m.state[k], torch.tensor(getattr(ref, a), dtype=torch.float64), b[k], f"{kind} {k}")
              for k, a in (("v_eps", "veps"), ("eps", "eps"))}
    worst = max(worst, _check_state(m, ref, b, kind), _check_log(log, want, b, kind))
    print(f"NPT-RATIO {kind}: largest error / bound {worst:.3g}; v_eps {ratios['v_eps']:.3g}, eps {ratios['eps']:.3g}; "
          f"|d v_eps| {d_ve:.3g}, |d tr vir| {d_tr:.3g}, |dx| {d_x:.3g}, G_x {grad:.3g}, K_b {stiff:.3g}, "
          f"G_x |dx| {grad * d_x:.3g}")
    assert m.host_reads == 3 + m.recaptures
    assert abs(float(m.state["eps"].abs().max())) > 0 and int(m.state["error"].sum()) == 0
    # the cell is C0 e^eps to an ulp, the shape untouched
    c0 = ex["cell"].reshape(-1, 3, 3).double()
    want_cell = c0 * torch.exp(m.state["eps"]).view(-1, 1, 1)
    assert float((m.state["cell"] - want_cell).abs().max()) <= 2.0 ** -52 * float(want_cell.abs().max())


@pytest.mark.timeout(900)
def test_float32_model_matches_the_host_loop():
    """The water box with a float32 model, 20 steps: against the host loop of the eager float32 model, to ``_bounds``
    with the float32 agreement F_AGREE of tests/test_md_run_gpu.py."""
    system = _npt_system("water", torch.float32)
    ex, model = system[:2]
    m, st0, prm = _start(system)
    n = 20
    log = m.run(n, block=8)
    states, want = _host_loop(model, ex, st0, prm, n, m.dt)
    b = _bounds(n, m.dt, prm, st0, states, want, agree=F_AGREE)
    worst = max(_close(m.state["pos"], states[-1].pos, b["pos"], "f32 pos"),
                _close(m.state["eps"], torch.tensor(states[-1].eps, dtype=torch.float64), b["eps"], "f32 eps"),
                _check_log(log, want, b, "f32"))
    print(f"NPT-RATIO float32: largest error / bound {worst:.3g}")


@pytest.mark.timeout(900)
def test_each_frame_equals_the_frame_run_alone():
    """The batch of five periodic frames (per-frame T, P, tau_T, tau_P) for 20 steps against each frame run on its
    own with its own bath, to ``_bounds`` of 20 steps."""
    ex, model, masses, bath = _npt_system("mixed_batch")
    m, st0, prm = _start((ex, model, masses, bath))
    log = m.run(20, block=10)
    ptr = prm.ptr
    for f in range(m.num_frames):
        a, b_ = ptr[f], ptr[f + 1]
        one = {"pos": ex["pos"][a:b_], "atom_types": ex["atom_types"][a:b_], "cell": ex["cell"][f:f + 1],
               "batch": torch.zeros(b_ - a, dtype=torch.int64, device="cuda"),
               "num_atoms": torch.tensor([b_ - a], device="cuda"), "pbc": ex["pbc"][f:f + 1]}
        fb = {k: [v[f]] for k, v in bath.items()}
        g = GraphedNPT(model, one, masses, DT_FS, fb["temperature"], fb["pressure"], tdamp_fs=fb["tdamp_fs"],
                       pdamp_fs=fb["pdamp_fs"], velocities=st0.vel[a:b_].cpu())
        lg = g.run(20, block=10)
        sub = no.Params([b_ - a], ex["cell"][f:f + 1].cpu(), fb["temperature"], fb["pressure"],
                        torch.tensor(fb["tdamp_fs"]) * mo.FS, torch.tensor(fb["pdamp_fs"]) * mo.FS, 3, 3)
        want = torch.stack([lg[k] for k in LOG_FIELDS], 2)
        ref_states = [no.State(g.state["pos"], g.state["vel"], g.state["forces"], g._mass, g.state["virial"].cpu(),
                               sub)]
        bd = _bounds(20, m.dt, sub, ref_states[0], ref_states, want)
        _close(m.state["pos"][a:b_], g.state["pos"], bd["pos"], f"frame {f} pos")
        _close(m.state["eps"][f], g.state["eps"], bd["eps"], f"frame {f} eps")
        for j, name in enumerate(LOG_FIELDS):
            _close(log[name][:, f], want[:, 0, j], bd[name], f"frame {f} {name}")


@pytest.mark.timeout(900)
def test_blocks_log_ring_and_split_runs_give_one_trajectory():
    """120 steps of the water box in blocks of 1, 7, 20 (the block of steps 100-119 wraps the 100-row log) and 150
    (longer than the log: a new log and a re-capture), and 70 + 50 steps over two calls; every run against the
    blocks-of-7 run to ``_bounds`` of 120 steps.  ``run(0)`` reads nothing, ``host_reads`` is the number of blocks,
    ``on_block`` sees the returned rows."""
    system = _npt_system("water")
    n = 120
    runs = {}
    for block in (7, 1, 20, 150):
        m, st0, prm = _start(system)
        seen = []
        log = m.run(n, block=block, on_block=seen.append)
        assert m.host_reads == math.ceil(n / block) + m.recaptures and int(m.state["step"]) == n
        for k in LOG_FIELDS:
            assert torch.equal(torch.cat([b[k] for b in seen]), log[k]) and log[k].shape == (n, 1)
        runs[block] = (m, log)
    m, _st, _p = _start(system)
    none = m.run(0)
    assert all(v.shape == (0, 1) for v in none.values()) and m.host_reads == 0
    first, second = m.run(70, block=30), m.run(50, block=40)
    runs["split"] = (m, {k: torch.cat([first[k], second[k]]) for k in LOG_FIELDS})
    ma, la = runs[7]
    want = torch.stack([la[k] for k in LOG_FIELDS], 2)
    ref = no.State(ma.state["pos"], ma.state["vel"], ma.state["forces"], ma._mass, ma.state["virial"].cpu(), prm)
    ref.eps, ref.veps = ma.state["eps"].tolist(), ma.state["v_eps"].tolist()
    b = _bounds(n, ma.dt, prm, st0, [ref], want)
    for key in (1, 20, 150, "split"):
        mb, lb = runs[key]
        _check_log(lb, want, b, f"block {key}")
        _close(mb.state["pos"], ma.state["pos"], b["pos"], f"block {key} pos")
        _close(mb.state["eps"], ma.state["eps"], b["eps"], f"block {key} eps")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("how", ["half_capacity", "compressing"])
def test_rollback_matches_a_large_capacity_run(how):
    """30 steps in blocks of 10 from capacity E0 // 2 (the first block overflows), or from capacity E0 under 10 GPa
    with tau_P = 50 fs (the box shrinks, so the list outgrows E0 during the run): recaptures >= 1, every block's rows
    reach the log once, and the run agrees with a run of capacity 4 E0 to ``_bounds`` of 30 steps."""
    system = _npt_system("water")
    ex = system[0]
    E0 = ops.neighbor_list(ex["pos"], ex["cell"], ex["pbc"], R_MAX, batch=ex["batch"])["edge_index"].shape[1]
    over = {} if how == "half_capacity" else dict(pressure=10 * GPA, pdamp_fs=50.0)
    small, st0, prm = _start(system, capacity=E0 // 2 if how == "half_capacity" else E0, **over)
    seen = []
    log_s = small.run(30, block=10, on_block=lambda b: seen.append(b["e_pot"].shape[0]))
    big, _s, _p = _start(system, capacity=4 * E0, **over)
    log_b = big.run(30, block=10)
    assert small.recaptures >= 1 and seen == [10, 10, 10]
    assert big.recaptures == 0 or how == "compressing"
    assert small.host_reads == 3 + small.recaptures
    if how == "compressing":
        assert float(log_s["volume"][-1, 0]) < float(log_s["volume"][0, 0])
    want = torch.stack([log_b[k] for k in LOG_FIELDS], 2)
    ref = no.State(big.state["pos"], big.state["vel"], big.state["forces"], big._mass, big.state["virial"].cpu(), prm)
    ref.veps = big.state["v_eps"].tolist()
    b = _bounds(30, big.dt, prm, st0, [ref], want)
    _check_log(log_s, want, b, f"rollback {how}")
    _close(small.state["pos"], big.state["pos"], b["pos"], f"rollback {how} pos")
    _close(small.state["eps"], big.state["eps"], b["eps"], f"rollback {how} eps")


# ------------------------------------------------------------------------------------------------------------------
# NPH: energy drift and time reversal
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_nph_drift_scales_as_dt_squared_and_retraces_its_path():
    """NPH (no chains) on the float64 water box: the largest |H(t) - H(0)| over 50 fs falls by 4 +- 1 from dt = 0.5 fs
    to 0.25 fs; then 50 steps, every velocity negated, 50 more: positions and eps return to the start to ``_bounds``
    of 100 steps."""
    system = _npt_system("water")
    drift = {}
    for dt in (0.5, 0.25):
        ex, model, masses, bath = system
        m = GraphedNPT(model, ex, masses, dt, bath["temperature"], 2 * GPA, tdamp_fs=50.0, pdamp_fs=50.0, tchain=0,
                       pchain=0, seed=3)
        m0 = {k: v.clone() for k, v in m.state.items()}
        log = m.run(int(round(50 / dt)), block=50)
        e0 = _eager(model, ex, m0["pos"], m0["cell"])[0]
        h0 = float(e0[0]) + 0.5 * float(m0["K2"][0]) + 2 * GPA * float(m._prm[0, 4])  # v_eps = 0 at the start
        drift[dt] = float((log["conserved"][:, 0] - h0).abs().max())
        assert float(log["volume"].max() - log["volume"].min()) > 0
    assert 3.0 <= drift[0.5] / drift[0.25] <= 5.0, drift
    m, st0, prm = _start(system, tchain=0, pchain=0, pressure=2 * GPA, pdamp_fs=50.0)
    x0 = m.state["pos"].clone()
    log = m.run(50, block=25)
    assert float((m.state["pos"] - x0).abs().max()) > 1e-3 and float(m.state["eps"].abs().max()) > 0
    for k in ("vel", "v_eps"):
        m.state[k].neg_()
    m.run(50, block=25)
    want = torch.stack([log[k] for k in LOG_FIELDS], 2)
    ref = no.State(m.state["pos"], m.state["vel"], m.state["forces"], m._mass, m.state["virial"].cpu(), prm)
    ref.veps = m.state["v_eps"].tolist()
    b = _bounds(100, m.dt, prm, st0, [ref], want)
    _close(m.state["pos"], x0, b["pos"], "reversal pos")
    _close(m.state["eps"], torch.zeros(1), b["eps"], "reversal eps")


# ------------------------------------------------------------------------------------------------------------------
# the error flag
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_non_finite_barostat_discards_the_block_and_names_the_frame():
    """A NaN v_eps put into frame 2 of the batch between blocks: nqb_npt_pre finds a non-finite update for that frame
    before anything moves, so it keeps the frame's positions and cell (the neighbour list only ever sees the unchanged,
    finite ones) and sets its flag; the block raises naming frame 2, and every state buffer is the block's starting
    state again.  With v_eps repaired the run continues."""
    m, _st, _p = _start(_npt_system("mixed_batch"))
    m.run(5, block=5)
    m.state["v_eps"][2] = float("nan")
    before = {k: v.clone() for k, v in m.state.items()}
    reads = m.host_reads
    with pytest.raises(RuntimeError, match=r"frame\(s\) \[2\]"):
        m.run(5, block=5)
    for k, v in m.state.items():
        assert torch.equal(v.view(torch.int8) if v.dtype != torch.float64 else v.view(torch.int64),
                           before[k].view(torch.int8) if v.dtype != torch.float64 else before[k].view(torch.int64)), k
    assert bool(torch.isfinite(m.state["pos"]).all()) and bool(torch.isfinite(m.state["cell"]).all())
    assert m.host_reads == reads + 1 and int(m.plan.cell_error.sum()) == 0
    m.state["v_eps"][2] = 0.0
    log = m.run(3, block=3)
    assert bool(torch.isfinite(log["conserved"]).all()) and int(m.state["step"]) == 8
