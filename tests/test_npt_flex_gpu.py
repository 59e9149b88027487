"""``GraphedNPT(barostat="flexible")`` and the nqb_nptf kernels on the GPU: every kernel against one step of the float64
oracle (tests/npt_flex_oracle.py) with its write contract, the frozen paths on guarded buffers, float64 trajectories
against a host loop of the oracle around ``ops.neighbor_list`` and the eager model with stress, a float32 model,
frame independence, blocks and the log ring, rollback, NPH energy drift and time reversal, the isotropic reduction
against ``barostat="isotropic"`` and the error flag.

The trajectory bound is tests/test_npt_gpu.py's ``_bounds`` with v_eps replaced by the largest entry of v_g, W by W_g
and its two measured terms generalised from tr(virial) to every virial component: G_x, the largest sum over positions
of |d virial_ij / d x| (``_virial_gradient9``), and K_b, the largest row sum of |d virial_ij / d strain_kl| over the 6
symmetric strain directions (``_stiffness6``).  Nothing in it is fitted."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import md_oracle as mo
import npt_flex_oracle as fo
from kernel_contracts import guarded
from nequip_b200 import _capi, ops
from nequip_b200.npt import GPA, LOG_FIELDS, GraphedNPT
from test_batched_md_step_gpu import _model as _model_any
from test_md_run_gpu import F_AGREE, R_MAX
from test_npt_gpu import DT_FS, F64_AGREE, LI3PO4_MASSES, _bounds, _close, _eager, _npt_system

pytestmark = pytest.mark.gpu

FIELDS = LOG_FIELDS + ("cell", "pressure_tensor")


@pytest.fixture(autouse=True)
def _deterministic():
    prev = ops.deterministic()
    ops.set_deterministic(True)
    yield
    ops.set_deterministic(prev)


def _sym(rng, F, scale):
    w = rng.standard_normal((F, 3, 3))
    return (w + w.transpose(0, 2, 1)) * scale


# ------------------------------------------------------------------------------------------------------------------
# kernels against one oracle step
# ------------------------------------------------------------------------------------------------------------------
def _kernel_cases():
    cases = []
    for name, counts in (("cta_edges", [255, 256, 257]), ("above_64_ctas", [16385, 3])):
        driver = min(64, -(-max(counts) // 256))
        for nblk in sorted({1, 2, driver}):
            for M, Mp in ((0, 0), (1, 3), (3, 1), (3, 3)):
                cases.append(pytest.param(counts, nblk, M, Mp, "general", id=f"{name}-nblk{nblk}-t{M}p{Mp}-general"))
            for vg in ("diagonal", "degenerate"):
                cases.append(pytest.param(counts, nblk, 3, 3, vg, id=f"{name}-nblk{nblk}-t3p3-{vg}"))
    return cases


def _vg(kind, rng, F):
    if kind == "general":
        return _sym(rng, F, 0.01)
    if kind == "diagonal":
        return np.stack([np.diag(0.02 * rng.standard_normal(3)) for _ in range(F)])
    out = []
    for _ in range(F):  # a doubly degenerate v_g in a random frame
        q, _r = np.linalg.qr(rng.standard_normal((3, 3)))
        out.append(q @ np.diag([0.01, 0.01, -0.02]) @ q.T)
    return np.stack(out)


def _kernel_state(counts, M, Mp, vg, seed):
    rng = np.random.default_rng(seed)
    F, N = len(counts), sum(counts)
    C0 = torch.tensor(np.stack([np.diag([20.0, 21.0, 22.0]) + rng.standard_normal((3, 3)) for _ in counts]))
    prm = fo.Params(counts, C0, [300.0 + 50 * f for f in range(F)], [0.01 * (f - 1) for f in range(F)],
                    [40.0 * mo.FS] * F, [300.0 * mo.FS + f for f in range(F)], M, Mp, 2, 2)
    t = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
    mass = t(rng.uniform(1.0, 30.0, N))
    st = fo.State(t(rng.standard_normal((N, 3)) * 10), t(rng.standard_normal((N, 3)) * 0.05),
                  t(rng.standard_normal((N, 3))), mass, t(_sym(rng, F, 5.0)), prm)
    g = _vg(vg, rng, F)
    for f in range(F):
        st.g[f] = g[f].reshape(-1).tolist()
        st.kt[f] = [x * (1.0 + 1e-3 * f) for x in st.kt[f]]  # the tracked Kt need not be the recomputed one
        for xs in (st.xi[f], st.vxi[f], st.eta[f], st.veta[f]):
            xs[:] = (0.1 * rng.standard_normal(len(xs))).tolist()
    return rng, prm, st, mass


def _buffers(st, prm, F, N, nblk, err=None):
    cu = dict(device="cuda")
    b = {}
    b["pos"] = guarded(N, 3, torch.float64, body=st.pos, **cu)
    b["vel"] = guarded(N, 3, torch.float64, body=st.vel, **cu)
    b["frc"] = guarded(N, 3, torch.float64, body=st.forces, **cu)
    b["st"] = guarded(F, fo.STATE, torch.float64, body=st.rows(), **cu)
    b["vir"] = guarded(F, 9, torch.float64, body=st.vir.reshape(F, 9), **cu)
    b["cell"] = guarded(F, 9, torch.float64, body=st.cell.reshape(F, 9), **cu)
    b["coef"] = guarded(F, 39, torch.float64, **cu)
    e0 = torch.zeros(F, 1, dtype=torch.int32) if err is None else torch.tensor(err, dtype=torch.int32).view(F, 1)
    b["err"] = guarded(F, 1, torch.int32, body=e0, **cu)
    b["work"] = guarded(F, fo.STATE, torch.float64, **cu)
    b["part"] = guarded(F * nblk, 6, torch.float64, **cu)
    b["log"] = guarded(2 * F, fo.LOG, torch.float64, **cu)
    return {k: v[0] for k, v in b.items()}, [v[1] for v in b.values()]


@pytest.mark.parametrize("counts,nblk,M,Mp,vg", _kernel_cases())
def test_kernels_match_one_oracle_step_and_write_only_their_outputs(counts, nblk, M, Mp, vg):
    """pre, move, kick (new forces), post (new virial), scale and log against one oracle step, tloop = ploop = 2, on a
    state with every barostat and chain variable non-zero and a general, diagonal or doubly degenerate v_g; each
    output within 1e-14 of its magnitude, and no kernel writes outside its buffers."""
    F, N = len(counts), sum(counts)
    rng, prm, st, mass = _kernel_state(counts, M, Mp, vg, sum(counts) + nblk + 10 * M + Mp)
    t = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
    f1 = t(rng.standard_normal((N, 3)))
    vir1 = t(_sym(rng, F, 5.0))
    e1 = t(rng.standard_normal(F))
    d, checks = _buffers(st, prm, F, N, nblk)
    dprm, aptr = prm.table().cuda(), torch.tensor(prm.ptr).cuda()
    dmass, df1, dvir1, de1 = mass.cuda(), f1.cuda(), vir1.reshape(F, 9).cuda(), e1.cuda()
    cu = dict(device="cuda")
    zero64, zero32 = torch.zeros(1, dtype=torch.int64, **cu), torch.zeros(1, dtype=torch.int32, **cu)
    one32 = torch.ones(1, dtype=torch.int32, **cu)
    step = torch.zeros(1, dtype=torch.int64, **cu)
    flags = torch.tensor([0, 0, -1, 0], dtype=torch.int64, **cu)
    P, L, s = ops._ptr, _capi.lib(), ops._stream()
    dt = DT_FS * mo.FS
    _capi.check(L.nqb_nptf_pre(F, M, Mp, 2, 2, dt, P(dprm), P(d["vir"]), P(d["st"]), P(d["cell"]), P(d["coef"]),
                               P(d["err"]), P(d["work"]), s))
    _capi.check(L.nqb_nptf_move(F, nblk, P(aptr), P(dmass), P(d["frc"]), P(d["coef"]), P(d["pos"]), P(d["vel"]), s))
    _capi.check(L.nqb_nptf_kick(F, nblk, P(aptr), P(dmass), P(df1), P(d["coef"]), P(d["vel"]), P(d["frc"]),
                                P(d["part"]), s))
    _capi.check(L.nqb_nptf_post(F, nblk, M, Mp, 2, 2, dt, P(dprm), P(d["part"]), P(dvir1), P(d["cell"]), P(d["st"]),
                                P(d["vir"]), P(d["coef"]), P(d["err"]), P(d["work"]), s))
    _capi.check(L.nqb_nptf_scale(F, nblk, P(aptr), P(d["coef"]), P(d["vel"]), s))
    _capi.check(L.nqb_nptf_log(F, M, Mp, P(de1), P(dprm), P(d["st"]), P(d["vir"]), P(d["cell"]), P(zero64),
                               P(zero32), P(one32), 2, P(step), P(d["log"]), P(flags), s))
    torch.cuda.synchronize()
    for c in checks:
        c()
    g0 = [list(g) for g in st.g]
    fo.step(st, prm, dt, lambda pos, cell: (e1, f1, vir1))

    def close(got, ref, what):
        ref = ref.double().cpu()
        got = got.cpu().reshape(ref.shape)
        assert not torch.isnan(got).any(), what
        err = (got - ref).abs()
        tol = 1e-14 * max(1.0, float(ref.abs().max()))
        assert float(err.max()) <= tol, (what, float(err.max()), tol, torch.nonzero(err > tol)[:5].tolist())

    close(d["pos"], st.pos, "pos")
    close(d["vel"], st.vel, "vel")
    close(d["frc"], f1, "forces")
    close(d["st"], st.rows(), "state")
    close(d["vir"], st.vir.reshape(F, 9), "virial")
    close(d["cell"], st.cell.reshape(F, 9), "cell")
    close(d["log"].view(2, F, fo.LOG)[0], fo.log_row(st, prm), "log")
    assert int(d["err"].sum()) == 0 and int(step) == 1 and flags.cpu().tolist() == [0, 0, -1, 0]
    sv = d["st"].cpu()[:, :9].reshape(F, 3, 3)
    assert torch.equal(sv, sv.transpose(1, 2))  # v_g stays exactly symmetric
    assert any(max(abs(x) for x in g) > 0 for g in g0)


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int64) if t.dtype == torch.float64 else t


@pytest.mark.parametrize("nblk", [1, 2])
def test_frozen_frames_keep_their_state_and_atoms(nblk):
    """The frozen paths, on guarded buffers: frame 0 enters with err set, frame 2 with a NaN in v_g (pre finds a
    non-finite update), frame 1 gets a NaN virial from the model (post finds it), frame 3 is an ordinary frame.  pre
    gives frames 0 and 2 the coefficients {1, 0, 1, I, 0, I, 0} and leaves their state rows and cells bitwise as they
    were; move, kick and scale leave their atoms untouched and kick writes 0 into their partial sums; post flags frame
    1, sets its final scale to 1 and leaves its state row (as pre left it) and its virial unchanged; frame 3 steps."""
    counts = [5, 300, 7, 9]
    F, N = len(counts), sum(counts)
    rng, prm, st, mass = _kernel_state(counts, 3, 3, "general", nblk)
    st.g[2][5] = float("nan")
    rows0 = st.rows()
    d, checks = _buffers(st, prm, F, N, nblk, err=[1, 0, 0, 0])
    dprm, aptr, dmass = prm.table().cuda(), torch.tensor(prm.ptr).cuda(), mass.cuda()
    f1 = torch.randn(N, 3, generator=torch.Generator().manual_seed(nblk), dtype=torch.float64).cuda()
    vir1 = torch.randn(F, 9, generator=torch.Generator().manual_seed(9), dtype=torch.float64).cuda()
    vir1[1, 4] = float("nan")
    P, L, s_ = ops._ptr, _capi.lib(), ops._stream()
    dt = DT_FS * mo.FS
    ptr = prm.ptr
    at = lambda x, f: x[ptr[f]:ptr[f + 1]]  # noqa: E731
    pos0, vel0, frc0, cell0, vir0 = (d[k].clone() for k in ("pos", "vel", "frc", "cell", "vir"))
    _capi.check(L.nqb_nptf_pre(F, 3, 3, 2, 2, dt, P(dprm), P(d["vir"]), P(d["st"]), P(d["cell"]), P(d["coef"]),
                               P(d["err"]), P(d["work"]), s_))
    torch.cuda.synchronize()
    eye, zero = torch.eye(3, dtype=torch.float64).reshape(9), torch.zeros(9, dtype=torch.float64)
    frozen = torch.cat([torch.tensor([1.0, 0.0, 1.0], dtype=torch.float64), eye, zero, eye, zero])
    for f in (0, 2):
        assert torch.equal(d["coef"][f].cpu(), frozen), f
        assert torch.equal(_bits(d["st"][f]), _bits(rows0[f])) and torch.equal(d["cell"][f], cell0[f]), f
    assert d["err"].view(-1).cpu().tolist() == [1, 0, 1, 0]
    assert float(d["coef"][1, 1]) == 1.0 and float(d["coef"][3, 1]) == 1.0
    st_pre = d["st"].clone()
    _capi.check(L.nqb_nptf_move(F, nblk, P(aptr), P(dmass), P(d["frc"]), P(d["coef"]), P(d["pos"]), P(d["vel"]), s_))
    _capi.check(L.nqb_nptf_kick(F, nblk, P(aptr), P(dmass), P(f1), P(d["coef"]), P(d["vel"]), P(d["frc"]),
                                P(d["part"]), s_))
    torch.cuda.synchronize()
    vel_kick = d["vel"].clone()
    _capi.check(L.nqb_nptf_post(F, nblk, 3, 3, 2, 2, dt, P(dprm), P(d["part"]), P(vir1), P(d["cell"]), P(d["st"]),
                                P(d["vir"]), P(d["coef"]), P(d["err"]), P(d["work"]), s_))
    _capi.check(L.nqb_nptf_scale(F, nblk, P(aptr), P(d["coef"]), P(d["vel"]), s_))
    torch.cuda.synchronize()
    for c in checks:
        c()
    assert d["err"].view(-1).cpu().tolist() == [1, 1, 1, 0]
    part = d["part"].view(F, nblk * 6).cpu()
    for f in (0, 2):
        for x, x0 in ((d["pos"], pos0), (d["vel"], vel0), (d["frc"], frc0)):
            assert torch.equal(at(x, f), at(x0, f)), f
        assert torch.equal(part[f], torch.zeros(nblk * 6, dtype=torch.float64))
        assert torch.equal(_bits(d["st"][f]), _bits(rows0[f])) and torch.equal(d["vir"][f], vir0[f])
        assert torch.equal(d["cell"][f], cell0[f])
    assert float(d["coef"][1, 2]) == 1.0
    assert torch.equal(d["st"][1], st_pre[1]) and torch.equal(d["vir"][1], vir0[1])
    assert torch.equal(at(d["vel"], 1), at(vel_kick, 1)) and torch.equal(at(d["frc"], 1), at(f1, 1))
    assert not torch.equal(at(d["pos"], 1), at(pos0, 1)) and bool(torch.isfinite(d["pos"]).all())
    assert torch.equal(d["vir"][3], vir1[3]) and not torch.equal(d["st"][3], st_pre[3])
    assert bool(torch.isfinite(d["st"][3]).all()) and not torch.equal(d["cell"][3], cell0[3])


# ------------------------------------------------------------------------------------------------------------------
# the host loop and the bound
# ------------------------------------------------------------------------------------------------------------------
def _start(system, tchain=3, pchain=3, capacity=None, seed=7, velocities=None, **over):
    ex, model, masses, bath = system
    bath = dict(bath, **over)
    m = GraphedNPT(model, ex, masses, DT_FS, bath["temperature"], bath["pressure"], tdamp_fs=bath["tdamp_fs"],
                   pdamp_fs=bath["pdamp_fs"], tchain=tchain, pchain=pchain, capacity=capacity, seed=seed,
                   velocities=velocities, barostat="flexible")
    counts = ex["num_atoms"].cpu().tolist()
    prm = fo.Params(counts, ex["cell"].cpu(), bath["temperature"], bath["pressure"],
                    torch.tensor(bath["tdamp_fs"], dtype=torch.float64) * mo.FS,
                    torch.tensor(bath["pdamp_fs"], dtype=torch.float64) * mo.FS, tchain, pchain)
    e0, f0, v0 = _eager(model, ex, ex["pos"].double(), ex["cell"])
    st = fo.State(ex["pos"].double(), m.state["vel"].clone(), f0, m._mass, v0, prm)
    st.kt = m.state["kinetic"].cpu().reshape(-1, 9).tolist()  # the driver's correctly rounded start
    st.e_pot = e0.tolist()
    return m, st, prm


def _host_loop(model, ex, st, prm, n, dt):
    st = st.clone()
    states, rows = [], []
    for _ in range(n):
        fo.step(st, prm, dt, lambda p, c: _eager(model, ex, p, c))
        states.append(st.clone())
        rows.append(fo.log_row(st, prm))
    return states, torch.stack(rows)


_STRAINS = [(0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1)]


def _stiffness6(model, ex, st0, h=1e-5):
    """K_b = max over frames and virial components of the row sum over the 6 symmetric strain directions of
    |d virial_ij / d strain_kl| at the initial state (central differences of the eager model)."""
    F = st0.cell.shape[0]
    dv = torch.zeros(F, 9, 6, dtype=torch.float64)
    for c, (k, l) in enumerate(_STRAINS):
        E = torch.zeros(3, 3, dtype=torch.float64)
        E[k, l] = E[l, k] = 1.0
        vs = []
        for sg in (h, -h):
            Fd = (torch.eye(3, dtype=torch.float64) + sg * E).cuda()
            frame = ex["batch"]
            pos = torch.einsum("nj,nij->ni", st0.pos.cuda(), Fd.expand(F, 3, 3)[frame])
            vs.append(_eager(model, ex, pos, st0.cell.cuda() @ Fd.T)[2].reshape(F, 9))
        dv[:, :, c] = (vs[0] - vs[1]) / (2 * h)
    return float(dv.abs().sum(2).max())


def _virial_gradient9(model, ex, st0, h=1e-5, chunk_atoms=30000):
    """G_x = max over frames and virial components of sum_i |d virial_ij / d x_i| at the initial state, by central
    differences of the eager model (as test_npt_gpu._virial_gradient does for the trace)."""
    counts = ex["num_atoms"].cpu().tolist()
    ptr = [0] + torch.tensor(counts).cumsum(0).tolist()
    F, N = len(counts), st0.pos.shape[0]
    C = 3 * max(counts)
    jobs = [(c, sg) for c in range(C) for sg in (1.0, -1.0)]
    K = max(1, chunk_atoms // N)
    vir = torch.zeros(len(jobs), F, 9, dtype=torch.float64)
    pos0 = st0.pos.cuda()
    for a in range(0, len(jobs), K):
        part = jobs[a:a + K]
        k = len(part)
        pos = pos0.repeat(k, 1)
        for j, (c, sg) in enumerate(part):
            for f in range(F):
                if c < 3 * counts[f]:
                    pos[j * N + ptr[f] + c // 3, c % 3] += sg * h
        big = {"atom_types": ex["atom_types"].repeat(k), "num_atoms": ex["num_atoms"].repeat(k),
               "pbc": ex["pbc"].reshape(F, 3).repeat(k, 1),
               "batch": ex["batch"].repeat(k) + F * torch.arange(k, device="cuda").repeat_interleave(N)}
        vir[a:a + k] = _eager(model, big, pos, st0.cell.cuda().repeat(k, 1, 1))[2].reshape(k, F, 9)
    g = (vir[0::2] - vir[1::2]) / (2 * h)  # [C, F, 9]
    mask = (torch.arange(C).unsqueeze(1) < 3 * torch.tensor(counts).unsqueeze(0)).unsqueeze(2)
    return float((g.abs() * mask).sum(0).max())


def _shim(st):
    """A flexible oracle state seen by test_npt_gpu._bounds: v_eps its largest |v_g| entry, K2 its tr Kt."""
    return SimpleNamespace(pos=st.pos, vel=st.vel, forces=st.forces, mass=st.mass, vir=st.vir,
                           veps=[max(abs(x) for x in g) for g in st.g], K2=[k[0] + k[4] + k[8] for k in st.kt],
                           vxi=st.vxi, veta=st.veta)


def _fbounds(n, dt, prm, st0, states, log, **kw):
    b = _bounds(n, dt, prm, _shim(st0), [_shim(s) for s in states], log[:, :, :6], **kw)
    cmax = float(log[:, :, 6:15].abs().max())
    b["v_g"] = b["v_eps"]
    b["cell"] = 3 * cmax * b["eps"] + 1e-13
    b["pressure_tensor"] = b["pressure"] * 3
    return b


def _check_state(m, ref, b, what):
    s = m.state
    F = m.num_frames
    r = [_close(s["pos"], ref.pos, b["pos"], f"{what} pos"), _close(s["vel"], ref.vel, b["vel"], f"{what} vel"),
         _close(s["v_g"], torch.tensor(ref.g, dtype=torch.float64), b["v_g"], f"{what} v_g"),
         _close(s["cell"], ref.cell, b["cell"], f"{what} cell")]
    for k, name in (("xi", "xi"), ("vxi", "v_xi"), ("eta", "eta"), ("veta", "v_eta")):
        want = torch.tensor(getattr(ref, k), dtype=torch.float64).reshape(F, -1)
        r.append(_close(s[name], want, b[name], f"{what} {name}"))
    return max(r)


def _check_log(log, want, b, what):
    r = [_close(log[name], want[:, :, j], b[name], f"{what} {name}") for j, name in enumerate(LOG_FIELDS)]
    n, F = want.shape[:2]
    r.append(_close(log["cell"], want[:, :, 6:15].reshape(n, F, 3, 3), b["cell"], f"{what} cell"))
    r.append(_close(log["pressure_tensor"], want[:, :, 15:].reshape(n, F, 3, 3), b["pressure_tensor"],
                    f"{what} pressure_tensor"))
    return max(r)


def _want(log):
    n, F = log["e_pot"].shape
    return torch.cat([torch.stack([log[k] for k in LOG_FIELDS], 2), log["cell"].reshape(n, F, 9),
                      log["pressure_tensor"].reshape(n, F, 9)], 2)


# ------------------------------------------------------------------------------------------------------------------
# trajectories against the host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["water", "li3po4_zbl_table", "left_handed", "mixed_batch"])
def test_float64_trajectory_matches_the_host_loop(kind):
    """40 steps of 0.5 fs in blocks of 16 with both chains against the host loop: the state at the end of the run
    (positions, velocities, v_g, the cell, the chains) and every log row (with the cell and the pressure tensor) to
    ``_fbounds``.  The off-diagonal cell entries must move: the shape changes, not only the scale."""
    system = _npt_system(kind)
    ex, model = system[:2]
    m, st0, prm = _start(system)
    n, block = 40, 16
    log = m.run(n, block=block)
    states, want = _host_loop(model, ex, st0, prm, n, m.dt)
    stiff, grad = _stiffness6(model, ex, st0), _virial_gradient9(model, ex, st0)
    b = _fbounds(n, m.dt, prm, st0, states, want, stiff=stiff, grad=grad)
    worst = max(_check_state(m, states[-1], b, kind), _check_log(log, want, b, kind))
    d_g = float((m.state["v_g"].cpu() - torch.tensor(states[-1].g, dtype=torch.float64).view(-1, 3, 3)).abs().max())
    print(f"NPTF-RATIO {kind}: largest error / bound {worst:.3g}; |d v_g| {d_g:.3g}, G_x {grad:.3g}, K_b {stiff:.3g}")
    assert m.host_reads == 3 + m.recaptures and int(m.state["error"].sum()) == 0
    cell, c0 = m.state["cell"].cpu(), ex["cell"].reshape(-1, 3, 3).double().cpu()
    off = ~torch.eye(3, dtype=torch.bool)
    assert float((cell - c0)[:, off].abs().max()) > 0  # the shape moved, not only the scale
    sv = m.state["v_g"].cpu()
    assert torch.equal(sv, sv.transpose(1, 2))


@pytest.mark.timeout(900)
def test_float32_model_matches_the_host_loop():
    """The water box with a float32 model, 20 steps, against the host loop of the eager float32 model to ``_fbounds``
    with the float32 agreement F_AGREE."""
    system = _npt_system("water", torch.float32)
    ex, model = system[:2]
    m, st0, prm = _start(system)
    n = 20
    log = m.run(n, block=8)
    states, want = _host_loop(model, ex, st0, prm, n, m.dt)
    b = _fbounds(n, m.dt, prm, st0, states, want, agree=F_AGREE)
    worst = max(_close(m.state["pos"], states[-1].pos, b["pos"], "f32 pos"),
                _close(m.state["cell"], states[-1].cell, b["cell"], "f32 cell"), _check_log(log, want, b, "f32"))
    print(f"NPTF-RATIO float32: largest error / bound {worst:.3g}")


@pytest.mark.timeout(900)
def test_each_frame_equals_the_frame_run_alone():
    """The batch of five periodic frames (per-frame T, P, tau_T, tau_P, one of one atom) for 20 steps against each
    frame run on its own, to ``_fbounds`` of 20 steps."""
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
                       pdamp_fs=fb["pdamp_fs"], velocities=st0.vel[a:b_].cpu(), barostat="flexible")
        lg = g.run(20, block=10)
        sub = fo.Params([b_ - a], ex["cell"][f:f + 1].cpu(), fb["temperature"], fb["pressure"],
                        torch.tensor(fb["tdamp_fs"]) * mo.FS, torch.tensor(fb["pdamp_fs"]) * mo.FS, 3, 3)
        want = _want(lg)
        ref = fo.State(g.state["pos"], g.state["vel"], g.state["forces"], g._mass, g.state["virial"].cpu(), sub,
                       cell=g.state["cell"].cpu())
        ref.g = g.state["v_g"].cpu().reshape(-1, 9).tolist()
        bd = _fbounds(20, m.dt, sub, ref, [ref], want)
        _close(m.state["pos"][a:b_], g.state["pos"], bd["pos"], f"frame {f} pos")
        _close(m.state["cell"][f], g.state["cell"][0], bd["cell"], f"frame {f} cell")
        _close(m.state["v_g"][f], g.state["v_g"][0], bd["v_g"], f"frame {f} v_g")
        for j, name in enumerate(LOG_FIELDS):
            _close(log[name][:, f], want[:, 0, j], bd[name], f"frame {f} {name}")


def _ref_from(m, prm):
    ref = fo.State(m.state["pos"], m.state["vel"], m.state["forces"], m._mass, m.state["virial"].cpu(), prm,
                   cell=m.state["cell"].cpu())
    ref.g = m.state["v_g"].cpu().reshape(-1, 9).tolist()
    return ref


@pytest.mark.timeout(900)
def test_blocks_log_ring_and_split_runs_give_one_trajectory():
    """120 steps of the water box in blocks of 1, 7, 20 and 150 (a new log and a re-capture) and 70 + 50 steps over
    two calls, each against the blocks-of-7 run to ``_fbounds`` of 120 steps; ``run(0)`` reads nothing and returns
    empty fields of the right shapes; ``on_block`` sees the returned rows."""
    system = _npt_system("water")
    n = 120
    runs = {}
    for block in (7, 1, 20, 150):
        m, st0, prm = _start(system)
        seen = []
        log = m.run(n, block=block, on_block=seen.append)
        assert m.host_reads == math.ceil(n / block) + m.recaptures and int(m.state["step"]) == n
        for k in FIELDS:
            assert torch.equal(torch.cat([b[k] for b in seen]), log[k])
        assert log["e_pot"].shape == (n, 1) and log["cell"].shape == (n, 1, 3, 3)
        runs[block] = (m, log)
    m, _st, _p = _start(system)
    none = m.run(0)
    assert set(none) == set(FIELDS) and m.host_reads == 0
    assert none["e_pot"].shape == (0, 1) and none["pressure_tensor"].shape == (0, 1, 3, 3)
    first, second = m.run(70, block=30), m.run(50, block=40)
    runs["split"] = (m, {k: torch.cat([first[k], second[k]]) for k in FIELDS})
    ma, la = runs[7]
    want = _want(la)
    b = _fbounds(n, ma.dt, prm, st0, [_ref_from(ma, prm)], want)
    for key in (1, 20, 150, "split"):
        mb, lb = runs[key]
        _check_log(lb, want, b, f"block {key}")
        _close(mb.state["pos"], ma.state["pos"], b["pos"], f"block {key} pos")
        _close(mb.state["cell"], ma.state["cell"], b["cell"], f"block {key} cell")


@pytest.mark.timeout(900)
@pytest.mark.parametrize("how", ["half_capacity", "compressing"])
def test_rollback_matches_a_large_capacity_run(how):
    """30 steps in blocks of 10 from capacity E0 // 2, or from E0 under 10 GPa with tau_P = 50 fs: recaptures >= 1,
    every block's rows reach the log once, and the run agrees with a run of capacity 4 E0 to ``_fbounds``."""
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
    assert small.host_reads == 3 + small.recaptures
    if how == "compressing":
        assert float(log_s["volume"][-1, 0]) < float(log_s["volume"][0, 0])
    want = _want(log_b)
    b = _fbounds(30, big.dt, prm, st0, [_ref_from(big, prm)], want)
    _check_log(log_s, want, b, f"rollback {how}")
    _close(small.state["pos"], big.state["pos"], b["pos"], f"rollback {how} pos")
    _close(small.state["cell"], big.state["cell"], b["cell"], f"rollback {how} cell")


# ------------------------------------------------------------------------------------------------------------------
# NPH, the isotropic reduction, the error flag
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_nph_drift_scales_as_dt_squared_and_retraces_its_path():
    """NPH on the float64 water box: the largest |H(t) - H(0)| over 50 fs falls by 4 +- 1 from dt = 0.5 fs to
    0.25 fs; then 50 steps, every velocity negated (v, v_g), 50 more: positions and cell return to the start to
    ``_fbounds`` of 100 steps."""
    system = _npt_system("water")
    drift = {}
    for dt in (0.5, 0.25):
        ex, model, masses, bath = system
        m = GraphedNPT(model, ex, masses, dt, bath["temperature"], 2 * GPA, tdamp_fs=50.0, pdamp_fs=50.0, tchain=0,
                       pchain=0, seed=3, barostat="flexible")
        m0 = {k: v.clone() for k, v in m.state.items()}
        log = m.run(int(round(50 / dt)), block=50)
        e0 = _eager(model, ex, m0["pos"], m0["cell"])[0]
        V0 = float(torch.linalg.det(m0["cell"][0]).abs())
        h0 = float(e0[0]) + 0.5 * float(m0["kinetic"][0].trace()) + 2 * GPA * V0  # v_g = 0 at the start
        drift[dt] = float((log["conserved"][:, 0] - h0).abs().max())
        off = ~torch.eye(3, dtype=torch.bool, device="cuda")
        assert float(m.state["cell"][0][off].abs().max()) > 0
    print(f"NPH drift {drift}")
    assert 3.0 <= drift[0.5] / drift[0.25] <= 5.0, drift
    m, st0, prm = _start(system, tchain=0, pchain=0, pressure=2 * GPA, pdamp_fs=50.0)
    x0, c0 = m.state["pos"].clone(), m.state["cell"].clone()
    log = m.run(50, block=25)
    assert float((m.state["pos"] - x0).abs().max()) > 1e-3 and float((m.state["cell"] - c0).abs().max()) > 0
    for k in ("vel", "v_g"):
        m.state[k].neg_()
    m.run(50, block=25)
    b = _fbounds(100, m.dt, prm, st0, [_ref_from(m, prm)], _want(log))
    _close(m.state["pos"], x0, b["pos"], "reversal pos")
    _close(m.state["cell"], c0, b["cell"], "reversal cell")


def _fcc_li(a=3.6, reps=3):
    basis = torch.tensor([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]], dtype=torch.float64)
    r = torch.arange(reps, dtype=torch.float64)
    cells = torch.cartesian_prod(r, r, r)
    pos = (cells[:, None, :] + basis[None]).reshape(-1, 3) * a
    N = pos.shape[0]
    return {"pos": pos.cuda(), "atom_types": torch.zeros(N, dtype=torch.int64, device="cuda"),
            "cell": (a * reps * torch.eye(3, dtype=torch.float64)).view(1, 3, 3).cuda(),
            "batch": torch.zeros(N, dtype=torch.int64, device="cuda"), "num_atoms": torch.tensor([N], device="cuda"),
            "pbc": torch.ones(1, 3, dtype=torch.bool)}


@pytest.mark.timeout(900)
def test_isotropic_start_follows_the_isotropic_barostat():
    """A perfect fcc lattice of one species at rest (forces 0, virial a multiple of I to round-off) under 1 GPa with
    pchain = 0: 60 steps of the flexible barostat follow ``barostat="isotropic"`` with the same arguments -- positions,
    cell, v_g against v_eps I, and every log field -- to 1e-9 relative, and the off-diagonal cell entries stay at
    round-off (1e-12 of the cell)."""
    ex = _fcc_li()
    model = _model_any(["Li", "P", "O"], torch.float64, 12.0)
    N = ex["pos"].shape[0]
    kw = dict(tdamp_fs=50.0, pdamp_fs=100.0, tchain=3, pchain=0, velocities=torch.zeros(N, 3, dtype=torch.float64))
    iso = GraphedNPT(model, ex, LI3PO4_MASSES, DT_FS, 300.0, GPA, **kw)
    flex = GraphedNPT(model, ex, LI3PO4_MASSES, DT_FS, 300.0, GPA, barostat="flexible", **kw)
    li, lf = iso.run(60, block=20), flex.run(60, block=20)
    cell, ci = flex.state["cell"].cpu(), iso.state["cell"].cpu()
    assert abs(float(iso.state["eps"][0])) > 1e-4
    scale = float(ci.abs().max())
    assert float((cell - ci).abs().max()) <= 1e-9 * scale
    off = ~torch.eye(3, dtype=torch.bool)
    assert float(cell[0][off].abs().max()) <= 1e-12 * scale
    ve = float(iso.state["v_eps"][0])
    g = flex.state["v_g"][0].cpu()
    assert float((g - ve * torch.eye(3, dtype=torch.float64)).abs().max()) <= 1e-9 * abs(ve)
    pos_scale = float(iso.state["pos"].abs().max())
    assert float((flex.state["pos"] - iso.state["pos"]).abs().max()) <= 1e-9 * pos_scale
    for name in LOG_FIELDS:
        a, b = lf[name], li[name]
        assert float((a - b).abs().max()) <= 1e-9 * max(float(b.abs().max()), 1e-300) + 1e-12, name


@pytest.mark.timeout(900)
def test_non_finite_cell_velocity_discards_the_block_and_names_the_frame():
    """A NaN put into v_g of frame 2 of the batch between blocks: nqb_nptf_pre keeps that frame's positions and cell
    and sets its flag; the block raises naming frame 2, and every state buffer is the block's starting state again.
    With v_g repaired the run continues."""
    m, _st, _p = _start(_npt_system("mixed_batch"))
    m.run(5, block=5)
    m.state["v_g"][2, 0, 1] = float("nan")
    before = {k: v.clone() for k, v in m.state.items()}
    reads = m.host_reads
    with pytest.raises(RuntimeError, match=r"frame\(s\) \[2\]"):
        m.run(5, block=5)
    for k, v in m.state.items():
        assert torch.equal(v.view(torch.int8) if v.dtype != torch.float64 else v.view(torch.int64),
                           before[k].view(torch.int8) if v.dtype != torch.float64 else before[k].view(torch.int64)), k
    assert bool(torch.isfinite(m.state["pos"]).all()) and bool(torch.isfinite(m.state["cell"]).all())
    assert m.host_reads == reads + 1 and int(m.plan.cell_error.sum()) == 0
    m.state["v_g"][2, 0, 1] = m.state["v_g"][2, 1, 0]
    log = m.run(3, block=3)
    assert bool(torch.isfinite(log["conserved"]).all()) and int(m.state["step"]) == 8
