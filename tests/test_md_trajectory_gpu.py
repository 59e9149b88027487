"""Float64 ``GraphedMD`` trajectories against a float64 host loop, and the paths of ``GraphedMD.run`` that only a
float64 comparison can pin down: the log ring's wrap-around, a block longer than the log, runs split over several
calls, rollback under the bath in a batch, time reversal and a frame of more than 64 CTAs x 256 atoms.

The host loop is ``md_oracle.nh_step`` (the reference's Nose-Hoover step restated in float64; NVE freezes the bath)
around ``ops.neighbor_list`` and the eager model.  Under ``ops.set_deterministic(True)`` a float64 model's graphed
forces agree with its eager forces to F64_AGREE max|F| (tests/test_md_step_gpu.py), and the null edges of a padded
list add exact zeros, so two float64 trajectories from one state differ only by what that agreement lets grow over n
steps.  ``_bounds`` derives the bound in the form of tests/test_md_run_gpu.py's float32 one; it is about five orders
of magnitude tighter.  Each docstring gives the largest error seen on an H100, as a fraction of its bound."""
import math

import pytest
import torch

import md_oracle as mo
from batched_oracle import concat_frames
from cell_frames import cell_frame
from nequip_b200 import data as D
from nequip_b200 import md, ops
from nequip_b200.nn.model import NequIPEnergyModel
from test_batched_md_step_gpu import LI3PO4_TABLE, _mixed_frames
from test_batched_md_step_gpu import _model as _model_f64
from test_md_run_gpu import MASSES, R_MAX, _case

pytestmark = pytest.mark.gpu

F64_AGREE = 1e-12  # graphed against eager float64 forces in deterministic mode, relative to max|F|
LI3PO4_MASSES = [6.94, 30.974, 15.999]  # Li, P, O
DT_FS = 0.5
KINDS = ["water", "slab", "molecule", "li3po4_zbl_table", "mixed_batch"]


@pytest.fixture(autouse=True)
def _deterministic():
    prev = ops.deterministic()
    ops.set_deterministic(True)
    yield
    ops.set_deterministic(prev)


# ------------------------------------------------------------------------------------------------------------------
# systems, the eager reference and the bound
# ------------------------------------------------------------------------------------------------------------------
def _system(kind):
    """(example on cuda, float64 model, per-type masses, temperature [F], nvt_q [F])."""
    if kind in ("water", "slab", "molecule"):
        ex, meta = _case(kind)
        ex["pos"] = ex["pos"].double()
        model = _model_f64(meta["type_names"], torch.float64, meta["avg_num_neighbors"])
        return ex, model, MASSES, [300.0], [5.0]
    if kind == "li3po4_zbl_table":
        d = cell_frame("li3po4", 3, "tilted", seed=10, outside=True)
        meta = d.pop("_meta")
        ex = {k: d[k].cuda() for k in ("pos", "atom_types", "cell")}
        model = _model_f64(meta["type_names"], torch.float64, meta["avg_num_neighbors"], LI3PO4_TABLE, zbl=True)
        return ex, model, LI3PO4_MASSES, [400.0], [10.0]
    # a periodic frame, a slab, a molecule, one atom and an empty frame
    frames, pbcs = _mixed_frames()
    keep = [0, 5, 6, 7, 8]
    b = concat_frames([frames[k] for k in keep], [pbcs[k] for k in keep])
    ann = b["edge_index"].shape[1] / b["pos"].shape[0]
    ex = {k: b[k].cuda() for k in ("pos", "atom_types", "cell", "batch", "num_atoms", "pbc")}
    model = _model_f64(["Li", "P", "O"], torch.float64, ann)
    return ex, model, LI3PO4_MASSES, [300.0, 450.0, 200.0, 600.0, 350.0], [5.0, 10.0, 3.0, 20.0, 8.0]


def _counts(ex):
    return ex["num_atoms"].cpu().tolist() if "batch" in ex else [ex["pos"].shape[0]]


def _velocities(mass, temperature, counts, seed):
    """Maxwell-Boltzmann velocities [N, 3] at each frame's temperature, on the host."""
    g = torch.Generator().manual_seed(seed)
    t = torch.repeat_interleave(torch.tensor(temperature, dtype=torch.float64), torch.tensor(counts))
    return torch.randn(mass.shape[0], 3, generator=g, dtype=torch.float64) * torch.sqrt(mo.KB * t / mass).unsqueeze(1)


def _eager(model, ex, pos):
    """(E_pot [F], forces [N, 3]) of ``ops.neighbor_list`` (pruned by the model's per-edge-type table) and the eager
    model at ``pos``."""
    kw = {} if "batch" not in ex else {"batch": ex["batch"]}
    if model.per_edge_type_cutoff is not None:
        kw.update(atom_types=ex["atom_types"], edge_type_cutoff=model.per_edge_type_cutoff)
    nl = ops.neighbor_list(pos, ex.get("cell"), ex.get("pbc", ex.get("cell") is not None), R_MAX, **kw)
    d = {k: v for k, v in ex.items() if k != "pbc"}
    d.update(pos=pos, edge_index=nl["edge_index"], edge_cell_shift=nl["edge_cell_shift"])
    out = model(d)
    return out["total_energy"].detach().double().view(-1), out["forces"].detach().double()


class _Ref:
    """The host loop's inputs for one system: masses, frames, the bath's g k_B T and Q, the initial velocities (after
    GraphedMD's clean-up) and forces."""

    def __init__(self, ex, masses, temperature, nvt_q, nh, vel, forces):
        self.mass = torch.tensor(masses, dtype=torch.float64, device="cuda")[ex["atom_types"].view(-1)]
        counts = _counts(ex)
        self.ptr = [0] + torch.tensor(counts).cumsum(0).tolist()
        F = len(counts)
        c = torch.tensor(counts, dtype=torch.float64)
        zero = torch.zeros(F, dtype=torch.float64)
        self.gkT = ((3 * c + 1) * mo.KB * torch.tensor(temperature, dtype=torch.float64).expand(F) if nh
                    else zero).cuda()
        self.Q = (torch.tensor(nvt_q, dtype=torch.float64).expand(F) if nh else zero).cuda()
        self.dof_kB = (3 * c * mo.KB).clamp_min(1e-300).cuda()
        self.nh, self.vel, self.forces = nh, vel, forces


def _host_loop(model, ex, ref, n, dt):
    """n steps of ``md_oracle.nh_step`` around the eager list and model from (ex["pos"], ref.vel, ref.forces) with
    zeta = eta = 0: the (pos, vel, zeta, eta) after every step and the log rows [n, F, 6] of LOG_FIELDS."""
    pos, vel, f = ex["pos"].double().clone(), ref.vel.clone(), ref.forces.clone()
    F = len(ref.ptr) - 1
    zeta = torch.zeros(F, dtype=torch.float64, device="cuda")
    eta = torch.zeros_like(zeta)
    states, rows = [], []
    for _ in range(n):
        pos, vel, f, zeta, eta, e = mo.nh_step(pos, vel, f, ref.mass, zeta, eta, lambda p: _eager(model, ex, p), dt,
                                               ref.gkT, ref.Q, ref.ptr, ref.nh)
        ke = mo.kinetic(vel, ref.mass, ref.ptr)
        h = mo.conserved(e, vel, ref.mass, zeta, eta, ref.gkT, ref.Q, ref.ptr)
        states.append((pos.clone(), vel.clone(), zeta.clone(), eta.clone()))
        rows.append(torch.stack([e, ke, 2 * ke / ref.dof_kB, zeta, eta, h], 1))
    return states, torch.stack(rows).cpu()


def _bounds(n, dt, ref, fmax, vmax, log):
    """Bounds after ``n`` steps on two float64 trajectories from one state whose forces agree to e = F64_AGREE max|F|
    at equal positions.  As for the float32 host-loop test: e moves the velocities by at most n dt e / m_min and the
    positions by at most sum_k k dt^2 e / m_min < n^2 dt^2 e / m_min, each with a factor 10 of slack for the growth of
    the difference through the forces.  The log fields follow to first order:
      E_pot: N max|F| dx;   E_kin: N m_max v_max dv;   T: 2 dE_kin / (3 N_f k_B) (smallest non-empty N_f);
      zeta: n dt dE_kin / Q_min (d zeta/dt = (2 K - g k_B T) / (2 Q));   eta: n dt dzeta;
      H: dE_pot + dE_kin + 2 Q_max max|zeta| dzeta + max(g k_B T) deta.
    Every energy also carries F64_AGREE of its largest magnitude (float64 sums in another order), and positions and
    velocities 1e-12 (the rounding of the update itself).  NVE has Q = 0: zeta and eta must match exactly.  ``log``
    [n, F, 6] is the reference's.  Returns (dx, dv, [6] bounds in the order of LOG_FIELDS)."""
    mass = ref.mass
    N, m_min, m_max = mass.numel(), float(mass.min()), float(mass.max())
    e = F64_AGREE * fmax
    dx = 10 * n * n * dt * dt * e / m_min + 1e-12
    dv = 10 * n * dt * e / m_min + 1e-12
    mag = log.abs().amax(dim=(0, 1)).tolist() if log.numel() else [0.0] * len(md.LOG_FIELDS)
    de = N * fmax * dx + F64_AGREE * mag[0]
    dk = N * m_max * vmax * dv + F64_AGREE * mag[1]
    dof = ref.dof_kB[ref.dof_kB > 1e-300]
    dT = 2 * dk / float(dof.min())
    Q = ref.Q[ref.Q > 0]
    dz = n * dt * dk / float(Q.min()) if Q.numel() else 0.0
    deta = n * dt * dz
    dh = de + dk + 2 * float(ref.Q.max()) * mag[3] * dz + float(ref.gkT.max()) * deta + F64_AGREE * mag[5]
    return dx, dv, [de, dk, dT, dz, deta, dh]


def _close(got, want, bound, what):
    """max |got - want| <= bound (a NaN fails)."""
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    err = float((got - want).abs().max()) if want.numel() else 0.0
    assert err <= bound, f"{what}: max |err| {err:.3g} > bound {bound:.3g}"


def _close_log(log, want, bounds, what=""):
    for j, name in enumerate(md.LOG_FIELDS):
        _close(log[name], want[:, :, j], bounds[j], f"{what}{name}")


def _start(system, thermostat, capacity=None, seed=7):
    """(example, model, GraphedMD, host-loop inputs) of a ``_system``; the initial velocities are drawn here and F(0)
    is the test's own eager call."""
    ex, model, masses, temp, q = system
    nh = thermostat is not None
    mass = torch.tensor(masses, dtype=torch.float64)[ex["atom_types"].view(-1).cpu()]
    vel0 = _velocities(mass, temp, _counts(ex), seed)
    f0 = _eager(model, ex, ex["pos"])[1]
    m = md.GraphedMD(model, ex, masses, DT_FS, thermostat, temperature=temp if nh else None,
                     nvt_q=q if nh else None, velocities=vel0, capacity=capacity)
    return ex, model, m, _Ref(ex, masses, temp, q, nh, m.state["vel"].clone(), f0)


def _snapshot(m):
    return {k: v.clone() for k, v in m.state.items()}


# ------------------------------------------------------------------------------------------------------------------
# trajectories against the host loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("thermostat", [None, "nose_hoover"], ids=["nve", "nh"])
def test_float64_trajectory_matches_the_host_loop(kind, thermostat):
    """40 steps of 0.5 fs in blocks of 16.  F(0) right after construction against the test's own eager call (to
    F64_AGREE max|F|); the state at the end of every block and every log row against the host loop, to ``_bounds``.
    Largest error / bound on an H100 over two runs (NVE, Nose-Hoover): water 6.9e-4, 6.9e-4; slab 7.3e-4, 6.9e-4;
    molecule 2.8e-4, 5.5e-4; Li3PO4 with ZBL and the table 3.3e-4, 1.6e-4; the mixed batch 1.1e-3, 6.2e-4.  The
    positions differ by at most 3.6e-15 Angstrom after 40 steps, and F(0) by at most 5.1e-4 of its bound."""
    ex, model, m, ref = _start(_system(kind), thermostat)
    fmax = float(ref.forces.abs().max())
    _close(m.state["forces"], ref.forces, F64_AGREE * fmax, "F(0)")
    n, block = 40, 16
    ends = []
    log = m.run(n, block=block, on_block=lambda b: ends.append(_snapshot(m)))
    states, want = _host_loop(model, ex, ref, n, m.dt)
    vmax = max(float(s[1].abs().max()) for s in states)
    for k, got in enumerate(ends):
        s = min(n, (k + 1) * block)
        dx, dv, _ = _bounds(s, m.dt, ref, fmax, vmax, want[:s])
        pos, vel, zeta, eta = states[s - 1]
        _close(got["pos"], pos, dx, f"pos after {s}")
        _close(got["vel"], vel, dv, f"vel after {s}")
        assert int(got["step"]) == s
    _, _, bl = _bounds(n, m.dt, ref, fmax, vmax, want)
    _close_log(log, want, bl)
    _close(m.state["zeta"], states[-1][2], bl[3], "state zeta")
    _close(m.state["eta"], states[-1][3], bl[4], "state eta")
    assert m.host_reads == 3 + m.recaptures


@pytest.mark.timeout(600)
def test_frame_above_64_ctas_matches_the_host_loop():
    """A periodic water box of 26^3 = 17 576 atoms, more than 64 CTAs x 256 atoms: the driver caps nblk at 64 and every
    CTA of the update kernels loops over its atoms.  A float64 model of 3 layers and 8 features, Nose-Hoover, 5 steps
    against the host loop.  Largest error / bound on an H100: 6.7e-3 (positions, 7.1e-15 of 1.1e-12 Angstrom)."""
    s = D.make_system("water", 26, r_max=R_MAX, seed=2)
    meta = s["_meta"]
    ex = {"pos": s["pos"].double().cuda(), "atom_types": s["atom_types"].view(-1).cuda(),
          "cell": s["cell"].double().view(3, 3).cuda()}
    N = ex["pos"].shape[0]
    assert N > 64 * 256
    model = NequIPEnergyModel(r_max=R_MAX, type_names=meta["type_names"], avg_num_neighbors=meta["avg_num_neighbors"],
                              model_dtype=torch.float64, parity=True, l_max=2, num_layers=3, num_features=8,
                              radial_mlp_depth=1, radial_mlp_width=16).cuda()
    for p in model.parameters():
        p.requires_grad_(False)
    mass = torch.tensor(MASSES, dtype=torch.float64)[ex["atom_types"].cpu()]
    vel0 = _velocities(mass, [300.0], [N], seed=3)
    f0 = _eager(model, ex, ex["pos"])[1]
    m = md.GraphedMD(model, ex, MASSES, DT_FS, "nose_hoover", temperature=300.0, nvt_q=50.0, velocities=vel0)
    assert m._nblk == 64
    fmax = float(f0.abs().max())
    _close(m.state["forces"], f0, F64_AGREE * fmax, "F(0)")
    ref = _Ref(ex, MASSES, [300.0], [50.0], True, m.state["vel"].clone(), f0)
    n = 5
    log = m.run(n, block=n)
    states, want = _host_loop(model, ex, ref, n, m.dt)
    dx, dv, bl = _bounds(n, m.dt, ref, fmax, max(float(s[1].abs().max()) for s in states), want)
    _close(m.state["pos"], states[-1][0], dx, "pos")
    _close(m.state["vel"], states[-1][1], dv, "vel")
    _close(m.state["zeta"], states[-1][2], bl[3], "zeta")
    _close(m.state["eta"], states[-1][3], bl[4], "eta")
    _close_log(log, want, bl)


# ------------------------------------------------------------------------------------------------------------------
# the log ring, blocks longer than the log, several calls, rollback
# ------------------------------------------------------------------------------------------------------------------
def _compare_runs(a, b, n, ref, what):
    """Run ``b`` against run ``a`` of one system, each (GraphedMD, log) after ``n`` steps: the logs and the final
    states, to ``_bounds``."""
    (ma, la), (mb, lb) = a, b
    fmax = max(float(ref.forces.abs().max()), float(ma.state["forces"].abs().max()))
    vmax = float(ma.state["vel"].abs().max())
    want = torch.stack([la[k] for k in md.LOG_FIELDS], 2)
    dx, dv, bl = _bounds(n, ma.dt, ref, fmax, vmax, want)
    _close_log(lb, want, bl, f"{what}: ")
    _close(mb.state["pos"], ma.state["pos"], dx, f"{what}: pos")
    _close(mb.state["vel"], ma.state["vel"], dv, f"{what}: vel")
    _close(mb.state["zeta"], ma.state["zeta"], bl[3], f"{what}: zeta")
    _close(mb.state["eta"], ma.state["eta"], bl[4], f"{what}: eta")
    assert int(mb.state["step"]) == int(ma.state["step"]), what


@pytest.mark.timeout(600)
def test_log_ring_wrap_and_long_blocks_give_one_trajectory():
    """120 steps of the float64 batch under the bath, in blocks of 10, 30 (the block of steps 90-119 wraps around the
    end of the 100-row log) and 150 (longer than the log: a new log and a re-capture, which is not an overflow), and
    split over two calls, 70 steps in blocks of 30 then 50 in blocks of 40 (steps 70-109 wrap).  The blocks-of-10 run
    against the host loop and every other run against it, to ``_bounds`` of 120 steps; ``host_reads`` is the number
    of blocks, ``on_block`` sees the returned log, ``run(0)`` reads nothing.  Largest error / bound on an H100: 2.7e-4
    (the blocks-of-10 run against the host loop), 1.3e-4 between runs."""
    n = 120
    system = _system("mixed_batch")
    ex = system[0]
    E0 = ops.neighbor_list(ex["pos"], ex["cell"], ex["pbc"], R_MAX, batch=ex["batch"])["edge_index"].shape[1]
    runs = {}
    for block in (10, 30, 150):
        _ex, _model, m, ref = _start(system, "nose_hoover", capacity=2 * E0)
        seen = []
        log = m.run(n, block=block, on_block=seen.append)
        assert m.recaptures == 0 and m.host_reads == math.ceil(n / block) and int(m.state["step"]) == n, block
        assert m._log.shape[0] == max(md.DEFAULT_LOG_ROWS, block)
        for k in md.LOG_FIELDS:
            assert torch.equal(torch.cat([b[k] for b in seen]), log[k]), (block, k)
            assert log[k].shape == (n, 5)
        runs[block] = (m, log)
    # the blocks-of-10 run itself against the host loop
    m, log = runs[10]
    states, want = _host_loop(system[1], ex, ref, n, m.dt)
    fmax = max(float(ref.forces.abs().max()), float(m.state["forces"].abs().max()))
    dx, dv, bl = _bounds(n, m.dt, ref, fmax, max(float(s[1].abs().max()) for s in states), want)
    _close_log(log, want, bl, "block 10 against the host loop: ")
    _close(m.state["pos"], states[-1][0], dx, "block 10 against the host loop: pos")
    _close(m.state["vel"], states[-1][1], dv, "block 10 against the host loop: vel")
    _ex, _model, m, ref = _start(system, "nose_hoover", capacity=2 * E0)
    none = m.run(0)
    assert all(v.shape == (0, 5) and v.dtype == torch.float64 for v in none.values()) and m.host_reads == 0
    first, second = m.run(70, block=30), m.run(50, block=40)
    assert m.host_reads == 3 + 2 and m.recaptures == 0
    split = {k: torch.cat([first[k], second[k]]) for k in md.LOG_FIELDS}
    for what, run in (("block 30", runs[30]), ("block 150", runs[150]), ("split", (m, split))):
        _compare_runs(runs[10], run, n, ref, what)


@pytest.mark.timeout(600)
def test_rollback_restores_the_bath_and_every_frame():
    """30 steps of the float64 batch under the bath in blocks of 10, from capacity E0 // 2 (the first block overflows,
    is rolled back, re-captured and run again) and from the default capacity.  zeta, eta, the step, the state and
    every log field agree to ``_bounds`` of 30 steps.  A different capacity only changes the null edges, which add
    exact zeros, yet on an H100 the energies were bitwise equal for the first 0 and the first 6 steps in two runs and
    never over all 30: F(0) comes from two eager calls and the forces and a frame's energy are float64 atomic sums in
    arrival order, so the last bits part and then grow.  So nothing is asserted bitwise.  Largest error / bound on an
    H100 over two runs: 2.6e-3 (positions, 3.6e-15 of 1.4e-12 Angstrom)."""
    system = _system("mixed_batch")
    ex = system[0]
    E0 = ops.neighbor_list(ex["pos"], ex["cell"], ex["pbc"], R_MAX, batch=ex["batch"])["edge_index"].shape[1]
    _ex, _model, small, ref = _start(system, "nose_hoover", capacity=E0 // 2)
    seen = []
    log_s = small.run(30, block=10, on_block=lambda b: seen.append(b["e_pot"].shape[0]))
    _ex, _model, ample, _r = _start(system, "nose_hoover")
    log_a = ample.run(30, block=10)
    assert small.recaptures >= 1 and small.capacity >= E0 and seen == [10, 10, 10]
    assert small.host_reads == 3 + small.recaptures and ample.host_reads == 3 + ample.recaptures
    _compare_runs((ample, log_a), (small, log_s), 30, ref, "rollback")


# ------------------------------------------------------------------------------------------------------------------
# time reversal
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(600)
def test_nve_retraces_its_path_with_negated_velocities():
    """50 NVE steps of the float64 model on the periodic water box, then the velocities negated in place and 50 more:
    velocity Verlet is time-reversible, so the positions return to the start and the velocities to minus the initial
    ones, to ``_bounds`` of 100 steps (a kick that is not symmetric about the drift moves the end point by O(dt^2)).
    Largest error / bound on an H100: 8.6e-4 (positions, 1.5e-14 of 1.8e-11 Angstrom)."""
    _ex, _model, m, ref = _start(_system("water"), None)
    x0, v0 = m.state["pos"].clone(), m.state["vel"].clone()
    n = 50
    m.run(n, block=25)
    fmax = max(float(ref.forces.abs().max()), float(m.state["forces"].abs().max()))
    dx, dv, _ = _bounds(2 * n, m.dt, ref, fmax, 0.0, torch.zeros(0, 1, 6))
    assert float((m.state["pos"] - x0).abs().max()) > 1e3 * dx  # the atoms went somewhere
    m.state["vel"].neg_()
    m.run(n, block=25)
    _close(m.state["pos"], x0, dx, "pos")
    _close(m.state["vel"], -v0, dv, "vel")
    assert int(m.state["step"]) == 2 * n
