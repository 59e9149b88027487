"""CPU checks of the device MD driver's physics (nequip_b200/md.py) on the float64 oracle (tests/md_oracle.py): the unit
constants, time reversibility and the dt^2 energy error of velocity Verlet, the Nose-Hoover conserved quantity and the
bath's control of the temperature, the initial-velocity clean-up, and the argument checks of ``GraphedMD``."""
import pytest
import torch

import md_oracle as mo
from nequip_b200 import data as D
from nequip_b200 import md
from nequip_b200.nn.model import NequIPEnergyModel


def test_unit_constants_match_codata_2014():
    assert md.KB == pytest.approx(mo.KB, rel=1e-15)
    assert md.FS == pytest.approx(mo.FS, rel=1e-15)


def _harmonic_crystal(n=4, a=2.0, k=3.0, seed=0):
    """A periodic simple-cubic crystal of n^3 atoms joined to their 6 neighbours by springs on the displacement vectors,
    E = k/2 sum_bonds |u_j - u_i|^2 (plus a weak tether that pins the lattice's translation), with masses 1..4 amu."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.arange(n ** 3).view(n, n, n)
    i_list, j_list = [], []
    for d in range(3):
        i_list.append(idx.reshape(-1))
        j_list.append(torch.roll(idx, -1, dims=d).reshape(-1))
    bi, bj = torch.cat(i_list), torch.cat(j_list)
    grid = torch.stack(torch.meshgrid(*[torch.arange(n, dtype=torch.float64)] * 3, indexing="ij"), -1).view(-1, 3)
    x0 = a * grid
    mass = 1.0 + torch.randint(0, 4, (n ** 3,), generator=g).double()
    u0 = 0.05 * torch.randn(n ** 3, 3, generator=g, dtype=torch.float64)

    def force_fn(pos):
        u = pos - x0
        du = u[bj] - u[bi]
        e = 0.5 * k * (du ** 2).sum() + 0.5 * 1e-3 * (u ** 2).sum()
        f = torch.zeros_like(pos).index_add_(0, bj, -k * du).index_add_(0, bi, k * du) - 1e-3 * u
        return e.view(1), f

    return x0 + u0, mass, force_fn


def _run(pos, vel, mass, force_fn, dt, n):
    ptr = [0, pos.shape[0]]
    gkT, Q = torch.zeros(1, dtype=torch.float64), torch.ones(1, dtype=torch.float64)
    zeta, eta = torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    e, f = force_fn(pos)
    H = [mo.conserved(e, vel, mass, zeta, eta, gkT, Q, ptr)]
    for _ in range(n):
        pos, vel, f, zeta, eta, e = mo.nh_step(pos, vel, f, mass, zeta, eta, force_fn, dt, gkT, Q, ptr, False)
        H.append(mo.conserved(e, vel, mass, zeta, eta, gkT, Q, ptr))
    return pos, vel, torch.cat(H)


def test_verlet_is_time_reversible_and_its_energy_error_scales_as_dt2():
    pos0, mass, force_fn = _harmonic_crystal()
    vel0 = md.maxwell_boltzmann(mass, torch.full((mass.shape[0],), 300.0), seed=1)
    dt = 1.0 * mo.FS
    pos, vel, *_ = _run(pos0, vel0, mass, force_fn, dt, 200)
    back, vback, *_ = _run(pos, -vel, mass, force_fn, dt, 200)
    assert float((back - pos0).abs().max()) <= 1e-12 * float(pos0.abs().max())
    assert float((vback + vel0).abs().max()) <= 1e-12 * float(vel0.abs().max())
    # the largest energy error over the same time span, at dt and dt / 2
    errs = []
    for h in (dt, dt / 2, dt / 4):
        _, _, H = _run(pos0, vel0, mass, force_fn, h, int(round(200 * dt / h)))
        errs.append(float((H - H[0]).abs().max()))
    for coarse, fine in zip(errs, errs[1:]):
        assert 3.5 <= coarse / fine <= 4.5, errs


def _nose_hoover(dt_fs, span_fs=2000.0, Q=50.0, T=300.0):
    """The harmonic crystal started at 2 T under the bath at T: H, H with the bath term Q zeta^2 / 2, and 2 K."""
    pos0, mass, force_fn = _harmonic_crystal()
    N = mass.shape[0]
    vel = md.maxwell_boltzmann(mass, torch.full((N,), 2 * T), seed=2)
    gkT = torch.tensor([(3 * N + 1) * mo.KB * T], dtype=torch.float64)
    Q = torch.tensor([Q], dtype=torch.float64)
    ptr = [0, N]
    pos, (e, f) = pos0, force_fn(pos0)
    zeta, eta = torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)
    H, H_half, twoK = [], [], []
    for _ in range(int(round(span_fs / dt_fs))):
        pos, vel, f, zeta, eta, e = mo.nh_step(pos, vel, f, mass, zeta, eta, force_fn, dt_fs * mo.FS, gkT, Q, ptr)
        H.append(float(mo.conserved(e, vel, mass, zeta, eta, gkT, Q, ptr)))
        H_half.append(H[-1] - 0.5 * float(Q * zeta ** 2))
        twoK.append(float(2 * mo.kinetic(vel, mass, ptr)))
    f64 = dict(dtype=torch.float64)
    return torch.tensor(H, **f64), torch.tensor(H_half, **f64), torch.tensor(twoK, **f64), (3 * N + 1) * mo.KB


def test_nose_hoover_conserves_h_and_controls_the_temperature():
    """Over 2 ps from twice the target temperature, H = E_pot + E_kin + Q zeta^2 + g k_B T eta drifts by less than 3 %
    of the kinetic energy at 0.5 fs, and the drift halves with dt: the reference's update conserves H to first order
    in dt (its bath half-steps use v(t) and v(t + dt/2), both before the new forces).  H with the bath term
    Q zeta^2 / 2 (wrong for the reference's zeta rate (2K - g k_B T) / (2Q)) keeps a drift of ~9 % that does not
    shrink with dt.  The time average of 2 K / (g k_B) over the last 3/4 of the run is within 3 % of T."""
    T = 300.0
    H1, Hw1, twoK1, gk = _nose_hoover(0.5, T=T)
    H2, Hw2, _, _ = _nose_hoover(0.25, T=T)
    K0 = 0.5 * float(twoK1[0])
    d1, d2 = float((H1 - H1[0]).abs().max()), float((H2 - H2[0]).abs().max())
    assert d1 <= 0.03 * K0, d1 / K0
    assert 1.7 <= d1 / d2 <= 2.3, (d1, d2)
    assert float((Hw2 - Hw2[0]).abs().max()) >= 5 * d2
    assert twoK1[0] / gk > 1.5 * T
    t_avg = float(twoK1[len(twoK1) // 4:].mean()) / gk
    assert abs(t_avg - T) <= 0.03 * T, t_avg


def test_initial_velocities_have_no_momentum_and_no_rotation_per_frame():
    g = torch.Generator().manual_seed(3)
    counts = [7, 1, 12, 3]
    ptr = [0] + torch.cumsum(torch.tensor(counts), 0).tolist()
    N = ptr[-1]
    pos = 4 * torch.randn(N, 3, generator=g, dtype=torch.float64)
    pos[ptr[3]:ptr[4]] = torch.tensor([[0.0, 0, 0], [1, 1, 1], [2, 2, 2]], dtype=torch.float64)  # a line of atoms
    mass = 1 + 15 * torch.rand(N, generator=g, dtype=torch.float64)
    vel = md.maxwell_boltzmann(mass, torch.full((N,), 500.0), seed=4)
    out = md.zero_rotation_and_momentum(pos, vel, mass, ptr)
    for f in range(len(counts)):
        a, b = ptr[f], ptr[f + 1]
        m, r, v = mass[a:b, None], pos[a:b], out[a:b]
        p = (m * v).sum(0)
        assert float(p.abs().max()) <= 1e-12 * float((m * vel[a:b]).abs().sum())
        r = r - (m * r).sum(0) / m.sum()
        L = torch.cross(r, m * v, dim=1).sum(0)
        assert float(L.abs().max()) <= 1e-11 * float((r.norm(dim=1, keepdim=True) * m * vel[a:b].abs()).sum()) + 1e-300
    assert float(out[ptr[1]:ptr[2]].abs().max()) == 0.0  # one atom: nothing left
    assert float(out.abs().max()) > 0


def _cpu_case(**kw):
    s = D.make_system("water", 3, r_max=4.0, seed=0)
    meta = s.pop("_meta")
    model = NequIPEnergyModel(r_max=4.0, type_names=meta["type_names"], l_max=1, num_layers=1, num_features=8,
                              radial_mlp_depth=1, radial_mlp_width=8, avg_num_neighbors=meta["avg_num_neighbors"])
    ex = {"pos": s["pos"], "atom_types": s["atom_types"].view(-1), "cell": s["cell"]}
    args = dict(masses=[1.008, 15.999], timestep_fs=0.5)
    args.update(kw)
    return model, ex, args


@pytest.mark.parametrize("kw,match", [
    (dict(variable_cell=True), "variable_cell"),
    (dict(masses=[1.0, 2.0, 3.0]), "masses"),
    (dict(masses=[1.0, -2.0]), "masses"),
    (dict(thermostat="nose_hoover", nvt_q=334.0), "temperature and nvt_q"),
    (dict(thermostat="nose_hoover", temperature=300.0), "temperature and nvt_q"),
    (dict(thermostat="langevin", temperature=300.0, nvt_q=1.0), "thermostat"),
    (dict(timestep_fs=0.0), "timestep_fs"),
    (dict(thermostat="nose_hoover", temperature=[300.0, 310.0], nvt_q=334.0), "temperature"),
    (dict(thermostat="nose_hoover", temperature=300.0, nvt_q=-1.0), "nvt_q"),
    (dict(temperature=-5.0), "temperature"),
    (dict(velocities=torch.zeros(3, 3)), "velocities"),
])
def test_graphed_md_rejects_bad_arguments_on_cpu(kw, match):
    model, ex, args = _cpu_case(**kw)
    with pytest.raises(ValueError, match=match):
        md.GraphedMD(model, ex, **args)


def test_graphed_md_needs_cuda_after_the_checks():
    model, ex, args = _cpu_case(thermostat="nose_hoover", temperature=300.0, nvt_q=334.0)
    with pytest.raises(RuntimeError, match="CUDA"):
        md.GraphedMD(model, ex, **args)


def test_batch_arguments_are_per_frame():
    model, ex, args = _cpu_case()
    N = ex["pos"].shape[0]
    ex = dict(ex, batch=torch.zeros(N, dtype=torch.int64), num_atoms=torch.tensor([N - 1]))
    with pytest.raises(ValueError, match="num_atoms"):
        md.GraphedMD(model, ex, **args)
