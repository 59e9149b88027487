"""The float64 flexible-cell NPT oracle (tests/npt_flex_oracle.py) on the CPU, driven by the periodic shifted-force
Lennard-Jones of tests/test_relax.py (as tests/test_npt_integrator.py): the Jacobi-based matrix functions equal
scipy's matrix exponential and its integral, H is conserved to O(dt^2), the step is time-reversible and covariant
under a rotation of the whole system, an isotropic start follows the isotropic oracle, a sheared and strained crystal
relaxes its shape to the cube of the 1-D enthalpy minimum, and the barostat's kinetic energy equipartitions over its 6
degrees of freedom.  Also every new argument check of ``GraphedNPT`` raises ``ValueError`` on CPU tensors."""
import math

import numpy as np
import pytest
import scipy.linalg as sl
import torch
from scipy.optimize import minimize_scalar

import md_oracle as mo
import npt_flex_oracle as fo
import npt_oracle as no
from nequip_b200.npt import GraphedNPT
from test_npt_integrator import MASS, _cpu_example, lj_forces
from test_relax import fcc, lj_energy

# a symmetric shear and strain of a few percent (rows of the cell and positions map as a -> (I + STRAIN) a)
STRAIN = np.array([[0.02, 0.015, -0.01], [0.015, -0.01, 0.012], [-0.01, 0.012, 0.005]])


def _start(a, T, p, tchain, pchain, tdamp_fs, pdamp_fs, jitter=0.0, seed=0, tloop=1, ploop=1, strain=None,
           rot=None, vel=True):
    pos, cell = fcc(a)
    pos = pos + jitter * np.random.default_rng(seed).standard_normal(pos.shape)
    if strain is not None:
        Fd = np.eye(3) + strain
        pos, cell = pos @ Fd.T, cell @ Fd.T
    N = len(pos)
    m = torch.full((N,), MASS, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(N, 3, generator=g, dtype=torch.float64) * math.sqrt(mo.KB * T / MASS)
    v -= v.mean(0)
    if not vel:
        v.zero_()
    if rot is not None:
        pos, cell, v = pos @ rot.T, cell @ rot.T, v @ torch.tensor(rot).T
    prm = fo.Params([N], torch.tensor(cell), T, p, tdamp_fs * mo.FS, pdamp_fs * mo.FS, tchain, pchain, tloop, ploop)
    e, f, vir = lj_forces(torch.tensor(pos), torch.tensor(cell))
    st = fo.State(torch.tensor(pos), v, f, m, vir, prm)
    st.e_pot = [float(e)]
    return st, prm


def _offdiag(c):
    c = torch.as_tensor(c).reshape(3, 3)
    return float((c - torch.diag(c.diagonal())).abs().max())


# ------------------------------------------------------------------------------------------------------------------
# the matrix functions
# ------------------------------------------------------------------------------------------------------------------
def _random_rotation(rng):
    q, r = np.linalg.qr(rng.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _matrices():
    rng = np.random.default_rng(5)
    out = []
    for nu in np.logspace(-12, 0, 13):  # ||v_g dt||_2 = nu
        for _ in range(4):
            a = rng.standard_normal((3, 3))
            a = a + a.T
            out.append((f"random{nu:.0e}", a * nu / np.linalg.norm(a, 2)))
    R = _random_rotation(rng)
    out += [("diagonal", np.diag([0.3, -0.1, 0.02])), ("zero", np.zeros((3, 3))),
            ("double", R @ np.diag([0.2, 0.2, -0.5]) @ R.T), ("triple", R @ (0.4 * np.eye(3)) @ R.T),
            ("near_double", R @ np.diag([0.2, 0.2 * (1 + 1e-9), -0.5]) @ R.T),
            ("near_triple", R @ np.diag([0.4, 0.4 * (1 + 1e-12), 0.4 * (1 - 1e-12)]) @ R.T),
            ("tiny_offdiag", np.diag([0.1, 0.3, -0.2]) + 1e-200 * np.ones((3, 3)))]
    return out


def _integral(A, t):
    """int_0^t e^{A s} ds: the top-right block of expm([[A t, I t], [0, 0]])."""
    B = np.zeros((6, 6))
    B[:3, :3], B[:3, 3:] = A * t, np.eye(3) * t
    return sl.expm(B)[:3, 3:]


def test_matrix_functions_match_expm():
    """E_r = e^{v_g dt}, D = int_0^dt e^{v_g s} ds, E_v = e^{-M dt/2} and K = int_0^{dt/2} e^{-M s} ds (M = v_g + tr v_g
    / N_f I) from one Jacobi decomposition equal scipy's expm to 4e-15 of each matrix's size, for random symmetric v_g
    with ||v_g dt|| from 1e-12 to 1 and for diagonal, zero, doubly and triply degenerate and nearly degenerate ones;
    each is exactly symmetric."""
    dt, Nf = 1.0, 96.0
    worst = 0.0
    for name, a in _matrices():
        Ev, K, Er, D, _o = (np.array(x).reshape(3, 3) for x in fo.coefs(a.reshape(-1).tolist(), Nf, dt))
        M = a + np.trace(a) / Nf * np.eye(3)
        want = {"E_r": sl.expm(a * dt), "D": _integral(a, dt), "E_v": sl.expm(-M * dt / 2),
                "K": _integral(-M, dt / 2)}
        for key, got in (("E_r", Er), ("D", D), ("E_v", Ev), ("K", K)):
            assert np.array_equal(got, got.T), (name, key)
            err = np.abs(got - want[key]).max() / np.abs(want[key]).max()
            worst = max(worst, err)
            assert err <= 4e-15, (name, key, err)
    print(f"worst relative error {worst:.3g}")


def test_diagonal_v_g_takes_no_rotation_and_the_isotropic_formulas():
    """A diagonal v_g leaves O = I exactly, the matrices diagonal, and each axis's coefficients equal the isotropic
    oracle's formulas bitwise (E_r, D) or with mu = lambda + tr / N_f in place of alpha v_eps (E_v, K); for v_g = v I
    that mu differs from alpha v only by rounding (1e-15 relative)."""
    dt, Nf = 2.0 * mo.FS, 96.0
    for d in ([0.003, -0.001, 0.0005], [0.002, 0.002, 0.002], [0.0, 0.0, 0.0]):
        g = [d[0], 0.0, 0.0, 0.0, d[1], 0.0, 0.0, 0.0, d[2]]
        Ev, K, Er, D, o = fo.coefs(g, Nf, dt)
        assert o == fo.EYE
        tr = d[0] + d[1] + d[2]
        for k in range(3):
            ev, kf, _er, _df = no._coefs(d[k] + tr / Nf, 1.0, dt)
            _ev, _kf, er, df = no._coefs(d[k], 1.0, dt)
            assert (Ev[4 * k], K[4 * k], Er[4 * k], D[4 * k]) == (ev, kf, er, df)
            iso = no._coefs(d[k], 1.0 + 3.0 / Nf, dt)
            if d[0] == d[1] == d[2]:
                for got, want in zip((Ev[4 * k], K[4 * k], Er[4 * k], D[4 * k]), iso):
                    assert abs(got - want) <= 1e-15 * abs(want)
        for X in (Ev, K, Er, D):
            assert all(X[i] == 0.0 for i in (1, 2, 3, 5, 6, 7))


# ------------------------------------------------------------------------------------------------------------------
# the integrator
# ------------------------------------------------------------------------------------------------------------------
def _h_drift(dt_fs, n_fs, chains):
    st, prm = _start(1.56, 300.0, 0.05, *chains, 100.0, 1000.0, jitter=0.02, tloop=2, ploop=2, strain=STRAIN)
    h0 = fo.conserved(st, prm)[0]
    c0 = st.cell[0].clone()
    drift = shear = 0.0
    for _ in range(round(n_fs / dt_fs)):
        fo.step(st, prm, dt_fs * mo.FS, lj_forces)
        drift = max(drift, abs(fo.conserved(st, prm)[0] - h0))
        shear = max(shear, _offdiag(st.cell[0] - c0))
    return drift, shear


@pytest.mark.parametrize("chains", [(0, 0), (3, 3)], ids=["nph", "nhc3"])
def test_conserved_quantity_error_scales_as_dt_squared(chains):
    """1.5 ps of a rattled, sheared and strained 32-atom crystal at 300 K and 0.05 eV / Angstrom^3 at dt = 2 fs and
    1 fs (tloop = ploop = 2): the largest |H(t) - H(0)| falls by 4 +- 0.4, and the cell's off-diagonal entries moved."""
    big, shear = _h_drift(2.0, 1500.0, chains)
    small, _ = _h_drift(1.0, 1500.0, chains)
    print(f"H drift {big:.4g} / {small:.4g} = {big / small:.4f}, off-diagonal change {shear:.3g}")
    assert 3.6 <= big / small <= 4.4, (big, small)
    assert shear > 1e-3


def test_step_is_time_reversible():
    """100 steps with both chains (tloop = ploop = 2) from the sheared crystal, then every velocity negated (v, v_g,
    v_xi, v_eta) and 100 more: positions, cell and the chain positions return to the start to round-off."""
    st, prm = _start(1.56, 300.0, 0.05, 3, 3, 100.0, 1000.0, jitter=0.02, tloop=2, ploop=2, strain=STRAIN)
    x0, c0 = st.pos.clone(), st.cell.clone()
    dt = 2.0 * mo.FS
    for _ in range(100):
        fo.step(st, prm, dt, lj_forces)
    assert float((st.pos - x0).abs().max()) > 1e-2 and _offdiag(st.cell[0] - c0[0]) > 1e-4
    assert min(abs(x) for x in st.xi[0] + st.eta[0]) > 0
    fo.reverse(st)
    for _ in range(100):
        fo.step(st, prm, dt, lj_forces)
    print(f"reversal: |dx| {float((st.pos - x0).abs().max()):.3g}, |dC| {float((st.cell - c0).abs().max()):.3g}")
    assert float((st.pos - x0).abs().max()) <= 1e-12
    assert float((st.cell - c0).abs().max()) <= 1e-12
    assert max(abs(x) for x in st.xi[0] + st.eta[0]) <= 1e-10


def test_rotated_system_gives_the_rotated_trajectory():
    """The sheared crystal and its copy rotated by R (positions, cell rows and velocities; the LJ forces and virial
    rotate with them) for 60 steps with chains: positions, cell, v_g -> R v_g R^T and the chains agree to round-off."""
    R = _random_rotation(np.random.default_rng(11))
    a, prm = _start(1.56, 300.0, 0.05, 3, 3, 100.0, 1000.0, jitter=0.02, strain=STRAIN)
    b, prm_b = _start(1.56, 300.0, 0.05, 3, 3, 100.0, 1000.0, jitter=0.02, strain=STRAIN, rot=R)
    Rt = torch.tensor(R)
    dt = 2.0 * mo.FS
    for _ in range(60):
        fo.step(a, prm, dt, lj_forces)
        fo.step(b, prm_b, dt, lj_forces)
    ga, gb = (torch.tensor(s.g[0], dtype=torch.float64).view(3, 3) for s in (a, b))
    assert float(ga.abs().max()) > 1e-5
    assert float((b.pos - a.pos @ Rt.T).abs().max()) <= 1e-11
    assert float((b.vel - a.vel @ Rt.T).abs().max()) <= 1e-11 * float(a.vel.abs().max())
    assert float((b.cell[0] - a.cell[0] @ Rt.T).abs().max()) <= 1e-12
    assert float((gb - Rt @ ga @ Rt.T).abs().max()) <= 1e-11 * float(ga.abs().max())
    assert max(abs(x - y) for x, y in zip(a.xi[0] + a.eta[0], b.xi[0] + b.eta[0])) <= 1e-11


def test_isotropic_start_follows_the_isotropic_oracle():
    """A perfect fcc lattice at rest under p = 0.3 eV / Angstrom^3 with pchain = 0 (tchain = 3): 200 steps of the
    flexible oracle equal tests/npt_oracle.py with the same arguments (W = 3 W_g) to 1e-12 relative -- positions,
    the cell against C0 e^eps, volume and H; v_g against v_eps I to 5e-12 of the largest |v_eps| (1.3e-12 when
    written) -- and the off-diagonal cell entries stay at round-off."""
    dt = 2.0 * mo.FS
    st, prm = _start(1.56, 300.0, 0.3, 3, 0, 100.0, 500.0, vel=False)
    iprm = no.Params([st.pos.shape[0]], prm.C0, 300.0, 0.3, 100.0 * mo.FS, 500.0 * mo.FS, 3, 0)
    assert iprm.W[0] == pytest.approx(3 * prm.W[0], rel=1e-15)
    ist = no.State(st.pos, st.vel, st.forces, st.mass, st.vir, iprm)
    ist.e_pot = list(st.e_pot)
    vmax = 0.0
    for _ in range(200):
        fo.step(st, prm, dt, lj_forces)
        no.step(ist, iprm, dt, lj_forces)
        vmax = max(vmax, abs(ist.veps[0]))
    assert abs(ist.eps[0]) > 1e-3
    assert float((st.pos - ist.pos).abs().max()) <= 1e-12 * float(ist.pos.abs().max())
    assert float((st.cell - ist.cell).abs().max()) <= 1e-12 * float(ist.cell.abs().max())
    g = st.g[0]
    print(f"|v_g - v_eps I| / max|v_eps| = {max(abs(g[4 * k] - ist.veps[0]) for k in range(3)) / vmax:.3g}")
    assert max(abs(g[4 * k] - ist.veps[0]) for k in range(3)) <= 5e-12 * vmax
    assert max(abs(g[k]) for k in (1, 2, 3, 5, 6, 7)) <= 1e-12 * vmax  # driven by the virial's off-diagonal round-off
    assert _offdiag(st.cell[0]) <= 1e-14
    assert fo.volume(st)[0] == pytest.approx(no.volume(ist, iprm)[0], rel=1e-12)
    assert fo.conserved(st, prm)[0] == pytest.approx(no.conserved(ist, iprm)[0], rel=1e-12)


def test_sheared_crystal_relaxes_to_the_cube_of_the_enthalpy_minimum():
    """The 32-atom fcc crystal at 1 K started under the symmetric shear and strain STRAIN (up to 2 %), with chains
    (tau_T = 100 fs, tau_P = 20 ps as in the isotropic test): over 8 ps the mean metric C C^T of the last 4 ps is
    (2 a*)^2 I to 1e-3 relative, a* the minimum of E(a) + p V(a).  Isotropic NPT keeps the initial shear."""
    p = 0.05

    def H(a):
        pos, cell = fcc(a)
        return float(lj_energy(torch.tensor(pos), torch.tensor(cell), nimg=1)) + p * (2 * a) ** 3

    a_star = minimize_scalar(H, bracket=(1.5, 1.6), tol=1e-12).x
    st, prm = _start(a_star, 1.0, p, 3, 3, 100.0, 20000.0, strain=STRAIN)
    metric = []
    n = 4000
    for k in range(n):
        fo.step(st, prm, 2.0 * mo.FS, lj_forces)
        if k >= n // 2:
            c = st.cell[0]
            metric.append(c @ c.T)
    mean = torch.stack(metric).mean(0) / (2 * a_star) ** 2
    err = float((mean - torch.eye(3, dtype=torch.float64)).abs().max())
    print(f"mean metric / (2 a*)^2 - I: max {err:.3g}")
    assert err <= 1e-3
    assert _offdiag(prm.C0[0] @ prm.C0[0].T) / (2 * a_star) ** 2 > 2e-2  # the start was sheared


def test_barostat_kinetic_energy_equipartitions_over_six_degrees_of_freedom():
    """The rattled crystal at 300 K with chains of 3 and tau_P = 200 fs for 10 ps: over the last 9 ps
    <W_g tr(v_g^2)> = 6 kT within 3 standard errors of 10 block averages (1.08 +- 0.05 when written), and the error bar
    is below 15 %.  A barostat chain with 1 degree of freedom would hold it at kT instead."""
    st, prm = _start(1.56, 300.0, 0.05, 3, 3, 100.0, 200.0, jitter=0.02, strain=STRAIN)
    dt = 2.0 * mo.FS
    kb = []
    for _ in range(5000):
        fo.step(st, prm, dt, lj_forces)
        kb.append(prm.W[0] * fo.frob2(st.g[0]))
    x = np.array(kb[500:]) / (6 * prm.kT[0])
    blocks = x[: len(x) // 10 * 10].reshape(10, -1).mean(1)
    mean, err = x.mean(), blocks.std(ddof=1) / math.sqrt(10)
    print(f"<W_g tr v_g^2> / 6 kT = {mean:.4f} +- {err:.4f}")
    assert abs(mean - 1.0) <= 3 * err and err < 0.15


# ------------------------------------------------------------------------------------------------------------------
# arguments
# ------------------------------------------------------------------------------------------------------------------
_OK = dict(tdamp_fs=100.0, pdamp_fs=1000.0)


@pytest.mark.parametrize("barostat", ["anisotropic", "Flexible", None, 1])
def test_unknown_barostat_raises_before_cuda(barostat):
    with pytest.raises(ValueError, match="barostat"):
        GraphedNPT(None, _cpu_example(), [1.0] * 4, 1.0, 300.0, 0.0, barostat=barostat, **_OK)


@pytest.mark.parametrize("kw,match", [
    (dict(timestep_fs=0.0), "timestep_fs"),
    (dict(temperature=-1.0), "temperature"),
    (dict(pressure=float("nan")), "pressure"),
    (dict(pdamp_fs=-5.0), "pdamp_fs"),
    (dict(pchain=9), "pchain"),
    (dict(ploop=0), "ploop"),
    (dict(masses=[1.0, 1.0]), "masses"),
])
def test_flexible_keeps_the_argument_checks(kw, match):
    args = dict(masses=[1.0] * 4, timestep_fs=1.0, temperature=300.0, pressure=0.0, **_OK)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        GraphedNPT(None, _cpu_example(), args.pop("masses"), args.pop("timestep_fs"), args.pop("temperature"),
                   args.pop("pressure"), barostat="flexible", **args)
    with pytest.raises(ValueError, match="periodic"):
        GraphedNPT(None, _cpu_example(pbc=torch.tensor([True, True, False])), [1.0] * 4, 1.0, 300.0, 0.0,
                   barostat="flexible", **_OK)
    with pytest.raises(RuntimeError, match="CUDA"):  # valid arguments: only then the device check
        GraphedNPT(None, _cpu_example(), [1.0] * 4, 1.0, 300.0, 0.0, barostat="flexible", **_OK)
