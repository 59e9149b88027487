"""The float64 relaxation oracle (tests/relax_oracle.py) on the CPU: the Frechet cell filter's generalised forces are
the exact derivatives of the enthalpy, its block-matrix Frechet derivative is scipy's, FIRE follows ASE's sequence,
a Lennard-Jones fcc crystal relaxes to the lattice constant of a 1-D minimisation (with and without pressure), and
every argument check of ``GraphedRelax`` raises ``ValueError`` on CPU tensors."""
import itertools

import numpy as np
import pytest
import torch
from scipy.linalg import expm, expm_frechet
from scipy.optimize import minimize_scalar

import relax_oracle as ro
from nequip_b200.relax import FIRE_DEFAULTS, GraphedRelax


def lj_energy(pos, cell, rc=2.5, nimg=2):
    """Shifted-force Lennard-Jones (epsilon = sigma = 1) of a periodic frame, float64 torch, by explicit images."""
    r = torch.arange(-nimg, nimg + 1, dtype=torch.float64)
    shifts = torch.cartesian_prod(r, r, r)
    d = pos[None, :, None, :] - pos[:, None, None, :] + (shifts @ cell)[None, None]
    r2 = (d * d).sum(-1)
    n = pos.shape[0]
    self_pair = torch.eye(n, dtype=torch.bool)[:, :, None] & (shifts.abs().sum(1) == 0)[None, None]
    inside = (r2 < rc * rc) & ~self_pair
    rr = torch.sqrt(torch.where(inside, r2, torch.ones_like(r2)))

    def e(x):
        return 4 * (x ** -12 - x ** -6)

    de_rc = 4 * (-12 * rc ** -13 + 6 * rc ** -7)
    pair = torch.where(inside, e(rr) - e(torch.tensor(rc, dtype=torch.float64)) - (rr - rc) * de_rc,
                       torch.zeros_like(rr))
    return 0.5 * pair.sum()


def lj_eval(pos, cell, **kw):
    """(E, forces, virial = -dE/d(eps)) of ``lj_energy`` at numpy pos / cell."""
    eps = torch.zeros(3, 3, dtype=torch.float64, requires_grad=True)
    p = torch.tensor(pos, dtype=torch.float64, requires_grad=True)
    c = torch.tensor(cell, dtype=torch.float64)
    D = torch.eye(3, dtype=torch.float64) + eps
    E = lj_energy(p @ D.T, c @ D.T, **kw)
    gp, ge = torch.autograd.grad(E, (p, eps))
    return float(E.detach()), -gp.numpy(), -ge.numpy()


def fcc(a, reps=2):
    basis = np.array([[0, 0, 0], [0.5, 0.5, 0], [0.5, 0, 0.5], [0, 0.5, 0.5]])
    pts = [(b + np.array(o)) for o in itertools.product(range(reps), repeat=3) for b in basis]
    return a * np.array(pts), a * reps * np.eye(3)


def test_generalised_forces_are_enthalpy_derivatives():
    """p != 0 on a triclinic cell, at a deformation Q != 0: g and G equal central differences of
    H(s, Q) = E(s Fd^T, C0 Fd^T) + p |det(C0 Fd^T)| to 1e-7 relative."""
    rng = np.random.default_rng(3)
    C0 = np.array([[3.1, 0.0, 0.0], [0.6, 2.9, 0.0], [-0.4, 0.5, 3.3]])
    s = rng.random((5, 3)) @ C0
    Q = 0.05 * rng.standard_normal((3, 3))
    c, p = 5.0, 0.07

    def H(s_flat, Qm):
        Fd = torch.matrix_exp(Qm / c)
        cell = torch.tensor(C0) @ Fd.T
        return float(lj_energy(s_flat.reshape(-1, 3) @ Fd.T, cell) + p * torch.det(cell).abs())

    Fd = expm(Q / c)
    E, forces, virial = lj_eval(s @ Fd.T, C0 @ Fd.T)
    g, G = ro.generalized_forces(forces, virial, Q, c, C0 @ Fd.T, p)
    h = 1e-5
    s_t, Q_t = torch.tensor(s.reshape(-1)), torch.tensor(Q)
    fd_g = np.zeros(s.size)
    for k in range(s.size):
        e = torch.zeros(s.size, dtype=torch.float64)
        e[k] = h
        fd_g[k] = -(H(s_t + e, Q_t) - H(s_t - e, Q_t)) / (2 * h)
    fd_G = np.zeros((3, 3))
    for u, v in itertools.product(range(3), repeat=2):
        e = torch.zeros(3, 3, dtype=torch.float64)
        e[u, v] = h
        fd_G[u, v] = -(H(s_t, Q_t + e) - H(s_t, Q_t - e)) / (2 * h)
    scale = max(np.abs(g).max(), np.abs(G).max())
    assert np.abs(fd_g.reshape(-1, 3) - g).max() <= 1e-7 * scale
    assert np.abs(fd_G - G).max() <= 1e-7 * scale
    assert np.abs(G).max() > 1e-2 and np.abs(G - G.T).max() > 0  # a non-trivial cell force


def test_block_frechet_derivative_equals_scipy():
    rng = np.random.default_rng(0)
    for scale in (1e-3, 0.3, 2.0):
        L, E = scale * rng.standard_normal((3, 3)), rng.standard_normal((3, 3))
        _, ref = expm_frechet(L, E)
        assert np.abs(ro.dexp(L, E) - ref).max() <= 1e-13 * max(1.0, np.abs(ref).max())


def test_fire_sequence_on_a_quadratic_bowl():
    k = np.array([1.0, 2.0, 0.5])
    x0 = np.array([[0.3, -0.2, 0.1]])
    fr = ro.Frame(x0, None, False, fmax=1e-12)
    f = lambda: -(k * fr.s)  # noqa: E731
    fr.evaluate(0.0, f())
    g0 = fr.g.copy()
    fr.step()  # first step: no mixing, v = dt g
    assert np.allclose(fr.s, x0 + 0.1 * 0.1 * g0, rtol=0, atol=1e-15)
    assert fr.Nsteps == 0 and fr.dt == 0.1
    dts = []
    for _ in range(8):  # downhill: v.g > 0 every step; dt grows only after Nmin = 5 mixing steps
        fr.evaluate(0.0, f())
        assert np.vdot(fr.v, fr.g) > 0
        fr.step()
        dts.append(fr.dt)
    assert dts[:6] == [0.1] * 6
    assert dts[6] == pytest.approx(0.11, rel=1e-15) and dts[7] == pytest.approx(0.121, rel=1e-15)
    assert fr.a == pytest.approx(0.1 * 0.99 ** 2, rel=1e-15)
    # reset: a force against the velocity
    fr.evaluate(0.0, -fr.v)
    dt = fr.dt
    s = fr.s.copy()
    g = fr.g.copy()
    fr.step()
    assert fr.Nsteps == 0 and fr.a == 0.1 and fr.dt == pytest.approx(dt * 0.5, rel=1e-15)
    assert np.allclose(fr.s - s, fr.dt * fr.dt * g, rtol=0, atol=1e-15)
    # maxstep clip: |dr| = maxstep over the whole vector
    big = ro.Frame(np.zeros((2, 3)), None, False)
    big.evaluate(0.0, np.full((2, 3), 50.0))
    big.step()
    assert np.linalg.norm(big.s) == pytest.approx(0.2, rel=1e-14)


def _relax_lj(pos, cell, p, fmax, steps=5000):
    fr = ro.Frame(pos, cell, True, fmax=fmax, p=p)
    for _ in range(steps):
        E, forces, virial = lj_eval(fr.positions(), fr.cell())
        fr.evaluate(E, forces, virial)
        if fr.converged:
            return fr, virial
        fr.step()
    raise AssertionError("the LJ relaxation did not converge")


@pytest.mark.parametrize("p", [0.0, 0.05])
def test_lj_fcc_relaxes_to_the_1d_minimum(p):
    """A rattled, strained 2x2x2 fcc cell relaxed with the filter reaches the lattice constant that minimises the
    enthalpy E(a) + p V(a) of the perfect crystal, and its stress -virial / V is -p I within what fmax allows."""
    def H(a):
        pos, cell = fcc(a)
        return float(lj_energy(torch.tensor(pos), torch.tensor(cell))) + p * (2 * a) ** 3

    a_star = minimize_scalar(H, bracket=(1.5, 1.6), tol=1e-12).x
    rng = np.random.default_rng(1)
    pos, cell = fcc(1.04 * a_star)
    strain = np.eye(3) + 0.02 * np.array([[1, 0.5, 0], [0.5, -1, 0.3], [0, 0.3, 0.5]])
    pos, cell = pos @ strain.T + 0.02 * rng.standard_normal(pos.shape), cell @ strain.T
    fmax = 1e-4
    fr, virial = _relax_lj(pos, cell, p, fmax)
    V = abs(np.linalg.det(fr.cell()))
    a = V ** (1 / 3) / 2
    assert abs(a - a_star) <= 1e-4 * a_star
    stress = -virial / V
    tol = 2 * np.sqrt(3) * fr.c * fmax / V
    assert np.abs(stress + p * np.eye(3)).max() <= tol
    assert fr.steps > 10


def _cpu_example(**kw):
    ex = {"pos": torch.zeros(4, 3), "atom_types": torch.zeros(4, dtype=torch.int64), "cell": 5 * torch.eye(3)}
    ex.update(kw)
    return ex


@pytest.mark.parametrize("kw,match", [
    (dict(fmax=0.0), "fmax"),
    (dict(fmax=float("nan")), "fmax"),
    (dict(fail_force=-1.0), "fail_force"),
    (dict(cell_filter="ucf"), "cell_filter"),
    (dict(scalar_pressure=0.1), "cell_filter"),
    (dict(exp_cell_factor=4.0), "cell_filter"),
    (dict(cell_filter="frechet", scalar_pressure=float("inf")), "scalar_pressure"),
    (dict(cell_filter="frechet", exp_cell_factor=0.0), "exp_cell_factor"),
    (dict(dt=0.0), "dt"),
    (dict(maxstep=-0.1), "maxstep"),
    (dict(dtmax=float("inf")), "dtmax"),
    (dict(finc=0.0), "finc"),
    (dict(fdec=0.0), "fdec"),
    (dict(astart=1.5), "astart"),
    (dict(fa=-0.1), "fa"),
    (dict(a=2.0), "a must"),
    (dict(Nmin=-1), "Nmin"),
    (dict(Nmin=2.5), "Nmin"),
    (dict(beta=1.0), "unknown"),
])
def test_argument_checks_raise_before_cuda(kw, match):
    with pytest.raises(ValueError, match=match):
        GraphedRelax(None, _cpu_example(), **kw)


def test_example_checks_raise_before_cuda():
    with pytest.raises(ValueError, match="periodic"):  # the filter needs every frame fully periodic
        GraphedRelax(None, _cpu_example(pbc=torch.tensor([True, True, False])), cell_filter="frechet")
    with pytest.raises(ValueError, match="periodic"):
        GraphedRelax(None, _cpu_example(cell=None), cell_filter="frechet")
    with pytest.raises(ValueError, match="num_atoms"):
        GraphedRelax(None, _cpu_example(batch=torch.tensor([0, 0, 1, 1]), num_atoms=torch.tensor([2, 1]),
                                        cell=5 * torch.eye(3).expand(2, 3, 3)))
    with pytest.raises(ValueError, match="cell must be"):
        GraphedRelax(None, _cpu_example(cell=torch.eye(2)))
    with pytest.raises(ValueError, match="singular"):
        GraphedRelax(None, _cpu_example(cell=torch.zeros(3, 3)))
    with pytest.raises(ValueError, match="finite"):
        GraphedRelax(None, _cpu_example(cell=torch.full((3, 3), float("nan"))))
    with pytest.raises(RuntimeError, match="CUDA"):  # valid arguments: only then the device check
        GraphedRelax(None, _cpu_example())


def test_fire_defaults_are_ases():
    assert FIRE_DEFAULTS == ro.FIRE_DEFAULTS
