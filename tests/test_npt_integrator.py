"""The float64 NPT oracle (tests/npt_oracle.py) on the CPU, driven by the periodic shifted-force Lennard-Jones of
tests/test_relax.py (epsilon = 1 eV, sigma = 1 Angstrom, 400 amu atoms): H is conserved to O(dt^2), the step is
time-reversible, it reduces to velocity Verlet without chains and with an infinitely heavy barostat, the cell keeps
its shape, and the time-averaged lattice constant at pressure p is the minimum of E(a) + p V(a) that the relaxation
test finds.  Also every argument check of ``GraphedNPT`` raises ``ValueError`` on CPU tensors."""
import math

import numpy as np
import pytest
import torch
from scipy.optimize import minimize_scalar

import md_oracle as mo
import npt_oracle as no
from nequip_b200 import md, npt
from nequip_b200.npt import GPA, GraphedNPT
from test_relax import fcc, lj_energy, lj_eval

MASS = 400.0  # amu: an LJ vibration period of about 50 fs


def lj_forces(pos, cell):
    """(E [1], forces [N, 3], virial [1, 3, 3]) of one periodic LJ frame (box > r_c, so one image shell)."""
    E, f, v = lj_eval(pos.reshape(-1, 3).numpy(), cell.reshape(3, 3).numpy(), nimg=1)
    return torch.tensor([E], dtype=torch.float64), torch.tensor(f), torch.tensor(v).reshape(1, 3, 3)


def _start(a, T, p, tchain, pchain, tdamp_fs, pdamp_fs, jitter=0.0, seed=0, tloop=1, ploop=1):
    pos, cell = fcc(a)
    pos = pos + jitter * np.random.default_rng(seed).standard_normal(pos.shape)
    N = len(pos)
    m = torch.full((N,), MASS, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(N, 3, generator=g, dtype=torch.float64) * math.sqrt(mo.KB * T / MASS)
    v -= v.mean(0)
    prm = no.Params([N], cell, T, p, tdamp_fs * mo.FS, pdamp_fs * mo.FS, tchain, pchain, tloop, ploop)
    e, f, vir = lj_forces(torch.tensor(pos), torch.tensor(cell))
    st = no.State(torch.tensor(pos), v, f, m, vir, prm)
    st.e_pot = [float(e)]
    return st, prm


def _h_drift(dt_fs, n_fs, chains):
    st, prm = _start(1.56, 300.0, 0.05, *chains, 100.0, 1000.0, jitter=0.02, tloop=2, ploop=2)
    h0 = no.conserved(st, prm)[0]
    drift = swing = 0.0
    for _ in range(round(n_fs / dt_fs)):
        no.step(st, prm, dt_fs * mo.FS, lj_forces)
        drift = max(drift, abs(no.conserved(st, prm)[0] - h0))
        swing = max(swing, abs(st.eps[0]))
    return drift, swing


@pytest.mark.parametrize("chains", [(0, 0), (3, 3)], ids=["nph", "nhc3"])
def test_conserved_quantity_error_scales_as_dt_squared(chains):
    """1.5 ps of a rattled 32-atom crystal at 300 K and 0.05 eV / Angstrom^3 at dt = 2 fs and 1 fs: the largest
    |H(t) - H(0)| falls by 4 +- 0.4 (3.995 and 3.998 when written), and the cell did move."""
    big, swing = _h_drift(2.0, 1500.0, chains)
    small, _ = _h_drift(1.0, 1500.0, chains)
    assert 3.6 <= big / small <= 4.4, (big, small)
    assert swing > 1e-3


def test_step_is_time_reversible():
    """100 steps with both chains (tloop = ploop = 2), then every velocity negated (v, v_eps, v_xi, v_eta) and 100
    more: positions, cell, eps and the chain positions return to the start to round-off (7e-15 Angstrom when
    written; the LJ crystal is chaotic, and after 200 steps each way the round-off has grown to 1e-9)."""
    st, prm = _start(1.56, 300.0, 0.05, 3, 3, 100.0, 1000.0, jitter=0.02, tloop=2, ploop=2)
    x0, c0 = st.pos.clone(), st.cell.clone()
    dt = 2.0 * mo.FS
    for _ in range(100):
        no.step(st, prm, dt, lj_forces)
    assert float((st.pos - x0).abs().max()) > 1e-2 and abs(st.eps[0]) > 1e-3
    assert min(abs(x) for x in st.xi[0] + st.eta[0]) > 0
    no.reverse(st)
    for _ in range(100):
        no.step(st, prm, dt, lj_forces)
    assert float((st.pos - x0).abs().max()) <= 1e-12
    assert float((st.cell - c0).abs().max()) <= 1e-12
    assert abs(st.eps[0]) <= 1e-13
    assert max(abs(x) for x in st.xi[0] + st.eta[0]) <= 1e-10


def test_reduces_to_velocity_verlet():
    """No chains and tau_P = 1e100 fs (W ~ 1e198): v_eps stays ~1e-198, every exponential is 1, and 20 steps equal
    md_oracle.nh_step without the bath to 1e-12."""
    st, prm = _start(1.56, 300.0, 0.05, 0, 0, 100.0, 1e100, jitter=0.02)
    pos, vel, f = st.pos.clone(), st.vel.clone(), st.forces.clone()
    ptr = prm.ptr
    zero = torch.zeros(1, dtype=torch.float64)
    cell = st.cell.clone()
    dt = 2.0 * mo.FS
    for _ in range(20):
        no.step(st, prm, dt, lj_forces)
        pos, vel, f, *_ = mo.nh_step(pos, vel, f, st.mass, zero, zero, lambda p: lj_forces(p, cell)[:2], dt, zero,
                                     zero, ptr, thermostat=False)
    assert float((st.pos - pos).abs().max()) <= 1e-12
    assert float((st.vel - vel).abs().max()) <= 1e-12
    assert abs(st.veps[0]) < 1e-190 and torch.equal(st.cell, cell)


def test_cell_keeps_its_shape():
    """A triclinic, left-handed cell under 300 steps of NPT: the cell is C0 e^eps bit for bit, and its shape
    cell / |det cell|^(1/3) equals C0's to 1e-15."""
    pos, _ = fcc(1.56)
    C0 = torch.tensor([[0.0, 3.12, 0.0], [3.12, 0.0, 0.0], [0.3, -0.2, 3.12]], dtype=torch.float64)
    frac = torch.linalg.solve(torch.tensor(fcc(1.56)[1]).T, torch.tensor(pos).T).T
    pos = frac @ C0
    N = pos.shape[0]
    m = torch.full((N,), MASS, dtype=torch.float64)
    v = torch.randn(N, 3, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 1e-3
    prm = no.Params([N], C0, 300.0, 0.2, 100.0 * mo.FS, 1000.0 * mo.FS, 3, 3)
    st = no.State(pos, v, lj_forces(pos, C0)[1], m, lj_forces(pos, C0)[2], prm)
    for _ in range(300):
        no.step(st, prm, 2.0 * mo.FS, lj_forces)
    assert abs(st.eps[0]) > 1e-3
    assert torch.equal(st.cell[0], C0 * math.exp(st.eps[0]))
    shape = lambda c: c / abs(float(torch.linalg.det(c))) ** (1 / 3)  # noqa: E731
    assert float((shape(st.cell[0]) - shape(C0)).abs().max()) <= 1e-15 * 3.2


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_mean_lattice_constant_is_the_enthalpy_minimum(p):
    """The 32-atom fcc crystal at 1 K started 0.2 % off: over 6 ps (3000 steps of 2 fs; the barostat's period is about
    80 fs) the mean lattice constant of the last 4 ps is the a* that minimises E(a) + p V(a) to 1e-4 relative (5e-6
    and 6e-6 when written).  p = 0.5 eV / Angstrom^3 moves a* by 2.6e-3 relative, so a pressure of the wrong sign or
    scale fails by an order of magnitude.  tau_P = 20 ps: W is proportional to T, and at 1 K a shorter tau_P makes
    the barostat faster than the time step allows."""
    def H(a):
        pos, cell = fcc(a)
        return float(lj_energy(torch.tensor(pos), torch.tensor(cell), nimg=1)) + p * (2 * a) ** 3

    a_star = minimize_scalar(H, bracket=(1.5, 1.6), tol=1e-12).x
    st, prm = _start(1.002 * a_star, 1.0, p, 3, 3, 100.0, 20000.0)
    a = []
    for _ in range(3000):
        no.step(st, prm, 2.0 * mo.FS, lj_forces)
        a.append(no.volume(st, prm)[0] ** (1 / 3) / 2)
    assert abs(np.mean(a[1000:]) / a_star - 1) <= 1e-4
    assert np.std(a[1000:]) > 1e-5 * a_star  # the cell moved


def test_constants():
    assert npt.GPA == pytest.approx(1e9 / 1.6021766208e-19 / 1e30, rel=1e-15)
    assert npt.MAX_CHAIN == no.MAX_CHAIN
    assert md.KB == pytest.approx(mo.KB, rel=1e-15)


def _cpu_example(**kw):
    ex = {"pos": torch.zeros(4, 3), "atom_types": torch.zeros(4, dtype=torch.int64), "cell": 5 * torch.eye(3)}
    ex.update(kw)
    return ex


_OK = dict(tdamp_fs=100.0, pdamp_fs=1000.0)


@pytest.mark.parametrize("kw,match", [
    (dict(timestep_fs=0.0), "timestep_fs"),
    (dict(temperature=0.0), "temperature"),
    (dict(temperature=-1.0), "temperature"),
    (dict(temperature=[300.0, 300.0]), "temperature"),
    (dict(pressure=float("nan")), "pressure"),
    (dict(tdamp_fs=0.0), "tdamp_fs"),
    (dict(pdamp_fs=-5.0), "pdamp_fs"),
    (dict(pdamp_fs=float("inf")), "pdamp_fs"),
    (dict(tchain=-1), "tchain"),
    (dict(tchain=9), "tchain"),
    (dict(pchain=9), "pchain"),
    (dict(pchain=1.5), "pchain"),
    (dict(tloop=0), "tloop"),
    (dict(ploop=0), "ploop"),
    (dict(masses=[1.0, 1.0, 0.0, 1.0]), "masses"),
    (dict(masses=[1.0, 1.0]), "masses"),
    (dict(velocities=torch.zeros(3, 3)), "velocities"),
])
def test_argument_checks_raise_before_cuda(kw, match):
    args = dict(masses=[1.0] * 4, timestep_fs=1.0, temperature=300.0, pressure=0.0, **_OK)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        GraphedNPT(None, _cpu_example(), args.pop("masses"), args.pop("timestep_fs"), args.pop("temperature"),
                   args.pop("pressure"), **args)


def test_example_checks_raise_before_cuda():
    run = lambda ex, n=4: GraphedNPT(None, ex, [1.0] * n, 1.0, 300.0, 0.0, **_OK)  # noqa: E731
    with pytest.raises(ValueError, match="periodic"):
        run(_cpu_example(pbc=torch.tensor([True, True, False])))
    with pytest.raises(ValueError, match="periodic"):
        run(_cpu_example(cell=None))
    with pytest.raises(ValueError, match="at least one atom"):
        run(_cpu_example(batch=torch.tensor([0, 0, 0, 0]), num_atoms=torch.tensor([4, 0]),
                         cell=5 * torch.eye(3).expand(2, 3, 3)))
    with pytest.raises(ValueError, match="num_atoms"):
        run(_cpu_example(batch=torch.tensor([0, 0, 1, 1]), num_atoms=torch.tensor([2, 1]),
                         cell=5 * torch.eye(3).expand(2, 3, 3)))
    with pytest.raises(ValueError, match="cell must be"):
        run(_cpu_example(cell=torch.eye(2)))
    with pytest.raises(ValueError, match="singular"):
        run(_cpu_example(cell=torch.zeros(3, 3)))
    with pytest.raises(RuntimeError, match="CUDA"):  # valid arguments: only then the device check
        run(_cpu_example())


def test_graphed_md_still_has_no_variable_cell():
    with pytest.raises(ValueError, match="no barostat"):
        md.GraphedMD(None, _cpu_example(), [1.0] * 4, 1.0, variable_cell=True)
