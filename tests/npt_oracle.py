"""Float64 host restatement of the isotropic MTK NPT step with Nose-Hoover chains (Martyna, Tobias & Klein 1994; the
splitting of Tuckerman et al. 2006; the chain half-step of Martyna et al. 1996) per frame of a batch, and of the
quantity it conserves, in the arithmetic order of csrc/nqb_npt.cu (DESIGN.md section 4.16).  Per-frame scalars are
Python floats, the atoms torch tensors.  Units as md_oracle: Angstrom, eV, amu, time in Angstrom sqrt(amu / eV)."""
import math

import torch

import md_oracle as mo

SINHC_TAYLOR = 0.1  # NQB_NPT_SINHC_TAYLOR
MAX_CHAIN = 8  # NQB_NPT_MAX_CHAIN


def sinhc(x: float) -> float:
    """sinh(x) / x; the Taylor branch below SINHC_TAYLOR."""
    if abs(x) < SINHC_TAYLOR:
        x2 = x * x
        return 1.0 + x2 * (1.0 / 6.0 + x2 * (1.0 / 120.0 + x2 * (1.0 / 5040.0 + x2 * (1.0 / 362880.0))))
    return math.sinh(x) / x


def _chain_force(k, K2, Nf, kT, Q, v):
    return (K2 - Nf * kT) / Q[0] if k == 0 else (Q[k - 1] * v[k - 1] * v[k - 1] - kT) / Q[k]


def nhc_half(nloop, h, Nf, kT, Q, x, v, K2):
    """One chain half-step of length h in ``nloop`` sub-steps on (x, v, Q) (lists, updated in place; len(Q) members)
    coupled to K2 with Nf degrees of freedom.  Returns (the product of the scales, K2 scaled by its square)."""
    M = len(Q)
    if M == 0:
        return 1.0, K2
    d = h / nloop
    d2, d4 = 0.5 * d, 0.25 * d
    s = 1.0
    for _ in range(nloop):
        v[M - 1] = v[M - 1] + d2 * _chain_force(M - 1, K2, Nf, kT, Q, v)
        for k in range(M - 2, -1, -1):
            e = math.exp(-d4 * v[k + 1])
            v[k] = (v[k] * e + d2 * _chain_force(k, K2, Nf, kT, Q, v)) * e
        sc = math.exp(-d * v[0])
        s = s * sc
        K2 = K2 * (sc * sc)
        for k in range(M):
            x[k] = x[k] + d * v[k]
        for k in range(M - 1):
            e = math.exp(-d4 * v[k + 1])
            v[k] = (v[k] * e + d2 * _chain_force(k, K2, Nf, kT, Q, v)) * e
        v[M - 1] = v[M - 1] + d2 * _chain_force(M - 1, K2, Nf, kT, Q, v)
    return s, K2


class Params:
    """Per-frame constants: kT, P (eV / Angstrom^3), N_f = 3 N, V0 = |det C0|, C0 [F, 3, 3] and the masses
    Q_1 = N_f kT tau_T^2, Q_k = kT tau_T^2, W = (N_f + 3) kT tau_P^2, Q'_k = kT tau_P^2 (tau in time units)."""

    def __init__(self, counts, C0, temperature, pressure, tau_t, tau_p, tchain, pchain, tloop=1, ploop=1):
        F = len(counts)
        exp = lambda x: [float(v) for v in torch.as_tensor(x, dtype=torch.float64).reshape(-1).expand(F)]  # noqa
        T, P, tt, tp = exp(temperature), exp(pressure), exp(tau_t), exp(tau_p)
        self.kT = [mo.KB * t for t in T]
        self.P = P
        self.Nf = [3.0 * n for n in counts]
        self.NfkB = [3.0 * n * mo.KB for n in counts]
        self.C0 = torch.as_tensor(C0, dtype=torch.float64).reshape(F, 3, 3).clone()
        self.V0 = [abs(float(torch.linalg.det(c))) for c in self.C0]
        self.W = [(self.Nf[f] + 3.0) * self.kT[f] * tp[f] * tp[f] for f in range(F)]
        self.Q = [[(self.Nf[f] if k == 0 else 1.0) * self.kT[f] * tt[f] * tt[f] for k in range(tchain)]
                  for f in range(F)]
        self.Qp = [[self.kT[f] * tp[f] * tp[f] for _ in range(pchain)] for f in range(F)]
        self.tloop, self.ploop = tloop, ploop
        self.ptr = [0] + torch.tensor(counts).cumsum(0).tolist()

    def table(self):
        """[F, NQB_NPT_PARAMS] in the layout of nqb.h."""
        rows = []
        for f in range(len(self.kT)):
            Q = self.Q[f] + [1.0] * (MAX_CHAIN - len(self.Q[f]))
            Qp = self.Qp[f] + [1.0] * (MAX_CHAIN - len(self.Qp[f]))
            rows.append([self.kT[f], self.P[f], self.W[f], self.Nf[f], self.V0[f], self.NfkB[f]] + Q + Qp)
        return torch.tensor(rows, dtype=torch.float64)


class State:
    """pos, vel, forces [N, 3], mass [N], vir [F, 3, 3], cell [F, 3, 3] (torch) and per frame eps, veps, K2 and the
    chains xi, vxi (M each), eta, veta (M' each) (Python floats and lists)."""

    def __init__(self, pos, vel, forces, mass, vir, prm: Params):
        F = len(prm.kT)
        self.pos, self.vel, self.forces, self.mass = pos.clone(), vel.clone(), forces.clone(), mass.clone()
        self.vir = vir.clone().reshape(F, 3, 3)
        self.cell = prm.C0.clone()
        self.eps, self.veps = [0.0] * F, [0.0] * F
        self.K2 = [float(k) for k in mo.frame_sum(mass * (vel ** 2).sum(1), prm.ptr)]
        self.xi = [[0.0] * len(q) for q in prm.Q]
        self.vxi = [[0.0] * len(q) for q in prm.Q]
        self.eta = [[0.0] * len(q) for q in prm.Qp]
        self.veta = [[0.0] * len(q) for q in prm.Qp]
        self.e_pot = [0.0] * F

    def clone(self):
        c = object.__new__(State)
        for k, v in self.__dict__.items():
            c.__dict__[k] = v.clone() if torch.is_tensor(v) else [list(x) if isinstance(x, list) else x for x in v]
        return c

    def rows(self):
        """[F, NQB_NPT_STATE] in the layout of nqb.h."""
        pad = lambda xs: xs + [0.0] * (MAX_CHAIN - len(xs))  # noqa
        return torch.tensor([[self.eps[f], self.veps[f], self.K2[f]] + pad(self.xi[f]) + pad(self.vxi[f])
                             + pad(self.eta[f]) + pad(self.veta[f]) for f in range(len(self.eps))],
                            dtype=torch.float64)


def _coefs(veps, alpha, dt):
    a, b = alpha * veps * dt, veps * dt
    return (math.exp(-0.5 * a), 0.5 * dt * math.exp(-0.25 * a) * sinhc(0.25 * a), math.exp(b),
            dt * math.exp(0.5 * b) * sinhc(0.5 * b))


def pre(st: State, prm: Params, dt: float):
    """nqb_npt_pre for every frame: returns the coefficients [(s, ev, kf, er, df)] and moves eps, veps, K2, chains and
    the cell."""
    out = []
    hdt = 0.5 * dt
    for f in range(len(prm.kT)):
        kT, W, Nf = prm.kT[f], prm.W[f], prm.Nf[f]
        alpha = 1.0 + 3.0 / Nf
        v = st.vir[f].reshape(-1).tolist()
        trv = v[0] + v[4] + v[8]
        veps = st.veps[f]
        sb, _ = nhc_half(prm.ploop, hdt, 1.0, kT, prm.Qp[f], st.eta[f], st.veta[f], W * veps * veps)
        veps = veps * sb
        s, K2 = nhc_half(prm.tloop, hdt, Nf, kT, prm.Q[f], st.xi[f], st.vxi[f], st.K2[f])
        V = prm.V0[f] * math.exp(3.0 * st.eps[f])
        veps = veps + hdt * (alpha * K2 + trv - 3.0 * prm.P[f] * V) / W
        ev, kf, er, df = _coefs(veps, alpha, dt)
        st.eps[f] = st.eps[f] + dt * veps
        st.veps[f], st.K2[f] = veps, K2
        st.cell[f] = prm.C0[f] * math.exp(st.eps[f])
        out.append((s, ev, kf, er, df))
    return out


def move(st: State, prm: Params, coefs):
    m = st.mass.unsqueeze(1)
    for f, (s, ev, kf, er, df) in enumerate(coefs):
        a, b = prm.ptr[f], prm.ptr[f + 1]
        v1 = s * st.vel[a:b]
        v2 = v1 * ev + kf * (st.forces[a:b] / m[a:b])
        st.vel[a:b] = v2
        st.pos[a:b] = st.pos[a:b] * er + df * v2


def kick(st: State, prm: Params, coefs, f_new):
    m = st.mass.unsqueeze(1)
    for f, (_s, ev, kf, _er, _df) in enumerate(coefs):
        a, b = prm.ptr[f], prm.ptr[f + 1]
        st.vel[a:b] = st.vel[a:b] * ev + kf * (f_new[a:b] / m[a:b])
    st.forces = f_new.clone()


def post(st: State, prm: Params, dt: float, vir_new):
    """nqb_npt_post then nqb_npt_scale for every frame."""
    hdt = 0.5 * dt
    K2s = mo.frame_sum(st.mass * (st.vel ** 2).sum(1), prm.ptr)
    vir_new = vir_new.reshape(-1, 3, 3)
    for f in range(len(prm.kT)):
        kT, W, Nf = prm.kT[f], prm.W[f], prm.Nf[f]
        alpha = 1.0 + 3.0 / Nf
        v = vir_new[f].reshape(-1).tolist()
        trv = v[0] + v[4] + v[8]
        V = prm.V0[f] * math.exp(3.0 * st.eps[f])
        veps = st.veps[f] + hdt * (alpha * float(K2s[f]) + trv - 3.0 * prm.P[f] * V) / W
        s, K2 = nhc_half(prm.tloop, hdt, Nf, kT, prm.Q[f], st.xi[f], st.vxi[f], float(K2s[f]))
        sb, _ = nhc_half(prm.ploop, hdt, 1.0, kT, prm.Qp[f], st.eta[f], st.veta[f], W * veps * veps)
        st.veps[f], st.K2[f] = veps * sb, K2
        a, b = prm.ptr[f], prm.ptr[f + 1]
        st.vel[a:b] = s * st.vel[a:b]
    st.vir = vir_new.clone()


def step(st: State, prm: Params, dt: float, force_fn):
    """One NPT step in place.  ``force_fn(pos, cell) -> (e_pot [F], forces [N, 3], virial [F, 3, 3])``."""
    coefs = pre(st, prm, dt)
    move(st, prm, coefs)
    e, f_new, vir = force_fn(st.pos, st.cell)
    kick(st, prm, coefs, f_new)
    post(st, prm, dt, vir)
    st.e_pot = [float(x) for x in torch.as_tensor(e).reshape(-1)]
    return st


def volume(st: State, prm: Params):
    return [prm.V0[f] * math.exp(3.0 * st.eps[f]) for f in range(len(prm.kT))]


def conserved(st: State, prm: Params):
    """H = E_pot + K2/2 + W v_eps^2/2 + P V + sum Q_k v_xi_k^2/2 + N_f kT xi_1 + kT sum_{k>=2} xi_k
    + sum Q'_k v_eta_k^2/2 + kT sum eta_k, per frame, in the order of nqb_npt_log."""
    out = []
    for f, V in enumerate(volume(st, prm)):
        kT = prm.kT[f]
        h = st.e_pot[f] + 0.5 * st.K2[f] + 0.5 * prm.W[f] * st.veps[f] * st.veps[f] + prm.P[f] * V
        for k in range(len(prm.Q[f])):
            h += 0.5 * prm.Q[f][k] * st.vxi[f][k] * st.vxi[f][k] + (prm.Nf[f] * kT if k == 0 else kT) * st.xi[f][k]
        for k in range(len(prm.Qp[f])):
            h += 0.5 * prm.Qp[f][k] * st.veta[f][k] * st.veta[f][k] + kT * st.eta[f][k]
        out.append(h)
    return out


def log_row(st: State, prm: Params):
    """[F, 6]: E_pot, E_kin, T, V, the instantaneous pressure (K2 + tr vir) / (3 V) and H."""
    rows = []
    H = conserved(st, prm)
    for f, V in enumerate(volume(st, prm)):
        K2 = st.K2[f]
        trv = float(st.vir[f].diagonal().sum())
        rows.append([st.e_pot[f], 0.5 * K2, K2 / prm.NfkB[f], V, (K2 + trv) / (3.0 * V), H[f]])
    return torch.tensor(rows, dtype=torch.float64)


def reverse(st: State):
    """Negate every velocity: v, v_eps, v_xi and v_eta."""
    st.vel = -st.vel
    st.veps = [-v for v in st.veps]
    st.vxi = [[-v for v in r] for r in st.vxi]
    st.veta = [[-v for v in r] for r in st.veta]
