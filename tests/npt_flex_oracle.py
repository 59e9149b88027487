"""Float64 host restatement of the fully flexible MTK NPT step (``GraphedNPT(barostat="flexible")``; Martyna, Tobias &
Klein 1994, Martyna, Tuckerman, Tobias & Klein 1996, the splitting of Tuckerman et al. 2006) per frame of a batch, and
of the quantity it conserves, in the arithmetic order of the nqb_nptf kernels of csrc/nqb_npt.cu (DESIGN.md section
4.17).  The chain half-step and sinhc are tests/npt_oracle.py's.  Per-frame 3x3 matrices are row-major lists of 9
Python floats, the atoms torch tensors.  Units as md_oracle."""
import math

import torch

import md_oracle as mo
import npt_oracle as no

MAX_CHAIN = no.MAX_CHAIN
JACOBI_SWEEPS = 6  # NQB_NPTF_JACOBI_SWEEPS
NG = 6.0  # the barostat chain's degrees of freedom
STATE = 18 + 4 * MAX_CHAIN  # NQB_NPTF_STATE
LOG = 24  # NQB_NPTF_LOG_FIELDS
EYE = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]


def det3(c):
    return (c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6])
            + c[2] * (c[3] * c[7] - c[4] * c[6]))


def frob2(g):
    s = 0.0
    for x in g:
        s += x * x
    return s


def jacobi3(a):
    """Cyclic Jacobi (Golub & Van Loan's rotation) on the symmetric 3x3 ``a``: (eigenvalues [3], o [9]) with the
    eigenvectors in the columns of o.  An exactly zero off-diagonal entry takes no rotation."""
    a, o = list(a), list(EYE)
    for _ in range(JACOBI_SWEEPS):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            r = 3 - p - q
            apq = a[3 * p + q]
            if apq != 0.0:
                th = (a[3 * q + q] - a[3 * p + p]) / (2.0 * apq)
                t = (1.0 if th >= 0.0 else -1.0) / (abs(th) + math.hypot(1.0, th))
                c = 1.0 / math.sqrt(1.0 + t * t)
                s = t * c
                a[3 * p + p] = a[3 * p + p] - t * apq
                a[3 * q + q] = a[3 * q + q] + t * apq
                a[3 * p + q] = a[3 * q + p] = 0.0
                arp, arq = a[3 * r + p], a[3 * r + q]
                a[3 * r + p] = a[3 * p + r] = c * arp - s * arq
                a[3 * r + q] = a[3 * q + r] = s * arp + c * arq
                for i in range(3):
                    oip, oiq = o[3 * i + p], o[3 * i + q]
                    o[3 * i + p] = c * oip - s * oiq
                    o[3 * i + q] = s * oip + c * oiq
    return [a[0], a[4], a[8]], o


def sym_fn(o, f):
    """o diag(f) o^T, the upper triangle summed in index order and mirrored."""
    out = [0.0] * 9
    for i in range(3):
        for j in range(i, 3):
            e = 0.0
            for k in range(3):
                e = e + o[3 * i + k] * f[k] * o[3 * j + k]
            out[3 * i + j] = out[3 * j + i] = e
    return out


def coefs(g, Nf, dt):
    """(E_v, K, E_r, D) of the symmetric cell velocity g: E_v = e^{-(g + tr g / N_f) dt/2}, K = its integral over
    [0, dt/2], E_r = e^{g dt}, D = its integral over [0, dt]; also the eigenvector matrix o."""
    hdt = 0.5 * dt
    trg = g[0] + g[4] + g[8]
    lam, o = jacobi3(g)
    fev, fkf, fer, fdf = [], [], [], []
    for k in range(3):
        mu = lam[k] + trg / Nf
        am, b = mu * dt, lam[k] * dt
        fev.append(math.exp(-0.5 * am))
        fkf.append(hdt * math.exp(-0.25 * am) * no.sinhc(0.25 * am))
        fer.append(math.exp(b))
        fdf.append(dt * math.exp(0.5 * b) * no.sinhc(0.5 * b))
    return sym_fn(o, fev), sym_fn(o, fkf), sym_fn(o, fer), sym_fn(o, fdf), o


def cell_kick(g, kt, vr, PV, Nf, h, W):
    """v_g += h G_g / W_g, G_g = sym(Kt + vir) - P V I + (tr Kt / N_f) I (g updated in place)."""
    dg = (kt[0] + kt[4] + kt[8]) / Nf - PV
    for i in range(3):
        for j in range(i, 3):
            G = kt[3 * i + j] + 0.5 * (vr[3 * i + j] + vr[3 * j + i])
            if i == j:
                G = G + dg
            g[3 * i + j] = g[3 * i + j] + h * G / W
            g[3 * j + i] = g[3 * i + j]


class Params(no.Params):
    """The isotropic constants with W = W_g = (N_f + 3) kT tau_P^2 / 3 and Q'_1 = 6 kT tau_P^2."""

    def __init__(self, counts, C0, temperature, pressure, tau_t, tau_p, tchain, pchain, tloop=1, ploop=1):
        super().__init__(counts, C0, temperature, pressure, tau_t, tau_p, tchain, pchain, tloop, ploop)
        self.W = [w / 3.0 for w in self.W]
        for q in self.Qp:
            if q:
                q[0] = NG * q[0]


def kinetic(mass, vel, ptr):
    """Kt = sum m v (x) v per frame [F][9], from frame sums of {xx, yy, zz, yz, xz, xy} as the kick kernel forms
    them."""
    v = vel
    comps = [mo.frame_sum(mass * v[:, i] * v[:, j], ptr) for i, j in ((0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1))]
    out = []
    for f in range(len(ptr) - 1):
        xx, yy, zz, yz, xz, xy = (float(c[f]) for c in comps)
        out.append([xx, xy, xz, xy, yy, yz, xz, yz, zz])
    return out


class State:
    """pos, vel, forces [N, 3], mass [N], vir and cell [F, 3, 3] (torch) and per frame g (v_g), kt (Kt) [9] and the
    chains xi, vxi (M each), eta, veta (M' each) (Python floats and lists)."""

    def __init__(self, pos, vel, forces, mass, vir, prm: Params, cell=None):
        F = len(prm.kT)
        self.pos, self.vel, self.forces, self.mass = pos.clone(), vel.clone(), forces.clone(), mass.clone()
        self.vir = vir.clone().reshape(F, 3, 3).double().cpu()
        self.cell = (prm.C0 if cell is None else torch.as_tensor(cell)).clone().reshape(F, 3, 3).double().cpu()
        self.g = [[0.0] * 9 for _ in range(F)]
        self.kt = kinetic(mass, vel, prm.ptr)
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
        """[F, NQB_NPTF_STATE] in the layout of nqb.h."""
        pad = lambda xs: xs + [0.0] * (MAX_CHAIN - len(xs))  # noqa
        return torch.tensor([self.g[f] + self.kt[f] + pad(self.xi[f]) + pad(self.vxi[f]) + pad(self.eta[f])
                             + pad(self.veta[f]) for f in range(len(self.g))], dtype=torch.float64)


def _matvec(A, X):
    """Rows of X [n, 3] times the row-major 3x3 A: y_i = A_i0 x_0 + A_i1 x_1 + A_i2 x_2."""
    return torch.stack([A[3 * i] * X[:, 0] + A[3 * i + 1] * X[:, 1] + A[3 * i + 2] * X[:, 2] for i in range(3)], 1)


def pre(st: State, prm: Params, dt: float):
    """nqb_nptf_pre for every frame: returns the coefficients [(s, E_v, K, E_r, D)] and moves v_g, Kt, the chains and
    the cell."""
    out = []
    hdt = 0.5 * dt
    for f in range(len(prm.kT)):
        kT, W, Nf = prm.kT[f], prm.W[f], prm.Nf[f]
        vr = st.vir[f].reshape(-1).tolist()
        C = st.cell[f].reshape(-1).tolist()
        g = st.g[f]
        sb, _ = no.nhc_half(prm.ploop, hdt, NG, kT, prm.Qp[f], st.eta[f], st.veta[f], W * frob2(g))
        g = [x * sb for x in g]
        kt = st.kt[f]
        s, _ = no.nhc_half(prm.tloop, hdt, Nf, kT, prm.Q[f], st.xi[f], st.vxi[f], kt[0] + kt[4] + kt[8])
        kt = [x * (s * s) for x in kt]
        V = abs(det3(C))
        cell_kick(g, kt, vr, prm.P[f] * V, Nf, hdt, W)
        Ev, K, Er, D, _o = coefs(g, Nf, dt)
        nc = [Er[3 * i] * C[3 * r] + Er[3 * i + 1] * C[3 * r + 1] + Er[3 * i + 2] * C[3 * r + 2]
              for r in range(3) for i in range(3)]
        st.g[f], st.kt[f] = g, kt
        st.cell[f] = torch.tensor(nc, dtype=torch.float64).view(3, 3)
        out.append((s, Ev, K, Er, D))
    return out


def move(st: State, prm: Params, cf):
    m = st.mass.unsqueeze(1)
    for f, (s, Ev, K, Er, D) in enumerate(cf):
        a, b = prm.ptr[f], prm.ptr[f + 1]
        v1 = s * st.vel[a:b]
        v2 = _matvec(Ev, v1) + _matvec(K, st.forces[a:b] / m[a:b])
        st.vel[a:b] = v2
        st.pos[a:b] = _matvec(Er, st.pos[a:b]) + _matvec(D, v2)


def kick(st: State, prm: Params, cf, f_new):
    m = st.mass.unsqueeze(1)
    for f, (_s, Ev, K, _Er, _D) in enumerate(cf):
        a, b = prm.ptr[f], prm.ptr[f + 1]
        st.vel[a:b] = _matvec(Ev, st.vel[a:b]) + _matvec(K, f_new[a:b] / m[a:b])
    st.forces = f_new.clone()


def post(st: State, prm: Params, dt: float, vir_new):
    """nqb_nptf_post then nqb_nptf_scale for every frame."""
    hdt = 0.5 * dt
    kts = kinetic(st.mass, st.vel, prm.ptr)
    vir_new = torch.as_tensor(vir_new).reshape(-1, 3, 3).double().cpu()
    for f in range(len(prm.kT)):
        kT, W, Nf = prm.kT[f], prm.W[f], prm.Nf[f]
        vr = vir_new[f].reshape(-1).tolist()
        V = abs(det3(st.cell[f].reshape(-1).tolist()))
        g, kt = list(st.g[f]), kts[f]
        cell_kick(g, kt, vr, prm.P[f] * V, Nf, hdt, W)
        s, _ = no.nhc_half(prm.tloop, hdt, Nf, kT, prm.Q[f], st.xi[f], st.vxi[f], kt[0] + kt[4] + kt[8])
        kt = [x * (s * s) for x in kt]
        sb, _ = no.nhc_half(prm.ploop, hdt, NG, kT, prm.Qp[f], st.eta[f], st.veta[f], W * frob2(g))
        st.g[f], st.kt[f] = [x * sb for x in g], kt
        a, b = prm.ptr[f], prm.ptr[f + 1]
        st.vel[a:b] = s * st.vel[a:b]
    st.vir = vir_new.clone()


def step(st: State, prm: Params, dt: float, force_fn):
    """One flexible NPT step in place.  ``force_fn(pos, cell) -> (e_pot [F], forces [N, 3], virial [F, 3, 3])``."""
    cf = pre(st, prm, dt)
    move(st, prm, cf)
    e, f_new, vir = force_fn(st.pos, st.cell)
    kick(st, prm, cf, f_new)
    post(st, prm, dt, vir)
    st.e_pot = [float(x) for x in torch.as_tensor(e).reshape(-1)]
    return st


def volume(st: State):
    return [abs(det3(c.reshape(-1).tolist())) for c in st.cell]


def conserved(st: State, prm: Params):
    """H = E_pot + tr Kt/2 + W_g tr(v_g^2)/2 + P V + sum Q_k v_xi_k^2/2 + N_f kT xi_1 + kT sum_{k>=2} xi_k
    + sum Q'_k v_eta_k^2/2 + 6 kT eta_1 + kT sum_{k>=2} eta_k, per frame, in the order of nqb_nptf_log."""
    out = []
    for f, V in enumerate(volume(st)):
        kT, kt = prm.kT[f], st.kt[f]
        h = st.e_pot[f] + 0.5 * (kt[0] + kt[4] + kt[8]) + 0.5 * prm.W[f] * frob2(st.g[f]) + prm.P[f] * V
        for k in range(len(prm.Q[f])):
            h += 0.5 * prm.Q[f][k] * st.vxi[f][k] * st.vxi[f][k] + (prm.Nf[f] * kT if k == 0 else kT) * st.xi[f][k]
        for k in range(len(prm.Qp[f])):
            h += 0.5 * prm.Qp[f][k] * st.veta[f][k] * st.veta[f][k] + (NG * kT if k == 0 else kT) * st.eta[f][k]
        out.append(h)
    return out


def log_row(st: State, prm: Params):
    """[F, 24]: E_pot, E_kin, T, V, tr(P_int)/3, H, the cell [9] and P_int = (Kt + vir) / V [9]."""
    rows = []
    H = conserved(st, prm)
    for f, V in enumerate(volume(st)):
        kt = st.kt[f]
        K2 = kt[0] + kt[4] + kt[8]
        vr = st.vir[f].reshape(-1).tolist()
        rows.append([st.e_pot[f], 0.5 * K2, K2 / prm.NfkB[f], V, (K2 + (vr[0] + vr[4] + vr[8])) / (3.0 * V), H[f]]
                    + st.cell[f].reshape(-1).tolist() + [(kt[k] + vr[k]) / V for k in range(9)])
    return torch.tensor(rows, dtype=torch.float64)


def reverse(st: State):
    """Negate every velocity: v, v_g, v_xi and v_eta."""
    st.vel = -st.vel
    st.g = [[-x for x in g] for g in st.g]
    st.vxi = [[-v for v in r] for r in st.vxi]
    st.veta = [[-v for v in r] for r in st.veta]
