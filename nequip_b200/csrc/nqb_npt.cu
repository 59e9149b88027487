// Constant-pressure MD on the device: isotropic MTK (Martyna, Tobias & Klein, J. Chem. Phys. 101, 4177 (1994)) with
// Nose-Hoover chains on the particles and on the barostat (Martyna, Tuckerman, Tobias & Klein, Mol. Phys. 87, 1117
// (1996)), in the measure-preserving splitting of Tuckerman et al., J. Phys. A 39, 5629 (2006), per frame f of a
// batch, in float64, sm_90a.  One step of nequip_b200/npt.py (GraphedNPT) is
//   nqb_npt_pre -> nqb_npt_move -> nqb_nl_frames_set_cells -> neighbour list + model (stress) -> nqb_npt_kick
//   -> nqb_npt_post -> nqb_npt_scale -> nqb_npt_log
// captured as one CUDA graph (DESIGN.md section 4.16).  The atoms of frame f are [atom_ptr[f], atom_ptr[f+1]); the
// atom kernels run (nblk, F) CTAs of kNptThreads threads as the nqb_md kernels do, and the one sum over atoms (K2 =
// sum m v^2) is a per-CTA partial in a fixed order that nqb_npt_post adds in index order: no floating-point atomics,
// so a launch shape gives results that depend only on its inputs.
//
// The per-frame kernels update a copy of the frame's state row in a workspace and commit it only when every result
// is finite; otherwise the frame keeps its state, err[f] is set and the atom kernels leave its atoms alone, so a
// non-finite barostat or bath never moves positions or the cell.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/nqb.h"

extern "C" int nqb_set_error(const char* msg);
extern "C" void nqb_count_launch(void);

namespace {

constexpr int kNptThreads = 256;
constexpr int kS = NQB_NPT_STATE, kP = NQB_NPT_PARAMS, kC = NQB_NPT_COEF, kM = NQB_NPT_MAX_CHAIN;
// offsets in a state row and a parameter row (nqb.h)
constexpr int kEps = 0, kVeps = 1, kK2 = 2, kXi = 3, kVxi = 3 + kM, kEta = 3 + 2 * kM, kVeta = 3 + 3 * kM;
constexpr int kKT = 0, kPres = 1, kW = 2, kNf = 3, kV0 = 4, kNfkB = 5, kQ = 6, kQp = 6 + kM;

// sinh(x) / x; the Taylor branch below NQB_NPT_SINHC_TAYLOR (error < 3e-18 relative)
__device__ __forceinline__ double sinhc(double x) {
  if (fabs(x) < NQB_NPT_SINHC_TAYLOR) {
    const double x2 = x * x;
    return 1.0 + x2 * (1.0 / 6.0 + x2 * (1.0 / 120.0 + x2 * (1.0 / 5040.0 + x2 * (1.0 / 362880.0))));
  }
  return sinh(x) / x;
}

// the force on chain member k: G_0 = (K2 - Nf kT) / Q_0, G_k = (Q_{k-1} v_{k-1}^2 - kT) / Q_k
__device__ __forceinline__ double chain_force(int k, double K2, double Nf, double kT, const double* Q,
                                              const double* v) {
  return k == 0 ? (K2 - Nf * kT) / Q[0] : (Q[k - 1] * v[k - 1] * v[k - 1] - kT) / Q[k];
}

// One Nose-Hoover chain half-step of length h in nloop sub-steps d = h / nloop on the chain (x, v, Q) of M members
// coupled to K2 (sum m v^2, or W v_eps^2) with Nf degrees of freedom: per sub-step, kick inward from the chain end
// by d/2 (v_k damped by exp(-d v_{k+1} / 4) on each side of its kick), scale by exp(-d v_0) (K2 by its square),
// x_k += d v_k, kick outward.  Returns the product of the scales; M = 0 returns 1.  x and v are global memory (a
// workspace row), so the chain needs no stack.
__device__ double nhc_half(int M, int nloop, double h, double Nf, double kT, const double* Q, double* x, double* v,
                           double& K2) {
  if (M == 0) return 1.0;
  const double d = h / nloop, d2 = 0.5 * d, d4 = 0.25 * d;
  double s = 1.0;
  for (int l = 0; l < nloop; ++l) {
    v[M - 1] = v[M - 1] + d2 * chain_force(M - 1, K2, Nf, kT, Q, v);
    for (int k = M - 2; k >= 0; --k) {
      const double e = exp(-d4 * v[k + 1]);
      v[k] = (v[k] * e + d2 * chain_force(k, K2, Nf, kT, Q, v)) * e;
    }
    const double sc = exp(-d * v[0]);
    s = s * sc;
    K2 = K2 * (sc * sc);
    for (int k = 0; k < M; ++k) x[k] = x[k] + d * v[k];
    for (int k = 0; k < M - 1; ++k) {
      const double e = exp(-d4 * v[k + 1]);
      v[k] = (v[k] * e + d2 * chain_force(k, K2, Nf, kT, Q, v)) * e;
    }
    v[M - 1] = v[M - 1] + d2 * chain_force(M - 1, K2, Nf, kT, Q, v);
  }
  return s;
}

__device__ __forceinline__ bool row_finite(const double* w) {
  bool ok = true;
  for (int k = 0; k < kS; ++k) ok = ok && isfinite(w[k]);
  return ok;
}

__device__ __forceinline__ void frozen_coef(double* c) {
  c[0] = 1.0;  // s
  c[1] = 1.0;  // e^{-alpha v_eps dt/2}
  c[2] = 0.0;  // kick factor
  c[3] = 1.0;  // e^{v_eps dt}
  c[4] = 0.0;  // drift factor
  c[5] = 0.0;  // inactive
  c[6] = 1.0;  // final scale
}

// One thread per frame: NHC_baro(dt/2), NHC_part(dt/2), v_eps += dt/2 G_eps / W, the atoms' coefficients and the new
// eps and cell.
__global__ void k_npt_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* __restrict__ prm,
                          const double* __restrict__ C0, const double* __restrict__ vir, double* __restrict__ st,
                          double* __restrict__ cell, double* __restrict__ coef, int32_t* __restrict__ err,
                          double* __restrict__ wk) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* c = coef + kC * (int64_t)f;
  if (err[f]) {
    frozen_coef(c);
    return;
  }
  const double* p = prm + kP * (int64_t)f;
  double* s0 = st + kS * (int64_t)f;
  double* w = wk + kS * (int64_t)f;
  for (int k = 0; k < kS; ++k) w[k] = s0[k];
  const double kT = p[kKT], P = p[kPres], W = p[kW], Nf = p[kNf], hdt = 0.5 * dt;
  const double alpha = 1.0 + 3.0 / Nf;
  const double* vr = vir + 9 * (int64_t)f;
  const double trv = vr[0] + vr[4] + vr[8];
  double veps = w[kVeps], K2 = w[kK2];
  const double eps = w[kEps];
  double Kb = W * veps * veps;
  const double sb = nhc_half(Mp, ploop, hdt, 1.0, kT, p + kQp, w + kEta, w + kVeta, Kb);
  veps = veps * sb;
  const double s = nhc_half(M, tloop, hdt, Nf, kT, p + kQ, w + kXi, w + kVxi, K2);
  const double V = p[kV0] * exp(3.0 * eps);
  veps = veps + hdt * (alpha * K2 + trv - 3.0 * P * V) / W;
  const double a = alpha * veps * dt, b = veps * dt;
  const double ev = exp(-0.5 * a);
  const double kf = hdt * exp(-0.25 * a) * sinhc(0.25 * a);
  const double er = exp(b);
  const double df = dt * exp(0.5 * b) * sinhc(0.5 * b);
  const double eps_new = eps + dt * veps;
  const double g = exp(eps_new);
  w[kEps] = eps_new;
  w[kVeps] = veps;
  w[kK2] = K2;
  double nc[9];
  bool ok = row_finite(w) && isfinite(s) && isfinite(ev) && isfinite(kf) && isfinite(er) && isfinite(df);
  for (int k = 0; k < 9; ++k) {
    nc[k] = C0[9 * (int64_t)f + k] * g;
    ok = ok && isfinite(nc[k]);
  }
  if (!ok) {
    err[f] = 1;
    frozen_coef(c);
    return;
  }
  for (int k = 0; k < kS; ++k) s0[k] = w[k];
  for (int k = 0; k < 9; ++k) cell[9 * (int64_t)f + k] = nc[k];
  c[0] = s;
  c[1] = ev;
  c[2] = kf;
  c[3] = er;
  c[4] = df;
  c[5] = 1.0;
  c[6] = 1.0;
}

// the atoms of active frames: v <- s v;  v <- v ev + kf F/m;  r <- r er + df v
__global__ void __launch_bounds__(kNptThreads)
k_npt_move(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ forces,
           const double* __restrict__ coef, double* __restrict__ pos, double* __restrict__ vel) {
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kC * (int64_t)f;
  if (c[5] == 0.0) return;
  const double s = c[0], ev = c[1], kf = c[2], er = c[3], df = c[4];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads) {
    const double m = mass[i];
    for (int d = 0; d < 3; ++d) {
      const double v1 = s * vel[3 * i + d];
      const double v2 = v1 * ev + kf * (forces[3 * i + d] / m);
      vel[3 * i + d] = v2;
      pos[3 * i + d] = pos[3 * i + d] * er + df * v2;
    }
  }
}

__device__ __forceinline__ double cta_sum(double v, double* smem) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kNptThreads / 32; ++w) s += smem[w];
  __syncthreads();
  return s;
}

// the atoms of active frames: v <- v ev + kf F_new/m;  forces <- F_new;  part[f, b] = sum m v^2 of the CTA (0 for an
// inactive frame)
__global__ void __launch_bounds__(kNptThreads)
k_npt_kick(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ f_new,
           const double* __restrict__ coef, double* __restrict__ vel, double* __restrict__ forces,
           double* __restrict__ part) {
  __shared__ double smem[kNptThreads / 32];
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kC * (int64_t)f;
  const bool active = c[5] != 0.0;
  const double ev = c[1], kf = c[2];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  double acc = 0.0;
  if (active)
    for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads) {
      const double m = mass[i];
      double v[3];
      for (int d = 0; d < 3; ++d) {
        const double fd = f_new[3 * i + d];
        v[d] = vel[3 * i + d] * ev + kf * (fd / m);
        vel[3 * i + d] = v[d];
        forces[3 * i + d] = fd;
      }
      acc += m * (v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    }
  acc = cta_sum(acc, smem);
  if (threadIdx.x == 0) part[(int64_t)f * nblk + blockIdx.x] = acc;
}

// One thread per frame (frames with err set are skipped): K2 = sum of part in index order, v_eps += dt/2 G_eps / W
// with the new virial, NHC_part(dt/2), NHC_baro(dt/2); stores K2 and the virial, coef[6] = the particles' scale.
__global__ void k_npt_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt,
                           const double* __restrict__ prm, const double* __restrict__ part,
                           const double* __restrict__ vir_new, double* __restrict__ st, double* __restrict__ vir,
                           double* __restrict__ coef, int32_t* __restrict__ err, double* __restrict__ wk) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* c = coef + kC * (int64_t)f;
  if (err[f]) {
    c[6] = 1.0;
    return;
  }
  const double* p = prm + kP * (int64_t)f;
  double* s0 = st + kS * (int64_t)f;
  double* w = wk + kS * (int64_t)f;
  for (int k = 0; k < kS; ++k) w[k] = s0[k];
  double K2 = 0.0;
  for (int b = 0; b < nblk; ++b) K2 += part[(int64_t)f * nblk + b];
  const double kT = p[kKT], P = p[kPres], W = p[kW], Nf = p[kNf], hdt = 0.5 * dt;
  const double alpha = 1.0 + 3.0 / Nf;
  const double* vr = vir_new + 9 * (int64_t)f;
  const double trv = vr[0] + vr[4] + vr[8];
  const double V = p[kV0] * exp(3.0 * w[kEps]);
  double veps = w[kVeps] + hdt * (alpha * K2 + trv - 3.0 * P * V) / W;
  const double s = nhc_half(M, tloop, hdt, Nf, kT, p + kQ, w + kXi, w + kVxi, K2);
  double Kb = W * veps * veps;
  const double sb = nhc_half(Mp, ploop, hdt, 1.0, kT, p + kQp, w + kEta, w + kVeta, Kb);
  veps = veps * sb;
  w[kVeps] = veps;
  w[kK2] = K2;
  bool ok = row_finite(w) && isfinite(s);
  for (int k = 0; k < 9; ++k) ok = ok && isfinite(vr[k]);
  if (!ok) {
    err[f] = 1;
    c[6] = 1.0;
    return;
  }
  for (int k = 0; k < kS; ++k) s0[k] = w[k];
  for (int k = 0; k < 9; ++k) vir[9 * (int64_t)f + k] = vr[k];
  c[6] = s;
}

// the atoms of active frames: v <- coef[6] v
__global__ void __launch_bounds__(kNptThreads)
k_npt_scale(const int64_t* __restrict__ atom_ptr, const double* __restrict__ coef, double* __restrict__ vel) {
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kC * (int64_t)f;
  if (c[5] == 0.0) return;
  const double s = c[6];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads)
    for (int d = 0; d < 3; ++d) vel[3 * i + d] = s * vel[3 * i + d];
}

// One CTA.  Row step % rows of the log, per frame: E_pot, E_kin, T, V, the instantaneous pressure, H; the sticky flags
// as nqb_md_log writes them; then step += 1.
__global__ void __launch_bounds__(kNptThreads)
k_npt_log(int F, int M, int Mp, const double* __restrict__ e_pot, const double* __restrict__ prm,
          const double* __restrict__ st, const double* __restrict__ vir, const int64_t* __restrict__ num_edges,
          const int32_t* __restrict__ overflow, const int32_t* __restrict__ sorted, int64_t rows, int64_t* step,
          double* __restrict__ log, int64_t* __restrict__ flags) {
  const int64_t s = *step;
  double* row = log + (s % rows) * (int64_t)F * NQB_NPT_LOG_FIELDS;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const double* p = prm + kP * (int64_t)f;
    const double* w = st + kS * (int64_t)f;
    const double* vr = vir + 9 * (int64_t)f;
    const double kT = p[kKT], K2 = w[kK2], veps = w[kVeps];
    const double V = p[kV0] * exp(3.0 * w[kEps]);
    const double ep = e_pot[f], ke = 0.5 * K2;
    double h = ep + ke + 0.5 * p[kW] * veps * veps + p[kPres] * V;
    for (int k = 0; k < M; ++k)
      h += 0.5 * p[kQ + k] * w[kVxi + k] * w[kVxi + k] + (k == 0 ? p[kNf] * kT : kT) * w[kXi + k];
    for (int k = 0; k < Mp; ++k) h += 0.5 * p[kQp + k] * w[kVeta + k] * w[kVeta + k] + kT * w[kEta + k];
    double* r = row + (int64_t)f * NQB_NPT_LOG_FIELDS;
    r[0] = ep;
    r[1] = ke;
    r[2] = K2 / p[kNfkB];
    r[3] = V;
    r[4] = (K2 + (vr[0] + vr[4] + vr[8])) / (3.0 * V);
    r[5] = h;
  }
  __syncthreads();  // every thread has read *step
  if (threadIdx.x == 0) {
    if (*overflow != 0) {
      flags[0] = 1;
      if (flags[2] < 0) flags[2] = s;
    }
    if (*sorted != 1) flags[1] = 1;
    if (*num_edges > flags[3]) flags[3] = *num_edges;
    *step = s + 1;
  }
}

// ---- the fully flexible cell (DESIGN.md section 4.17) -----------------------------------------------------------
// One step of GraphedNPT(barostat="flexible") is
//   nqb_nptf_pre -> nqb_nptf_move -> nqb_nl_frames_set_cells -> list + model (stress) -> nqb_nptf_kick -> nqb_nptf_post
//   -> nqb_nptf_scale -> nqb_nptf_log
// with a symmetric cell velocity v_g [3x3] in place of v_eps, the kinetic tensor Kt = sum m v (x) v in place of K2 and
// the cell itself as state.  The parameter rows are the isotropic ones with W = W_g and Q' of the n_g = 6 barostat
// degrees of freedom.
constexpr int kFS = NQB_NPTF_STATE, kFC = NQB_NPTF_COEF;
// offsets in a flexible state row (nqb.h)
constexpr int kFG = 0, kFKt = 9, kFXi = 18, kFVxi = 18 + kM, kFEta = 18 + 2 * kM, kFVeta = 18 + 3 * kM;
// offsets in a flexible coefficient row: s, active, final scale, then the symmetric 3x3 E_v, K, E_r, D (row-major)
constexpr int kFEv = 3, kFK = 12, kFEr = 21, kFD = 30;
constexpr double kNg = 6.0;  // the barostat's degrees of freedom: the independent components of a symmetric v_g

__device__ __forceinline__ double det3(const double* c) {
  return c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6]) + c[2] * (c[3] * c[7] - c[4] * c[6]);
}

// sum of the squares of the 9 entries, in index order: tr(g^2) for a symmetric g
__device__ __forceinline__ double frob2(const double (&g)[9]) {
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < 9; ++k) s += g[k] * g[k];
  return s;
}

// v_g += h G_g / W with G_g = sym(Kt + vir) - P V I + (tr Kt / N_f) I, written to both triangles (g stays symmetric)
__device__ __forceinline__ void cell_kick(double (&g)[9], const double (&kt)[9], const double* vr, double PV, double Nf,
                                          double h, double W) {
  const double dg = (kt[0] + kt[4] + kt[8]) / Nf - PV;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) {
      double G = kt[3 * i + j] + 0.5 * (vr[3 * i + j] + vr[3 * j + i]);
      if (i == j) G = G + dg;
      g[3 * i + j] = g[3 * i + j] + h * G / W;
      g[3 * j + i] = g[3 * i + j];
    }
}

// Cyclic Jacobi on the symmetric a (row-major; on return its diagonal holds the eigenvalues) with the eigenvectors
// accumulated in the columns of o (o a_in o^T = diag): NQB_NPTF_JACOBI_SWEEPS sweeps over the pairs (0,1), (0,2), (1,2)
// with the rotation of Golub & Van Loan (Algorithm 8.5.1), which is backward stable, so functions of a nearly
// isotropic v_g stay accurate.  An off-diagonal entry that is exactly 0 takes no rotation: a diagonal a gives o = I.
// Fully unrolled: a and o live in registers.
__device__ __forceinline__ void jacobi3(double (&a)[9], double (&o)[9]) {
#pragma unroll
  for (int k = 0; k < 9; ++k) o[k] = (k % 4 == 0) ? 1.0 : 0.0;
#pragma unroll
  for (int sw = 0; sw < NQB_NPTF_JACOBI_SWEEPS; ++sw)
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2, r = 3 - p - q;
      const double apq = a[3 * p + q];
      if (apq != 0.0) {
        const double th = (a[3 * q + q] - a[3 * p + p]) / (2.0 * apq);
        const double t = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + hypot(1.0, th));
        const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
        a[3 * p + p] = a[3 * p + p] - t * apq;
        a[3 * q + q] = a[3 * q + q] + t * apq;
        a[3 * p + q] = 0.0;
        a[3 * q + p] = 0.0;
        const double arp = a[3 * r + p], arq = a[3 * r + q];
        a[3 * r + p] = c * arp - s * arq;
        a[3 * p + r] = a[3 * r + p];
        a[3 * r + q] = s * arp + c * arq;
        a[3 * q + r] = a[3 * r + q];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const double oip = o[3 * i + p], oiq = o[3 * i + q];
          o[3 * i + p] = c * oip - s * oiq;
          o[3 * i + q] = s * oip + c * oiq;
        }
      }
    }
}

// out = o diag(f) o^T, the upper triangle summed over k in index order and mirrored (exactly symmetric); returns
// whether every entry is finite
__device__ __forceinline__ bool sym_fn(const double (&o)[9], const double (&f)[3], double* out) {
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = i; j < 3; ++j) {
      double e = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) e += o[3 * i + k] * f[k] * o[3 * j + k];
      out[3 * i + j] = e;
      out[3 * j + i] = e;
      ok = ok && isfinite(e);
    }
  return ok;
}

__device__ __forceinline__ void frozen_coef_flex(double* c) {
  c[0] = 1.0;  // s
  c[1] = 0.0;  // inactive
  c[2] = 1.0;  // final scale
  for (int k = 0; k < 9; ++k) {
    const double one = (k % 4 == 0) ? 1.0 : 0.0;
    c[kFEv + k] = one;
    c[kFK + k] = 0.0;
    c[kFEr + k] = one;
    c[kFD + k] = 0.0;
  }
}

__device__ __forceinline__ bool flex_row_finite(const double* w) {
  bool ok = true;
  for (int k = 0; k < kFS; ++k) ok = ok && isfinite(w[k]);
  return ok;
}

// One thread per frame: NHC_baro(dt/2) (scales v_g), NHC_part(dt/2) (Kt *= s^2), v_g += dt/2 G_g / W_g, v_g = O
// diag(lambda) O^T by Jacobi, the atoms' matrices E_v, K, E_r, D and the new cell C <- C E_r (each lattice vector a,
// a row of C, becomes E_r a).
__global__ void k_nptf_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* __restrict__ prm,
                           const double* __restrict__ vir, double* __restrict__ st, double* __restrict__ cell,
                           double* __restrict__ coef, int32_t* __restrict__ err, double* __restrict__ wk) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* c = coef + kFC * (int64_t)f;
  if (err[f]) {
    frozen_coef_flex(c);
    return;
  }
  const double* p = prm + kP * (int64_t)f;
  double* s0 = st + kFS * (int64_t)f;
  double* w = wk + kFS * (int64_t)f;
  double* C = cell + 9 * (int64_t)f;
  for (int k = 0; k < kFS; ++k) w[k] = s0[k];
  const double kT = p[kKT], P = p[kPres], W = p[kW], Nf = p[kNf], hdt = 0.5 * dt;
  const double* vr = vir + 9 * (int64_t)f;
  double g[9], kt[9], C1[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    g[k] = w[kFG + k];
    C1[k] = C[k];
  }
  double Kb = W * frob2(g);
  const double sb = nhc_half(Mp, ploop, hdt, kNg, kT, p + kQp, w + kFEta, w + kFVeta, Kb);
#pragma unroll
  for (int k = 0; k < 9; ++k) g[k] = g[k] * sb;
  double K2 = w[kFKt] + w[kFKt + 4] + w[kFKt + 8];
  const double s = nhc_half(M, tloop, hdt, Nf, kT, p + kQ, w + kFXi, w + kFVxi, K2);
#pragma unroll
  for (int k = 0; k < 9; ++k) kt[k] = w[kFKt + k] * (s * s);
  const double V = fabs(det3(C1));
  cell_kick(g, kt, vr, P * V, Nf, hdt, W);
  const double trg = g[0] + g[4] + g[8];
  double a[9], o[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) a[k] = g[k];
  jacobi3(a, o);
  double fev[3], fkf[3], fer[3], fdf[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double lam = a[4 * k], mu = lam + trg / Nf;
    const double am = mu * dt, b = lam * dt;
    fev[k] = exp(-0.5 * am);
    fkf[k] = hdt * exp(-0.25 * am) * sinhc(0.25 * am);
    fer[k] = exp(b);
    fdf[k] = dt * exp(0.5 * b) * sinhc(0.5 * b);
  }
  double Ev[9], Kf[9], Er[9], Df[9];
  bool ok = sym_fn(o, fev, Ev) && sym_fn(o, fkf, Kf) && sym_fn(o, fer, Er) && sym_fn(o, fdf, Df) && isfinite(s);
  double nc[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      nc[3 * r + i] = Er[3 * i + 0] * C1[3 * r + 0] + Er[3 * i + 1] * C1[3 * r + 1] + Er[3 * i + 2] * C1[3 * r + 2];
      ok = ok && isfinite(nc[3 * r + i]);
    }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    w[kFG + k] = g[k];
    w[kFKt + k] = kt[k];
  }
  ok = ok && flex_row_finite(w);
  if (!ok) {
    err[f] = 1;
    frozen_coef_flex(c);
    return;
  }
  for (int k = 0; k < kFS; ++k) s0[k] = w[k];
  c[0] = s;
  c[1] = 1.0;
  c[2] = 1.0;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    C[k] = nc[k];
    c[kFEv + k] = Ev[k];
    c[kFK + k] = Kf[k];
    c[kFEr + k] = Er[k];
    c[kFD + k] = Df[k];
  }
}

// y = A x for a row-major 3x3 A read from global memory
__device__ __forceinline__ void matvec3(const double* A, const double (&x)[3], double (&y)[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = A[3 * i + 0] * x[0] + A[3 * i + 1] * x[1] + A[3 * i + 2] * x[2];
}

// the atoms of active frames: v <- s v;  v <- E_v v + K F/m;  r <- E_r r + D v
__global__ void __launch_bounds__(kNptThreads)
k_nptf_move(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ forces,
            const double* __restrict__ coef, double* __restrict__ pos, double* __restrict__ vel) {
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kFC * (int64_t)f;
  if (c[1] == 0.0) return;
  const double s = c[0];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads) {
    const double m = mass[i];
    double v1[3], a[3], r[3], ev[3], ka[3], er[3], dv[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      v1[d] = s * vel[3 * i + d];
      a[d] = forces[3 * i + d] / m;
      r[d] = pos[3 * i + d];
    }
    matvec3(c + kFEv, v1, ev);
    matvec3(c + kFK, a, ka);
    double v2[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) v2[d] = ev[d] + ka[d];
    matvec3(c + kFEr, r, er);
    matvec3(c + kFD, v2, dv);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      vel[3 * i + d] = v2[d];
      pos[3 * i + d] = er[d] + dv[d];
    }
  }
}

// the atoms of active frames: v <- E_v v + K F_new/m;  forces <- F_new;  part[f, b, :] = the CTA's sum of m v (x) v
// as {xx, yy, zz, yz, xz, xy} (0 for an inactive frame)
__global__ void __launch_bounds__(kNptThreads)
k_nptf_kick(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ f_new,
            const double* __restrict__ coef, double* __restrict__ vel, double* __restrict__ forces,
            double* __restrict__ part) {
  __shared__ double smem[kNptThreads / 32];
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kFC * (int64_t)f;
  const bool active = c[1] != 0.0;
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (active)
    for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads) {
      const double m = mass[i];
      double v0[3], a[3], ev[3], ka[3], v[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const double fd = f_new[3 * i + d];
        v0[d] = vel[3 * i + d];
        a[d] = fd / m;
        forces[3 * i + d] = fd;
      }
      matvec3(c + kFEv, v0, ev);
      matvec3(c + kFK, a, ka);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        v[d] = ev[d] + ka[d];
        vel[3 * i + d] = v[d];
      }
      acc[0] += m * v[0] * v[0];
      acc[1] += m * v[1] * v[1];
      acc[2] += m * v[2] * v[2];
      acc[3] += m * v[1] * v[2];
      acc[4] += m * v[0] * v[2];
      acc[5] += m * v[0] * v[1];
    }
  double* out = part + ((int64_t)f * nblk + blockIdx.x) * 6;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double t = cta_sum(acc[k], smem);
    if (threadIdx.x == 0) out[k] = t;
  }
}

// One thread per frame (frames with err set get coef[2] = 1 only): Kt = the sum of part in index order, v_g += dt/2
// G_g / W_g with the new virial and the new cell's volume, NHC_part(dt/2) (Kt *= s^2), NHC_baro(dt/2) (scales v_g);
// stores Kt and the virial, coef[2] = the particles' scale.
__global__ void k_nptf_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt,
                            const double* __restrict__ prm, const double* __restrict__ part,
                            const double* __restrict__ vir_new, const double* __restrict__ cell,
                            double* __restrict__ st, double* __restrict__ vir, double* __restrict__ coef,
                            int32_t* __restrict__ err, double* __restrict__ wk) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* c = coef + kFC * (int64_t)f;
  if (err[f]) {
    c[2] = 1.0;
    return;
  }
  const double* p = prm + kP * (int64_t)f;
  double* s0 = st + kFS * (int64_t)f;
  double* w = wk + kFS * (int64_t)f;
  for (int k = 0; k < kFS; ++k) w[k] = s0[k];
  double k6[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int b = 0; b < nblk; ++b) {
    const double* pb = part + ((int64_t)f * nblk + b) * 6;
#pragma unroll
    for (int k = 0; k < 6; ++k) k6[k] += pb[k];
  }
  double kt[9] = {k6[0], k6[5], k6[4], k6[5], k6[1], k6[3], k6[4], k6[3], k6[2]};
  const double kT = p[kKT], P = p[kPres], W = p[kW], Nf = p[kNf], hdt = 0.5 * dt;
  const double* vr = vir_new + 9 * (int64_t)f;
  double g[9], C1[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    g[k] = w[kFG + k];
    C1[k] = cell[9 * (int64_t)f + k];
  }
  const double V = fabs(det3(C1));
  cell_kick(g, kt, vr, P * V, Nf, hdt, W);
  double K2 = kt[0] + kt[4] + kt[8];
  const double s = nhc_half(M, tloop, hdt, Nf, kT, p + kQ, w + kFXi, w + kFVxi, K2);
#pragma unroll
  for (int k = 0; k < 9; ++k) kt[k] = kt[k] * (s * s);
  double Kb = W * frob2(g);
  const double sb = nhc_half(Mp, ploop, hdt, kNg, kT, p + kQp, w + kFEta, w + kFVeta, Kb);
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    w[kFG + k] = g[k] * sb;
    w[kFKt + k] = kt[k];
  }
  bool ok = flex_row_finite(w) && isfinite(s);
  for (int k = 0; k < 9; ++k) ok = ok && isfinite(vr[k]);
  if (!ok) {
    err[f] = 1;
    c[2] = 1.0;
    return;
  }
  for (int k = 0; k < kFS; ++k) s0[k] = w[k];
  for (int k = 0; k < 9; ++k) vir[9 * (int64_t)f + k] = vr[k];
  c[2] = s;
}

// the atoms of active frames: v <- coef[2] v
__global__ void __launch_bounds__(kNptThreads)
k_nptf_scale(const int64_t* __restrict__ atom_ptr, const double* __restrict__ coef, double* __restrict__ vel) {
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* c = coef + kFC * (int64_t)f;
  if (c[1] == 0.0) return;
  const double s = c[2];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  for (int64_t i = beg + (int64_t)blockIdx.x * kNptThreads + threadIdx.x; i < end; i += (int64_t)nblk * kNptThreads)
    for (int d = 0; d < 3; ++d) vel[3 * i + d] = s * vel[3 * i + d];
}

// One CTA.  Row step % rows of the log, per frame: E_pot, E_kin, T, V, tr(P_int)/3, H, the cell [9] and the pressure
// tensor P_int = (Kt + vir) / V [9]; the sticky flags as nqb_npt_log writes them; then step += 1.
__global__ void __launch_bounds__(kNptThreads)
k_nptf_log(int F, int M, int Mp, const double* __restrict__ e_pot, const double* __restrict__ prm,
           const double* __restrict__ st, const double* __restrict__ vir, const double* __restrict__ cell,
           const int64_t* __restrict__ num_edges, const int32_t* __restrict__ overflow,
           const int32_t* __restrict__ sorted, int64_t rows, int64_t* step, double* __restrict__ log,
           int64_t* __restrict__ flags) {
  const int64_t s = *step;
  double* row = log + (s % rows) * (int64_t)F * NQB_NPTF_LOG_FIELDS;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const double* p = prm + kP * (int64_t)f;
    const double* w = st + kFS * (int64_t)f;
    const double* vr = vir + 9 * (int64_t)f;
    const double* C = cell + 9 * (int64_t)f;
    double g[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) g[k] = w[kFG + k];
    const double kT = p[kKT], K2 = w[kFKt] + w[kFKt + 4] + w[kFKt + 8];
    const double V = fabs(det3(C));
    const double ep = e_pot[f], ke = 0.5 * K2;
    double h = ep + ke + 0.5 * p[kW] * frob2(g) + p[kPres] * V;
    for (int k = 0; k < M; ++k)
      h += 0.5 * p[kQ + k] * w[kFVxi + k] * w[kFVxi + k] + (k == 0 ? p[kNf] * kT : kT) * w[kFXi + k];
    for (int k = 0; k < Mp; ++k)
      h += 0.5 * p[kQp + k] * w[kFVeta + k] * w[kFVeta + k] + (k == 0 ? kNg * kT : kT) * w[kFEta + k];
    double* r = row + (int64_t)f * NQB_NPTF_LOG_FIELDS;
    r[0] = ep;
    r[1] = ke;
    r[2] = K2 / p[kNfkB];
    r[3] = V;
    r[4] = (K2 + (vr[0] + vr[4] + vr[8])) / (3.0 * V);
    r[5] = h;
    for (int k = 0; k < 9; ++k) {
      r[6 + k] = C[k];
      r[15 + k] = (w[kFKt + k] + vr[k]) / V;
    }
  }
  __syncthreads();  // every thread has read *step
  if (threadIdx.x == 0) {
    if (*overflow != 0) {
      flags[0] = 1;
      if (flags[2] < 0) flags[2] = s;
    }
    if (*sorted != 1) flags[1] = 1;
    if (*num_edges > flags[3]) flags[3] = *num_edges;
    *step = s + 1;
  }
}

int npt_launch_done() {
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

bool chains_ok(int M, int Mp, int tloop, int ploop) {
  return M >= 0 && M <= kM && Mp >= 0 && Mp <= kM && tloop >= 1 && ploop >= 1;
}

}  // namespace

extern "C" int nqb_npt_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* prm, const double* C0,
                           const double* vir, double* state, double* cell, double* coef, int32_t* err, double* work,
                           nqb_stream_t st) {
  if (F < 0 || !chains_ok(M, Mp, tloop, ploop))
    return nqb_set_error("nqb_npt_pre: needs F >= 0, chains in [0, NQB_NPT_MAX_CHAIN] and loops >= 1");
  if (F == 0) return 0;
  if (!prm || !C0 || !vir || !state || !cell || !coef || !err || !work) return nqb_set_error("nqb_npt_pre: null pointer");
  k_npt_pre<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, M, Mp, tloop, ploop, dt, prm, C0, vir, state,
                                                                      cell, coef, err, work);
  return npt_launch_done();
}

extern "C" int nqb_npt_move(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* forces,
                            const double* coef, double* pos, double* vel, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_npt_move: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_npt_move: at most 65535 frames");
  if (!atom_ptr || !mass || !forces || !coef || !pos || !vel) return nqb_set_error("nqb_npt_move: null pointer");
  k_npt_move<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, forces, coef, pos,
                                                                                    vel);
  return npt_launch_done();
}

extern "C" int nqb_npt_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new,
                            const double* coef, double* vel, double* forces, double* part, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_npt_kick: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_npt_kick: at most 65535 frames");
  if (!atom_ptr || !mass || !f_new || !coef || !vel || !forces || !part) return nqb_set_error("nqb_npt_kick: null pointer");
  k_npt_kick<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, f_new, coef, vel,
                                                                                    forces, part);
  return npt_launch_done();
}

extern "C" int nqb_npt_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt, const double* prm,
                            const double* part, const double* vir_new, double* state, double* vir, double* coef,
                            int32_t* err, double* work, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || !chains_ok(M, Mp, tloop, ploop))
    return nqb_set_error("nqb_npt_post: needs F >= 0, nblk >= 1, chains in [0, NQB_NPT_MAX_CHAIN] and loops >= 1");
  if (F == 0) return 0;
  if (!prm || !part || !vir_new || !state || !vir || !coef || !err || !work)
    return nqb_set_error("nqb_npt_post: null pointer");
  k_npt_post<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, nblk, M, Mp, tloop, ploop, dt, prm, part,
                                                                        vir_new, state, vir, coef, err, work);
  return npt_launch_done();
}

extern "C" int nqb_npt_scale(int F, int nblk, const int64_t* atom_ptr, const double* coef, double* vel,
                             nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_npt_scale: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_npt_scale: at most 65535 frames");
  if (!atom_ptr || !coef || !vel) return nqb_set_error("nqb_npt_scale: null pointer");
  k_npt_scale<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, coef, vel);
  return npt_launch_done();
}

extern "C" int nqb_npt_log(int F, int M, int Mp, const double* e_pot, const double* prm, const double* state,
                           const double* vir, const int64_t* num_edges, const int32_t* overflow, const int32_t* sorted,
                           int64_t rows, int64_t* step, double* log, int64_t* flags, nqb_stream_t st) {
  if (F < 0 || rows < 1 || M < 0 || M > kM || Mp < 0 || Mp > kM)
    return nqb_set_error("nqb_npt_log: needs F >= 0, rows >= 1 and chains in [0, NQB_NPT_MAX_CHAIN]");
  if (!e_pot || !prm || !state || !vir || !num_edges || !overflow || !sorted || !step || !log || !flags)
    return nqb_set_error("nqb_npt_log: null pointer");
  k_npt_log<<<1, kNptThreads, 0, (cudaStream_t)st>>>(F, M, Mp, e_pot, prm, state, vir, num_edges, overflow, sorted,
                                                    rows, step, log, flags);
  return npt_launch_done();
}

extern "C" int nqb_nptf_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* prm, const double* vir,
                            double* state, double* cell, double* coef, int32_t* err, double* work, nqb_stream_t st) {
  if (F < 0 || !chains_ok(M, Mp, tloop, ploop))
    return nqb_set_error("nqb_nptf_pre: needs F >= 0, chains in [0, NQB_NPT_MAX_CHAIN] and loops >= 1");
  if (F == 0) return 0;
  if (!prm || !vir || !state || !cell || !coef || !err || !work) return nqb_set_error("nqb_nptf_pre: null pointer");
  k_nptf_pre<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, M, Mp, tloop, ploop, dt, prm, vir, state,
                                                                       cell, coef, err, work);
  return npt_launch_done();
}

extern "C" int nqb_nptf_move(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* forces,
                             const double* coef, double* pos, double* vel, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_nptf_move: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_nptf_move: at most 65535 frames");
  if (!atom_ptr || !mass || !forces || !coef || !pos || !vel) return nqb_set_error("nqb_nptf_move: null pointer");
  k_nptf_move<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, forces, coef,
                                                                                     pos, vel);
  return npt_launch_done();
}

extern "C" int nqb_nptf_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new,
                             const double* coef, double* vel, double* forces, double* part, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_nptf_kick: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_nptf_kick: at most 65535 frames");
  if (!atom_ptr || !mass || !f_new || !coef || !vel || !forces || !part)
    return nqb_set_error("nqb_nptf_kick: null pointer");
  k_nptf_kick<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, f_new, coef,
                                                                                     vel, forces, part);
  return npt_launch_done();
}

extern "C" int nqb_nptf_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt, const double* prm,
                             const double* part, const double* vir_new, const double* cell, double* state, double* vir,
                             double* coef, int32_t* err, double* work, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || !chains_ok(M, Mp, tloop, ploop))
    return nqb_set_error("nqb_nptf_post: needs F >= 0, nblk >= 1, chains in [0, NQB_NPT_MAX_CHAIN] and loops >= 1");
  if (F == 0) return 0;
  if (!prm || !part || !vir_new || !cell || !state || !vir || !coef || !err || !work)
    return nqb_set_error("nqb_nptf_post: null pointer");
  k_nptf_post<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, nblk, M, Mp, tloop, ploop, dt, prm, part,
                                                                         vir_new, cell, state, vir, coef, err, work);
  return npt_launch_done();
}

extern "C" int nqb_nptf_scale(int F, int nblk, const int64_t* atom_ptr, const double* coef, double* vel,
                              nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_nptf_scale: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_nptf_scale: at most 65535 frames");
  if (!atom_ptr || !coef || !vel) return nqb_set_error("nqb_nptf_scale: null pointer");
  k_nptf_scale<<<dim3((unsigned)nblk, (unsigned)F), kNptThreads, 0, (cudaStream_t)st>>>(atom_ptr, coef, vel);
  return npt_launch_done();
}

extern "C" int nqb_nptf_log(int F, int M, int Mp, const double* e_pot, const double* prm, const double* state,
                            const double* vir, const double* cell, const int64_t* num_edges, const int32_t* overflow,
                            const int32_t* sorted, int64_t rows, int64_t* step, double* log, int64_t* flags,
                            nqb_stream_t st) {
  if (F < 0 || rows < 1 || M < 0 || M > kM || Mp < 0 || Mp > kM)
    return nqb_set_error("nqb_nptf_log: needs F >= 0, rows >= 1 and chains in [0, NQB_NPT_MAX_CHAIN]");
  if (!e_pot || !prm || !state || !vir || !cell || !num_edges || !overflow || !sorted || !step || !log || !flags)
    return nqb_set_error("nqb_nptf_log: null pointer");
  k_nptf_log<<<1, kNptThreads, 0, (cudaStream_t)st>>>(F, M, Mp, e_pot, prm, state, vir, cell, num_edges, overflow,
                                                     sorted, rows, step, log, flags);
  return npt_launch_done();
}
