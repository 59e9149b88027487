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
