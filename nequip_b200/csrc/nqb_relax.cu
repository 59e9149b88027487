// Structure relaxation on the device: ASE's FIRE (ase/optimize/fire.py, FIRE.step) per frame f of a batch, optionally
// on the degrees of freedom of ASE's FrechetCellFilter, in float64, sm_90a.  One relaxation step of
// nequip_b200/relax.py (GraphedRelax) is
//   nqb_relax_fire -> nqb_relax_move -> nqb_nl_frames_set_cells -> neighbour list + model -> nqb_relax_gforce
//   -> nqb_relax_finish
// captured as one CUDA graph.  The atoms of frame f are [atom_ptr[f], atom_ptr[f+1]); the atom kernels run (nblk, F)
// CTAs of kRxThreads threads as the nqb_md kernels do, and every sum over atoms is a per-CTA partial in a fixed order
// that the per-frame consumer adds in index order: no floating-point atomics, so a launch shape gives results that
// depend only on its inputs.
//
// Cell degrees of freedom (has_cell): Q = c log Fd (Fd the deformation gradient, c = cfac[f]); the atoms' DOF are s
// with r = s Fd^T (rows), the cell is C0 Fd^T.  Generalised forces: g_i = f_i Fd and, with W = virial - p V I,
// G = (1/c) D exp(L^T)[W Fd^-T], L = Q / c -- the adjoint form of G_uv = (1/c) sum_ab (W Fd^-T)_ab D exp(L)[E_uv]_ab,
// one 6x6 exponential [[L^T, M], [0, L^T]] whose upper-right block is the Frechet derivative.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/nqb.h"

extern "C" int nqb_set_error(const char* msg);
extern "C" void nqb_count_launch(void);

namespace {

constexpr int kRxThreads = 256;
constexpr int kTaylor = 18;  // degree of the Taylor polynomial after scaling to norm <= 1/2 (error < 1e-20)

struct FireParams {
  double maxstep, dtmax, finc, fdec, astart, fa;
  int nmin;
};

// z = x y (3x3 row-major; z distinct from x and y)
__device__ __forceinline__ void mm3(const double* x, const double* y, double* z) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) z[3 * i + j] = x[3 * i] * y[j] + x[3 * i + 1] * y[3 + j] + x[3 * i + 2] * y[6 + j];
}

// exp([[A, B], [0, A]]) = [[EA, EB], [0, EA]] by scaling and squaring: the 6x6 is kept as its two 3x3 blocks, since
// [[A1, B1], [0, A1]] [[A2, B2], [0, A2]] = [[A1 A2, A1 B2 + B1 A2], [0, A1 A2]].  B = 0 gives exp(A).  A non-finite
// input gives NaN.
__device__ void expm_pair(const double* A, const double* B, double* EA, double* EB) {
  double nrm = 0.0;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) s += fabs(A[3 * r + k]) + fabs(B[3 * r + k]);
    nrm = fmax(nrm, s);
  }
  bool finite = isfinite(nrm);
#pragma unroll
  for (int k = 0; k < 9; ++k) finite = finite && isfinite(A[k]) && isfinite(B[k]);
  if (!finite) {
#pragma unroll
    for (int k = 0; k < 9; ++k) EA[k] = EB[k] = NAN;
    return;
  }
  int sq = 0;
  double scale = 1.0;
  while (nrm * scale > 0.5) {
    scale *= 0.5;
    ++sq;
  }
  double XA[9], XB[9], TA[9], TB[9], UA[9], UB[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    XA[k] = A[k] * scale;
    XB[k] = B[k] * scale;
    TA[k] = (k % 4) == 0 ? 1.0 : 0.0;
    TB[k] = 0.0;
  }
  // Horner: T = I + X T / k for k = K .. 1
#pragma unroll 1
  for (int k = kTaylor; k >= 1; --k) {
    const double r = 1.0 / k;
    mm3(XA, TA, UA);
    mm3(XA, TB, UB);
    double V[9];
    mm3(XB, TA, V);
#pragma unroll
    for (int q = 0; q < 9; ++q) {
      TA[q] = ((q % 4) == 0 ? 1.0 : 0.0) + UA[q] * r;
      TB[q] = (UB[q] + V[q]) * r;
    }
  }
#pragma unroll 1
  for (int i = 0; i < sq; ++i) {
    mm3(TA, TA, UA);
    mm3(TA, TB, UB);
    double V[9];
    mm3(TB, TA, V);
#pragma unroll
    for (int q = 0; q < 9; ++q) {
      TA[q] = UA[q];
      TB[q] = UB[q] + V[q];
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    EA[k] = TA[k];
    EB[k] = TB[k];
  }
}

__device__ __forceinline__ double det3(const double* c) {
  return c[0] * (c[4] * c[8] - c[5] * c[7]) - c[1] * (c[3] * c[8] - c[5] * c[6]) + c[2] * (c[3] * c[7] - c[4] * c[6]);
}

// the CTA's sums of (a, b, c) and max of m, valid in thread 0; fixed order
__device__ __forceinline__ void cta_reduce(double& a, double& b, double& c, double& m, double (*smem)[4]) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    smem[warp][0] = a;
    smem[warp][1] = b;
    smem[warp][2] = c;
    smem[warp][3] = m;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = b = c = 0.0;
    m = 0.0;
    for (int w = 0; w < kRxThreads / 32; ++w) {
      a += smem[w][0];
      b += smem[w][1];
      c += smem[w][2];
      m = fmax(m, smem[w][3]);
    }
  }
}

// One thread per frame: the FIRE scalars and the cell DOF.  coef[f] = {cv, cg, sc, active}: the atoms then take
// v = cv v + cg g and s += sc v.
__global__ void k_relax_fire(int F, int nblk, const double* __restrict__ part, FireParams fp, int has_cell,
                             const double* __restrict__ cfac, const double* __restrict__ C0,
                             const double* __restrict__ gcell, double* __restrict__ Q, double* __restrict__ vcell,
                             double* __restrict__ Fd, double* __restrict__ cell, double* __restrict__ fs,
                             int64_t* __restrict__ is, double* __restrict__ coef) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double* cf = coef + 4 * (int64_t)f;
  int64_t* st = is + NQB_RELAX_ISTATE * (int64_t)f;
  if (st[2] || st[3]) {  // converged or failed: frozen
    cf[0] = 1.0;
    cf[1] = cf[2] = cf[3] = 0.0;
    return;
  }
  double vg = 0.0, vv = 0.0, gg = 0.0;
  for (int b = 0; b < nblk; ++b) {
    const double* p = part + 4 * ((int64_t)f * nblk + b);
    vg += p[0];
    vv += p[1];
    gg += p[2];
  }
  if (has_cell)
    for (int k = 0; k < 9; ++k) {
      const double v = vcell[9 * (int64_t)f + k], g = gcell[9 * (int64_t)f + k];
      vg += v * g;
      vv += v * v;
      gg += g * g;
    }
  double dt = fs[2 * (int64_t)f], a = fs[2 * (int64_t)f + 1], cv, cg;
  if (st[1]) {  // first step: v = 0
    cv = cg = 0.0;
    st[1] = 0;
  } else if (vg > 0.0) {
    cv = 1.0 - a;
    cg = a * sqrt(vv) / sqrt(gg);
    if (st[0] > fp.nmin) {
      dt = fmin(dt * fp.finc, fp.dtmax);
      a *= fp.fa;
    }
    st[0] += 1;
  } else {
    cv = cg = 0.0;
    a = fp.astart;
    dt *= fp.fdec;
    st[0] = 0;
  }
  cg += dt;  // v += dt g
  // |dr|^2 = dt^2 |cv v + cg g|^2 over the frame's whole vector
  const double nv2 = cv * cv * vv + 2.0 * cv * cg * vg + cg * cg * gg;
  const double ndr = dt * sqrt(fmax(nv2, 0.0));
  const double sc = ndr > fp.maxstep ? dt * (fp.maxstep / ndr) : dt;
  fs[2 * (int64_t)f] = dt;
  fs[2 * (int64_t)f + 1] = a;
  st[4] += 1;
  cf[0] = cv;
  cf[1] = cg;
  cf[2] = sc;
  cf[3] = 1.0;
  if (!has_cell) return;
  double L[9], Z[9], E[9], U[9];
  const double c = cfac[f];
  for (int k = 0; k < 9; ++k) {
    const int64_t i = 9 * (int64_t)f + k;
    const double v = cv * vcell[i] + cg * gcell[i];
    vcell[i] = v;
    Q[i] = Q[i] + sc * v;
    L[k] = Q[i] / c;
    Z[k] = 0.0;
  }
  expm_pair(L, Z, E, U);
  double c0[9], nc[9];
  for (int k = 0; k < 9; ++k) {
    Fd[9 * (int64_t)f + k] = E[k];
    c0[k] = C0[9 * (int64_t)f + k];
  }
  // cell = C0 Fd^T
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      nc[3 * i + j] = c0[3 * i] * E[3 * j] + c0[3 * i + 1] * E[3 * j + 1] + c0[3 * i + 2] * E[3 * j + 2];
  for (int k = 0; k < 9; ++k) cell[9 * (int64_t)f + k] = nc[k];
}

// v = cv v + cg g;  s += sc v;  pos = s Fd^T (has_cell) -- the atoms of active frames
__global__ void __launch_bounds__(kRxThreads)
k_relax_move(const int64_t* __restrict__ atom_ptr, const double* __restrict__ coef, int has_cell,
             const double* __restrict__ Fd, const double* __restrict__ g, double* __restrict__ vel,
             double* __restrict__ s, double* __restrict__ pos) {
  const int f = blockIdx.y, nblk = gridDim.x;
  const double* cf = coef + 4 * (int64_t)f;
  if (cf[3] == 0.0) return;
  const double cv = cf[0], cg = cf[1], sc = cf[2];
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  double D[9];
  if (has_cell)
    for (int k = 0; k < 9; ++k) D[k] = Fd[9 * (int64_t)f + k];
  for (int64_t i = beg + (int64_t)blockIdx.x * kRxThreads + threadIdx.x; i < end; i += (int64_t)nblk * kRxThreads) {
    double x[3];
    for (int d = 0; d < 3; ++d) {
      const double v = cv * vel[3 * i + d] + cg * g[3 * i + d];
      vel[3 * i + d] = v;
      x[d] = (has_cell ? s[3 * i + d] : pos[3 * i + d]) + sc * v;
    }
    if (has_cell) {
      for (int d = 0; d < 3; ++d) {
        s[3 * i + d] = x[d];
        pos[3 * i + d] = x[0] * D[3 * d] + x[1] * D[3 * d + 1] + x[2] * D[3 * d + 2];
      }
    } else {
      for (int d = 0; d < 3; ++d) pos[3 * i + d] = x[d];
    }
  }
}

// g = forces Fd (has_cell) or forces;  part[f, b] = {sum v.g, sum v.v, sum g.g, max |g_i|^2} of CTA (b, f), a
// non-finite row counting as +inf
__global__ void __launch_bounds__(kRxThreads)
k_relax_gforce(const int64_t* __restrict__ atom_ptr, int has_cell, const double* __restrict__ Fd,
               const double* __restrict__ forces, const double* __restrict__ vel, double* __restrict__ g,
               double* __restrict__ part) {
  __shared__ double smem[kRxThreads / 32][4];
  const int f = blockIdx.y, nblk = gridDim.x;
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  double D[9];
  if (has_cell)
    for (int k = 0; k < 9; ++k) D[k] = Fd[9 * (int64_t)f + k];
  double vg = 0.0, vv = 0.0, gg = 0.0, mx = 0.0;
  for (int64_t i = beg + (int64_t)blockIdx.x * kRxThreads + threadIdx.x; i < end; i += (int64_t)nblk * kRxThreads) {
    const double f0 = forces[3 * i], f1 = forces[3 * i + 1], f2 = forces[3 * i + 2];
    double r2 = 0.0;
    for (int d = 0; d < 3; ++d) {
      const double gd = has_cell ? f0 * D[d] + f1 * D[3 + d] + f2 * D[6 + d] : (d == 0 ? f0 : d == 1 ? f1 : f2);
      const double v = vel[3 * i + d];
      g[3 * i + d] = gd;
      vg += v * gd;
      vv += v * v;
      r2 += gd * gd;
    }
    gg += r2;
    mx = fmax(mx, isfinite(r2) ? r2 : INFINITY);
  }
  cta_reduce(vg, vv, gg, mx, smem);
  if (threadIdx.x == 0) {
    double* p = part + 4 * ((int64_t)f * nblk + blockIdx.x);
    p[0] = vg;
    p[1] = vv;
    p[2] = gg;
    p[3] = mx;
  }
}

// One CTA, thread t handling frames t, t + kRxThreads, ...: the cell's generalised force, the convergence and failure
// tests of frames that are not frozen, log row step % rows {E_pot, E_pot + p V, fmax, V}, the sticky flags as in
// nqb_md_log, then step += 1.
__global__ void __launch_bounds__(kRxThreads)
k_relax_finish(int F, int nblk, const double* __restrict__ part, int has_cell, double pressure,
               const double* __restrict__ cfac, const double* __restrict__ Q, const double* __restrict__ Fd,
               const double* __restrict__ cell, const double* __restrict__ virial, const double* __restrict__ e_pot,
               double fmax2, double fail2, double* __restrict__ gcell, int64_t* __restrict__ is,
               const int64_t* __restrict__ num_edges, const int32_t* __restrict__ overflow,
               const int32_t* __restrict__ sorted, int64_t rows, int64_t* step, double* __restrict__ log,
               int64_t* __restrict__ flags) {
  const int64_t s = *step;
  double* row = log + (s % rows) * (int64_t)F * NQB_RELAX_LOG_FIELDS;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    double mx = 0.0;
    for (int b = 0; b < nblk; ++b) mx = fmax(mx, part[4 * ((int64_t)f * nblk + b) + 3]);
    double c[9];
    for (int k = 0; k < 9; ++k) c[k] = cell[9 * (int64_t)f + k];
    const double V = fabs(det3(c));
    if (has_cell) {
      double D[9], L[9], M[9], W[9], Di[9], E[9], G[9];
      const double cf = cfac[f];
      for (int k = 0; k < 9; ++k) D[k] = Fd[9 * (int64_t)f + k];
      // W = virial - p V I;  M = W Fd^-T (Fd^-T = adj(Fd)^T / det Fd);  L = (Q / c)^T
      Di[0] = D[4] * D[8] - D[5] * D[7];
      Di[1] = D[5] * D[6] - D[3] * D[8];
      Di[2] = D[3] * D[7] - D[4] * D[6];
      Di[3] = D[2] * D[7] - D[1] * D[8];
      Di[4] = D[0] * D[8] - D[2] * D[6];
      Di[5] = D[1] * D[6] - D[0] * D[7];
      Di[6] = D[1] * D[5] - D[2] * D[4];
      Di[7] = D[2] * D[3] - D[0] * D[5];
      Di[8] = D[0] * D[4] - D[1] * D[3];
      const double dD = D[0] * Di[0] + D[1] * Di[1] + D[2] * Di[2];
      for (int k = 0; k < 9; ++k) {
        Di[k] /= dD;
        W[k] = virial[9 * (int64_t)f + k] - ((k % 4) == 0 ? pressure * V : 0.0);
        L[k] = Q[9 * (int64_t)f + 3 * (k % 3) + k / 3] / cf;
      }
      mm3(W, Di, M);
      expm_pair(L, M, E, G);
      for (int r = 0; r < 3; ++r) {
        double r2 = 0.0;
        for (int k = 0; k < 3; ++k) {
          const double gk = G[3 * r + k] / cf;
          gcell[9 * (int64_t)f + 3 * r + k] = gk;
          r2 += gk * gk;
        }
        mx = fmax(mx, isfinite(r2) ? r2 : INFINITY);
      }
    }
    int64_t* st = is + NQB_RELAX_ISTATE * (int64_t)f;
    if (!st[2] && !st[3]) {
      if (!(mx <= fail2)) st[3] = 1;
      else if (mx < fmax2) st[2] = 1;
    }
    const double ep = e_pot[f];
    double* r = row + (int64_t)f * NQB_RELAX_LOG_FIELDS;
    r[0] = ep;
    r[1] = ep + pressure * V;
    r[2] = sqrt(mx);
    r[3] = V;
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

int rx_launch_done() {
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

}  // namespace

extern "C" int nqb_relax_fire(int F, int nblk, const double* part, const double* fire_host, int has_cell,
                              const double* cfac, const double* C0, const double* gcell, double* Q, double* vcell,
                              double* Fd, double* cell, double* fs, int64_t* is, double* coef, nqb_stream_t st) {
  if (F < 0 || nblk < 1) return nqb_set_error("nqb_relax_fire: needs F >= 0 and nblk >= 1");
  if (F == 0) return 0;
  if (!part || !fire_host || !fs || !is || !coef) return nqb_set_error("nqb_relax_fire: null pointer");
  if (has_cell && (!cfac || !C0 || !gcell || !Q || !vcell || !Fd || !cell))
    return nqb_set_error("nqb_relax_fire: null cell pointer");
  FireParams fp{fire_host[0], fire_host[1], fire_host[2], fire_host[3], fire_host[4], fire_host[5], (int)fire_host[6]};
  k_relax_fire<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, nblk, part, fp, has_cell ? 1 : 0, cfac, C0,
                                                                          gcell, Q, vcell, Fd, cell, fs, is, coef);
  return rx_launch_done();
}

extern "C" int nqb_relax_move(int F, int nblk, const int64_t* atom_ptr, const double* coef, int has_cell,
                              const double* Fd, const double* g, double* vel, double* s, double* pos,
                              nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_relax_move: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_relax_move: at most 65535 frames");
  if (!atom_ptr || !coef || !g || !vel || !pos || (has_cell && (!Fd || !s)))
    return nqb_set_error("nqb_relax_move: null pointer");
  k_relax_move<<<dim3((unsigned)nblk, (unsigned)F), kRxThreads, 0, (cudaStream_t)st>>>(atom_ptr, coef, has_cell ? 1 : 0,
                                                                                      Fd, g, vel, s, pos);
  return rx_launch_done();
}

extern "C" int nqb_relax_gforce(int F, int nblk, const int64_t* atom_ptr, int has_cell, const double* Fd,
                                const double* forces, const double* vel, double* g, double* part, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_relax_gforce: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (F > 65535) return nqb_set_error("nqb_relax_gforce: at most 65535 frames");
  if (!atom_ptr || !forces || !vel || !g || !part || (has_cell && !Fd))
    return nqb_set_error("nqb_relax_gforce: null pointer");
  k_relax_gforce<<<dim3((unsigned)nblk, (unsigned)F), kRxThreads, 0, (cudaStream_t)st>>>(atom_ptr, has_cell ? 1 : 0, Fd,
                                                                                        forces, vel, g, part);
  return rx_launch_done();
}

extern "C" int nqb_relax_finish(int F, int nblk, const double* part, int has_cell, double pressure, const double* cfac,
                                const double* Q, const double* Fd, const double* cell, const double* virial,
                                const double* e_pot, double fmax, double fail_force, double* gcell, int64_t* is,
                                const int64_t* num_edges, const int32_t* overflow, const int32_t* sorted, int64_t rows,
                                int64_t* step, double* log, int64_t* flags, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || rows < 1) return nqb_set_error("nqb_relax_finish: needs F >= 0, nblk >= 1 and rows >= 1");
  if (!part || !cell || !e_pot || !is || !num_edges || !overflow || !sorted || !step || !log || !flags)
    return nqb_set_error("nqb_relax_finish: null pointer");
  if (has_cell && (!cfac || !Q || !Fd || !virial || !gcell)) return nqb_set_error("nqb_relax_finish: null cell pointer");
  k_relax_finish<<<1, kRxThreads, 0, (cudaStream_t)st>>>(F, nblk, part, has_cell ? 1 : 0, pressure, cfac, Q, Fd, cell,
                                                         virial, e_pot, fmax * fmax, fail_force * fail_force, gcell, is,
                                                         num_edges, overflow, sorted, rows, step, log, flags);
  return rx_launch_done();
}
