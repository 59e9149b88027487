// ZBL screened-nuclear repulsion (a per-edge pair energy added to the per-atom energies), fp64, sm_90a.
//
// Reference semantics (paths under /root/reference):
//   _ZBL / ZBL                    nequip/nn/pair_potential.py:230-271, 274-386
//   PolynomialCutoff              nequip/nn/embedding/cutoffs.py:17-27
//   appended before AtomwiseReduce nequip/model/energy_modules.py:10-35
//
// Per edge e = (i -> j), i = edge_index[0][e] the centre:
//   eps_e = A_ij / r * psi(x) * f_c(r / r_max),  x = (S_ij * r) / a0,  psi(x) = sum_k c_k exp(d_k x)
// with the per-ordered-type-pair table  A_ij = 0.5 * qqr2e * Z_i Z_j  and  S_ij = Z_i^0.23 + Z_j^0.23  (built on the
// host in the model dtype, as the reference rounds them, then widened to fp64).  eps_e is summed onto the centre.
//
//   k_zbl_fwd  one warp per centre row of the destination CSR: the lanes evaluate 32 edges of the row at a time and
//              every lane then adds them in CSR order (shuffle broadcast), so e_atom[i] = ((0 + eps_0) + eps_1) + ...
//              exactly as one thread walking the row would: bitwise repeatable, no atomics, each element written once.
//   k_zbl_bwd  one thread per edge: g_e = grad_e_atom[i] * d eps_e / dr * r_hat, accumulated into grad_pos with
//              fp64 atomics (grad_pos[j] += g_e, grad_pos[i] -= g_e, as nqb_edge_embed_bwd) and/or written to
//              grad_vec[e].
// Edges with x = r / r_max >= 1 (null edges of a padded list among them) return eps = 0 and d eps / dr = 0 before any
// exponential is evaluated, so they add exactly +0 to their row and nothing to the gradients.
// Per-edge-type cutoffs (kTyped, nqb_zbl_*_typed): the envelope takes x = r * recip[T * t_i + t_j]
// (pair_potential.py:374 reads the normalised length of EdgeLengthNormalizer); the ZBL physics keeps r.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/nqb.h"

extern "C" int nqb_set_error(const char* msg);  // defined in nqb_runtime.cu
extern "C" void nqb_count_launch(void);

namespace {

// LAMMPS pair_zbl_const.h (as restated in pair_potential.py:239-249)
constexpr double kA0 = 0.46850;
constexpr double kC1 = 0.02817, kC2 = 0.28022, kC3 = 0.50986, kC4 = 0.18175;
constexpr double kD1 = -0.20162, kD2 = -0.40290, kD3 = -0.94229, kD4 = -3.19980;

struct ZblGeom {
  const double* pos;      // [N,3] (NULL when vec is given)
  const int64_t* eidx;    // [2,E]: centre, neighbour (types always come from here)
  const double* shift;    // [E,3] or NULL
  const double* cell;     // [3,3] or NULL
  const double* vec;      // [E,3] given edge vectors or NULL
  int64_t E;
};

struct ZblParams {
  double r_max, p;
  int cutoff_f32;  // round f_c to float32 (float32 models: the reference casts the cutoff to the model dtype)
  int T;
};

// kFramed (nqb_zbl_*_frames): g.cell is [F, 3, 3] and edge e takes the cell of its centre's frame, frame[i0]
template <bool kFramed>
__device__ __forceinline__ void edge_vector(const ZblGeom& g, int64_t e, int64_t i0, int64_t i1,
                                            const int64_t* __restrict__ frame, double& vx, double& vy, double& vz) {
  if (g.vec != nullptr) {
    vx = g.vec[3 * e]; vy = g.vec[3 * e + 1]; vz = g.vec[3 * e + 2];
    return;
  }
  // the arithmetic of k_edge_embed_fwd: pos[j] - pos[i] + shift @ cell
  vx = g.pos[3 * i1] - g.pos[3 * i0];
  vy = g.pos[3 * i1 + 1] - g.pos[3 * i0 + 1];
  vz = g.pos[3 * i1 + 2] - g.pos[3 * i0 + 2];
  if (g.shift != nullptr && g.cell != nullptr) {
    const double s0 = g.shift[3 * e], s1 = g.shift[3 * e + 1], s2 = g.shift[3 * e + 2];
    const double* c = kFramed ? g.cell + 9 * frame[i0] : g.cell;
    vx += s0 * c[0] + s1 * c[3] + s2 * c[6];
    vy += s0 * c[1] + s1 * c[4] + s2 * c[7];
    vz += s0 * c[2] + s1 * c[5] + s2 * c[8];
  }
}

// eps and (when dedr != NULL) d eps / dr of one edge of length r; A, S from the type-pair table; recip = 1 / rc of the
// edge's type pair (read only when kTyped)
template <bool kTyped>
__device__ __forceinline__ double zbl_edge(double r, double A, double S, const ZblParams& q, double recip, double* dedr) {
  const double xc = kTyped ? r * recip : r * (1.0 / q.r_max);  // EdgeLengthNormalizer: r * (1 / r_max)
  if (!(xc < 1.0)) {
    if (dedr) *dedr = 0.0;
    return 0.0;
  }
  const double p = q.p;
  // PolynomialCutoff, in the reference's order of operations
  double fc = 1.0;
  fc = fc - ((p + 1.0) * (p + 2.0) / 2.0) * pow(xc, p);
  fc = fc + (p * (p + 2.0)) * pow(xc, p + 1.0);
  fc = fc - (p * (p + 1.0) / 2.0) * pow(xc, p + 2.0);
  if (q.cutoff_f32) fc = (double)(float)fc;
  const double x = (S * r) / kA0;
  const double e1 = exp(kD1 * x), e2 = exp(kD2 * x), e3 = exp(kD3 * x), e4 = exp(kD4 * x);
  const double psi = kC1 * e1 + kC2 * e2 + kC3 * e3 + kC4 * e4;
  const double inv_r = 1.0 / r;
  if (dedr) {
    const double dpsi = (kC1 * kD1 * e1 + kC2 * kD2 * e2 + kC3 * kD3 * e3 + kC4 * kD4 * e4) * (S / kA0);
    const double xpm1 = pow(xc, p - 1.0);
    const double dpoly = 0.5 * p * (p + 1.0) * (p + 2.0) * (-xpm1 + 2.0 * xpm1 * xc - xpm1 * xc * xc);
    const double dfc = kTyped ? dpoly * recip : dpoly / q.r_max;
    *dedr = A * inv_r * ((dpsi - psi * inv_r) * fc + psi * dfc);
  }
  return A * inv_r * psi * fc;
}

template <bool kTyped = false, bool kFramed = false>
__global__ void k_zbl_fwd(ZblGeom g, ZblParams q, const int64_t* __restrict__ types, const double* __restrict__ table,
                          const int64_t* __restrict__ row_ptr, const int64_t* __restrict__ perm, int64_t N,
                          double* __restrict__ e_atom, const double* __restrict__ recip,
                          const int64_t* __restrict__ frame) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= N) return;  // uniform over the warp
  const int64_t b = row_ptr[row], end = row_ptr[row + 1];
  const int64_t ti = types[row];
  double s = 0.0;
  for (int64_t base = b; base < end; base += 32) {
    const int64_t n = base + lane;
    double eps = 0.0;
    if (n < end) {
      const int64_t e = perm ? perm[n] : n;
      const int64_t i0 = g.eidx[e], i1 = g.eidx[g.E + e];
      double vx, vy, vz;
      edge_vector<kFramed>(g, e, i0, i1, frame, vx, vy, vz);
      const double r = sqrt(vx * vx + vy * vy + vz * vz);
      const int64_t tt = ti * q.T + types[i1];
      const double* t = table + 2 * tt;
      eps = zbl_edge<kTyped>(r, t[0], t[1], q, kTyped ? recip[tt] : 0.0, nullptr);
    }
    const int cnt = (int)min((int64_t)32, end - base);
    for (int k = 0; k < cnt; ++k) s += __shfl_sync(0xffffffffu, eps, k);  // CSR order
  }
  if (lane == 0) e_atom[row] = s;
}

template <bool kTyped = false, bool kFramed = false>
__global__ void k_zbl_bwd(ZblGeom g, ZblParams q, const int64_t* __restrict__ types, const double* __restrict__ table,
                          const double* __restrict__ grad_e, double* __restrict__ gpos, double* __restrict__ gvec,
                          const double* __restrict__ recip, const int64_t* __restrict__ frame) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g.E) return;
  const int64_t i0 = g.eidx[e], i1 = g.eidx[g.E + e];
  double vx, vy, vz;
  edge_vector<kFramed>(g, e, i0, i1, frame, vx, vy, vz);
  const double r = sqrt(vx * vx + vy * vy + vz * vz);
  const int64_t tt = types[i0] * q.T + types[i1];
  const double* t = table + 2 * tt;
  double dedr;
  zbl_edge<kTyped>(r, t[0], t[1], q, kTyped ? recip[tt] : 0.0, &dedr);
  const double c = dedr == 0.0 ? 0.0 : grad_e[i0] * dedr / r;
  const double gx = c * vx, gy = c * vy, gz = c * vz;
  if (gvec != nullptr) { gvec[3 * e] = gx; gvec[3 * e + 1] = gy; gvec[3 * e + 2] = gz; }
  if (gpos != nullptr) {
    atomicAdd(gpos + 3 * i1, gx); atomicAdd(gpos + 3 * i1 + 1, gy); atomicAdd(gpos + 3 * i1 + 2, gz);
    atomicAdd(gpos + 3 * i0, -gx); atomicAdd(gpos + 3 * i0 + 1, -gy); atomicAdd(gpos + 3 * i0 + 2, -gz);
  }
}

int check_common(const char* what, const double* pos, const int64_t* edge_index, const double* shift,
                 const double* cell, const double* vec, const int64_t* types, const double* table, int T,
                 int64_t N, int64_t E, double r_max, double poly_p) {
  static thread_local char msg[256];
  auto err = [&](const char* m) {
    snprintf(msg, sizeof(msg), "%s: %s", what, m);
    return nqb_set_error(msg);
  };
  if (N < 0 || E < 0) return err("negative size");
  if (T < 1) return err("need at least one type");
  if (!(r_max > 0.0) || !(poly_p >= 2.0)) return err("need r_max > 0 and p >= 2");
  // an empty shift array may come as NULL
  if (E > 0 && (shift == nullptr) != (cell == nullptr)) return err("shift and cell must come together");
  if (vec != nullptr && (pos != nullptr || shift != nullptr)) return err("give either vec or pos (+ shift, cell)");
  if (E > 0 && (!edge_index || (vec == nullptr && pos == nullptr))) return err("null edge_index / geometry");
  if (N > 0 && (!types || !table)) return err("null types / table");
  return 0;
}

}  // namespace

extern "C" int nqb_zbl_fwd(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                           const double* vec, const int64_t* types, const double* table, int T,
                           const int64_t* row_ptr, const int64_t* perm, int64_t N, int64_t E, double r_max,
                           double poly_p, int cutoff_f32, double* e_atom, nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_fwd", pos, edge_index, shift, cell, vec, types, table, T, N, E, r_max, poly_p))
    return rc;
  if (N == 0) return 0;
  if (!row_ptr || !e_atom) return nqb_set_error("nqb_zbl_fwd: null row_ptr / e_atom");
  ZblGeom g{pos, edge_index, shift, cell, vec, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((N + 3) / 4);  // 4 rows (warps) per 128-thread block
  k_zbl_fwd<<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, row_ptr, perm, N, e_atom, nullptr, nullptr);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_zbl_bwd(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                           const double* vec, const int64_t* types, const double* table, int T, int64_t N, int64_t E,
                           double r_max, double poly_p, int cutoff_f32, const double* grad_e_atom, double* grad_pos,
                           double* grad_vec, nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_bwd", pos, edge_index, shift, cell, vec, types, table, T, N, E, r_max, poly_p))
    return rc;
  if (grad_pos != nullptr && vec != nullptr) return nqb_set_error("nqb_zbl_bwd: grad_pos needs positions, not vec");
  if (E == 0) return 0;
  if (!grad_e_atom || (!grad_pos && !grad_vec)) return nqb_set_error("nqb_zbl_bwd: null grad_e_atom / outputs");
  ZblGeom g{pos, edge_index, shift, cell, vec, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((E + 127) / 128);
  k_zbl_bwd<<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, grad_e_atom, grad_pos, grad_vec, nullptr, nullptr);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Per-edge-type cutoffs: as above, with the envelope at x = r * recip[T * t_i + t_j] (recip [T * T] f64, device).
extern "C" int nqb_zbl_fwd_typed(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                                 const double* vec, const int64_t* types, const double* table, int T,
                                 const int64_t* row_ptr, const int64_t* perm, int64_t N, int64_t E, double r_max,
                                 double poly_p, int cutoff_f32, const double* recip, double* e_atom, nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_fwd_typed", pos, edge_index, shift, cell, vec, types, table, T, N, E, r_max,
                            poly_p))
    return rc;
  if (N == 0) return 0;
  if (!row_ptr || !e_atom) return nqb_set_error("nqb_zbl_fwd_typed: null row_ptr / e_atom");
  if (!recip) return nqb_set_error("nqb_zbl_fwd_typed: null recip");
  ZblGeom g{pos, edge_index, shift, cell, vec, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((N + 3) / 4);
  k_zbl_fwd<true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, row_ptr, perm, N, e_atom, recip, nullptr);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_zbl_bwd_typed(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                                 const double* vec, const int64_t* types, const double* table, int T, int64_t N,
                                 int64_t E, double r_max, double poly_p, int cutoff_f32, const double* recip,
                                 const double* grad_e_atom, double* grad_pos, double* grad_vec, nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_bwd_typed", pos, edge_index, shift, cell, vec, types, table, T, N, E, r_max,
                            poly_p))
    return rc;
  if (grad_pos != nullptr && vec != nullptr) return nqb_set_error("nqb_zbl_bwd_typed: grad_pos needs positions, not vec");
  if (E == 0) return 0;
  if (!grad_e_atom || (!grad_pos && !grad_vec)) return nqb_set_error("nqb_zbl_bwd_typed: null grad_e_atom / outputs");
  if (!recip) return nqb_set_error("nqb_zbl_bwd_typed: null recip");
  ZblGeom g{pos, edge_index, shift, cell, vec, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((E + 127) / 128);
  k_zbl_bwd<true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, grad_e_atom, grad_pos, grad_vec, recip, nullptr);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// A batch of frames: as nqb_zbl_fwd / nqb_zbl_bwd on positions with cells [F, 3, 3] (device) and frame [N] i64 (the
// frame of each atom); edge e takes the cell of frame[edge_index[0][e]].  Per-edge-type cutoffs when recip is given
// (as nqb_zbl_*_typed), none when it is NULL.
extern "C" int nqb_zbl_fwd_frames(const double* pos, const int64_t* edge_index, const double* shift,
                                  const double* cells, const int64_t* frame, const int64_t* types, const double* table,
                                  int T, const int64_t* row_ptr, const int64_t* perm, int64_t N, int64_t E,
                                  double r_max, double poly_p, int cutoff_f32, const double* recip, double* e_atom,
                                  nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_fwd_frames", pos, edge_index, shift, cells, nullptr, types, table, T, N, E, r_max,
                            poly_p))
    return rc;
  if (N == 0) return 0;
  if (!row_ptr || !e_atom) return nqb_set_error("nqb_zbl_fwd_frames: null row_ptr / e_atom");
  if (E > 0 && (!shift || !frame)) return nqb_set_error("nqb_zbl_fwd_frames: null shift / cells / frame");
  ZblGeom g{pos, edge_index, shift, cells, nullptr, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((N + 3) / 4);
  if (recip)
    k_zbl_fwd<true, true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, row_ptr, perm, N, e_atom, recip,
                                                                 frame);
  else
    k_zbl_fwd<false, true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, row_ptr, perm, N, e_atom, recip,
                                                                  frame);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_zbl_bwd_frames(const double* pos, const int64_t* edge_index, const double* shift,
                                  const double* cells, const int64_t* frame, const int64_t* types, const double* table,
                                  int T, int64_t N, int64_t E, double r_max, double poly_p, int cutoff_f32,
                                  const double* recip, const double* grad_e_atom, double* grad_pos, double* grad_vec,
                                  nqb_stream_t st) {
  if (int rc = check_common("nqb_zbl_bwd_frames", pos, edge_index, shift, cells, nullptr, types, table, T, N, E, r_max,
                            poly_p))
    return rc;
  if (E == 0) return 0;
  if (!grad_e_atom || (!grad_pos && !grad_vec)) return nqb_set_error("nqb_zbl_bwd_frames: null grad_e_atom / outputs");
  if (!shift || !frame) return nqb_set_error("nqb_zbl_bwd_frames: null shift / cells / frame");
  ZblGeom g{pos, edge_index, shift, cells, nullptr, E};
  ZblParams q{r_max, poly_p, cutoff_f32 ? 1 : 0, T};
  const unsigned blocks = (unsigned)((E + 127) / 128);
  if (recip)
    k_zbl_bwd<true, true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, grad_e_atom, grad_pos, grad_vec,
                                                                 recip, frame);
  else
    k_zbl_bwd<false, true><<<blocks, 128, 0, (cudaStream_t)st>>>(g, q, types, table, grad_e_atom, grad_pos, grad_vec,
                                                                  recip, frame);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}
