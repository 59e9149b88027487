// Velocity Verlet with the reference's Nose-Hoover thermostat (nequip/ase/nosehoover.py, NoseHoover.step), restated
// per frame f of a batch, in float64, sm_90a.  One MD step of nequip_b200/md.py (GraphedMD) is
//   nqb_md_kick_drift -> nqb_md_bath -> neighbour list + model -> nqb_md_kick -> nqb_md_log
// captured as one CUDA graph.  The atoms of frame f are the contiguous range [atom_ptr[f], atom_ptr[f+1]) (batch is
// non-decreasing, as in nqb_nl_bbox_frames); every kernel that touches atoms runs a grid of (nblk, F) CTAs of
// kMdThreads threads, CTA (b, f) visiting atoms atom_ptr[f] + b * kMdThreads + t + k * nblk * kMdThreads.
//
// Sums over atoms never use floating-point atomics: each CTA reduces its atoms with a fixed shuffle tree and a fixed
// order over warps into its own slot of a [F, nblk] workspace, and the consumer adds the nblk slots in index order.
// For a given launch shape the result is therefore a function of the inputs alone, so a block of steps that is
// rolled back and run again reproduces itself given the same forces.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/nqb.h"

extern "C" int nqb_set_error(const char* msg);
extern "C" void nqb_count_launch(void);

namespace {

constexpr int kMdThreads = 256;

// the CTA's sum of v (every thread passes its partial), valid in thread 0; fixed order
__device__ __forceinline__ double cta_sum(double v, double* smem) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kMdThreads / 32; ++w) s += smem[w];
  __syncthreads();
  return s;
}

__device__ __forceinline__ double msq(double m, double x, double y, double z) { return m * (x * x + y * y + z * z); }

// a = F/m - zeta v;  x += dt v + dt^2/2 a;  v <- v + dt/2 a;  part[f, b] = {sum m v^2, sum m v_h^2} of the CTA
__global__ void __launch_bounds__(kMdThreads)
k_md_kick_drift(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ forces,
                const double* __restrict__ zeta, double dt, double* __restrict__ pos, double* __restrict__ vel,
                double* __restrict__ part) {
  __shared__ double smem[kMdThreads / 32];
  const int f = blockIdx.y, nblk = gridDim.x;
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  const double z = zeta[f], hdt = 0.5 * dt, hdt2 = 0.5 * dt * dt;
  double s0 = 0.0, s1 = 0.0;
  for (int64_t i = beg + (int64_t)blockIdx.x * kMdThreads + threadIdx.x; i < end; i += (int64_t)nblk * kMdThreads) {
    const double m = mass[i];
    double v[3], a[3];
    for (int d = 0; d < 3; ++d) {
      v[d] = vel[3 * i + d];
      a[d] = forces[3 * i + d] / m - z * v[d];
    }
    s0 += msq(m, v[0], v[1], v[2]);
    for (int d = 0; d < 3; ++d) {
      pos[3 * i + d] = pos[3 * i + d] + dt * v[d] + hdt2 * a[d];
      v[d] = v[d] + hdt * a[d];
      vel[3 * i + d] = v[d];
    }
    s1 += msq(m, v[0], v[1], v[2]);
  }
  s0 = cta_sum(s0, smem);
  s1 = cta_sum(s1, smem);
  if (threadIdx.x == 0) {
    part[2 * ((int64_t)f * nblk + blockIdx.x)] = s0;
    part[2 * ((int64_t)f * nblk + blockIdx.x) + 1] = s1;
  }
}

// zeta_h = zeta + dt/2 (sum m v^2 - gkT) / (2Q);  zeta' = zeta_h + dt/2 (sum m v_h^2 - gkT) / (2Q);
// eta += dt/2 (zeta + zeta')  (trapezoid).  One thread per frame.
__global__ void k_md_bath(int F, int nblk, const double* __restrict__ part, const double* __restrict__ gkT,
                          const double* __restrict__ Q, double dt, double* __restrict__ zeta, double* __restrict__ eta) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double s0 = 0.0, s1 = 0.0;
  for (int b = 0; b < nblk; ++b) {
    s0 += part[2 * ((int64_t)f * nblk + b)];
    s1 += part[2 * ((int64_t)f * nblk + b) + 1];
  }
  const double hdt = 0.5 * dt, z = zeta[f];
  const double zh = z + hdt * (0.5 * (s0 - gkT[f])) / Q[f];
  const double zn = zh + hdt * (0.5 * (s1 - gkT[f])) / Q[f];
  eta[f] = eta[f] + hdt * (z + zn);
  zeta[f] = zn;
}

// v = (v_h + dt/2 F/m) / (1 + dt/2 zeta');  forces <- F;  ke_part[f, b] = sum m v^2 of the CTA
__global__ void __launch_bounds__(kMdThreads)
k_md_kick(const int64_t* __restrict__ atom_ptr, const double* __restrict__ mass, const double* __restrict__ f_new,
          const double* __restrict__ zeta, double dt, double* __restrict__ vel, double* __restrict__ forces,
          double* __restrict__ ke_part) {
  __shared__ double smem[kMdThreads / 32];
  const int f = blockIdx.y, nblk = gridDim.x;
  const int64_t beg = atom_ptr[f], end = atom_ptr[f + 1];
  const double hdt = 0.5 * dt, den = 1.0 + hdt * zeta[f];
  double s = 0.0;
  for (int64_t i = beg + (int64_t)blockIdx.x * kMdThreads + threadIdx.x; i < end; i += (int64_t)nblk * kMdThreads) {
    const double m = mass[i];
    double v[3];
    for (int d = 0; d < 3; ++d) {
      const double fd = f_new[3 * i + d];
      v[d] = (vel[3 * i + d] + hdt * (fd / m)) / den;
      vel[3 * i + d] = v[d];
      forces[3 * i + d] = fd;
    }
    s += msq(m, v[0], v[1], v[2]);
  }
  s = cta_sum(s, smem);
  if (threadIdx.x == 0) ke_part[(int64_t)f * nblk + blockIdx.x] = s;
}

// One CTA.  Row step % rows of the log, per frame: E_pot, E_kin, T, zeta, eta, H; the sticky flags; then step += 1.
__global__ void __launch_bounds__(kMdThreads)
k_md_log(int F, int nblk, const double* __restrict__ e_pot, const double* __restrict__ ke_part,
         const double* __restrict__ zeta, const double* __restrict__ eta, const double* __restrict__ Q,
         const double* __restrict__ gkT, const double* __restrict__ dof_kB, const int64_t* __restrict__ num_edges,
         const int32_t* __restrict__ overflow, const int32_t* __restrict__ sorted, int64_t rows, int64_t* step,
         double* __restrict__ log, int64_t* __restrict__ flags) {
  const int64_t s = *step;
  double* row = log + (s % rows) * (int64_t)F * NQB_MD_LOG_FIELDS;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    double ke = 0.0;
    for (int b = 0; b < nblk; ++b) ke += ke_part[(int64_t)f * nblk + b];
    ke *= 0.5;
    const double z = zeta[f], h = eta[f], ep = e_pot[f];
    double* r = row + (int64_t)f * NQB_MD_LOG_FIELDS;
    r[0] = ep;
    r[1] = ke;
    r[2] = 2.0 * ke / dof_kB[f];
    r[3] = z;
    r[4] = h;
    r[5] = ep + ke + Q[f] * z * z + gkT[f] * h;
  }
  __syncthreads();  // every thread has read *step
  if (threadIdx.x == 0) {
    const int32_t ov = *overflow != 0;
    if (ov) {
      flags[0] = 1;
      if (flags[2] < 0) flags[2] = s;
    }
    if (*sorted != 1) flags[1] = 1;
    if (*num_edges > flags[3]) flags[3] = *num_edges;
    *step = s + 1;
  }
}

int md_launch_done() {
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

}  // namespace

extern "C" int nqb_md_kick_drift(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* forces,
                                 const double* zeta, double dt, double* pos, double* vel, double* part,
                                 nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_md_kick_drift: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (!atom_ptr || !mass || !forces || !zeta || !pos || !vel || !part)
    return nqb_set_error("nqb_md_kick_drift: null pointer");
  if (F > 65535) return nqb_set_error("nqb_md_kick_drift: at most 65535 frames");
  k_md_kick_drift<<<dim3((unsigned)nblk, (unsigned)F), kMdThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, forces, zeta,
                                                                                         dt, pos, vel, part);
  return md_launch_done();
}

extern "C" int nqb_md_bath(int F, int nblk, const double* part, const double* gkT, const double* Q, double dt,
                           double* zeta, double* eta, nqb_stream_t st) {
  if (F < 0 || nblk < 1) return nqb_set_error("nqb_md_bath: needs F >= 0 and nblk >= 1");
  if (F == 0) return 0;
  if (!part || !gkT || !Q || !zeta || !eta) return nqb_set_error("nqb_md_bath: null pointer");
  k_md_bath<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, nblk, part, gkT, Q, dt, zeta, eta);
  return md_launch_done();
}

extern "C" int nqb_md_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new,
                           const double* zeta, double dt, double* vel, double* forces, double* ke_part,
                           nqb_stream_t st) {
  if (F < 0 || nblk < 1 || nblk > 65535) return nqb_set_error("nqb_md_kick: needs F >= 0 and 1 <= nblk <= 65535");
  if (F == 0) return 0;
  if (!atom_ptr || !mass || !f_new || !zeta || !vel || !forces || !ke_part)
    return nqb_set_error("nqb_md_kick: null pointer");
  if (F > 65535) return nqb_set_error("nqb_md_kick: at most 65535 frames");
  k_md_kick<<<dim3((unsigned)nblk, (unsigned)F), kMdThreads, 0, (cudaStream_t)st>>>(atom_ptr, mass, f_new, zeta, dt,
                                                                                   vel, forces, ke_part);
  return md_launch_done();
}

extern "C" int nqb_md_log(int F, int nblk, const double* e_pot, const double* ke_part, const double* zeta,
                          const double* eta, const double* Q, const double* gkT, const double* dof_kB,
                          const int64_t* num_edges, const int32_t* overflow, const int32_t* sorted, int64_t rows,
                          int64_t* step, double* log, int64_t* flags, nqb_stream_t st) {
  if (F < 0 || nblk < 1 || rows < 1) return nqb_set_error("nqb_md_log: needs F >= 0, nblk >= 1 and rows >= 1");
  if (!e_pot || !ke_part || !zeta || !eta || !Q || !gkT || !dof_kB || !num_edges || !overflow || !sorted || !step ||
      !log || !flags)
    return nqb_set_error("nqb_md_log: null pointer");
  k_md_log<<<1, kMdThreads, 0, (cudaStream_t)st>>>(F, nblk, e_pot, ke_part, zeta, eta, Q, gkT, dof_kB, num_edges,
                                                  overflow, sorted, rows, step, log, flags);
  return md_launch_done();
}
