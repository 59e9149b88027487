// Fused radial-MLP last layer -> tensor product -> scatter, forward (sm_90a).   SURVEY.md section 8(f)-1.
//
// Reference ops fused here:
//   edge_weight = h @ (W2 * alpha2)                      nequip/nn/mlp.py:262-268 (last ScalarLinearLayer of
//                                                         the radial MLP, built at interaction_block.py:119-127)
//   out = scatter(tp(x[src], edge_attr, edge_weight))     nequip/nn/_tp_scatter_base.py:35-38,
//                                                         nequip/nn/interaction_block.py:193-199
// so that the [E, W] edge-weight tensor never leaves the SM in an inference-only forward.
//
// Decomposition: PATH-parallel.  The W columns (path p, channel u) are cut into slices of 128 rows; a CTA owns ONE
// slice for a contiguous node range and keeps the slice's second-layer weights W2^T[128 (p,u), K <= 128] (tf32 hi
// and lo parts, 128 KB) RESIDENT in shared memory as the wgmma A operand for its whole life.  Per destination node
// (<= 64 edges per tile) it stages the node's h rows (fp32 = tf32 high operand, plus their low parts) and computes
//   D^T[(p,u), e] = sum_k W2^T[(p,u), k] * h[e, k]          (wgmma m64n64k8 tf32, 3xTF32 split, fp32 accumulators)
// Warpgroup g issues the MMAs of rows 64 g .. 64 g + 63, so the weights arrive in its registers in the accumulator
// fragment layout: thread = rows r, r + 8 (two channels of one path: paths are whole 32-channel blocks) x edge columns
// 8 j + 2 (lane % 4) + {0, 1}.  That is the thread mapping of the tensor-product arithmetic: each thread contracts
// its edge PAIRS (x = {x[src_e0], x[src_e1]}, w = adjacent accumulator columns) into per-channel float2 sums held in
// registers across the node's tiles; at the end of the node the four lanes that share a row add their sums in a fixed
// order (deterministic, no atomics) and one writes the output element.  Padded edges have weight exactly 0 (their h
// rows are zero-filled) and finite operands.
//
// CTA = 2 warpgroups (256 threads), one CTA per SM (about 192 KB of shared memory); h tiles are staged by all
// threads with 16-byte cp.async into the canonical K-major core-matrix layout.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "nqb_tc.cuh"

namespace {

constexpr int FT_TE = 64;                        // max edges per tile = wgmma N
constexpr int FT_KMAX = 128;                     // resident K (hidden width of the radial MLP)
constexpr int FT_ROWS = 128;                     // (path, channel) rows per slice
constexpr int FT_THREADS = 256;
constexpr int FT_N3MAX = 7;                      // output components of a path (l <= 3)

struct FusedFwdArgs {
  const float* x;        // [N, D_IN]  ir_mul layout
  const float* y;        // [E, S]
  const float* h;        // [E, ldh]   hidden activations of the radial MLP
  const float* wprep;    // [NSLICE][hi|lo][128 x FT_KMAX] canonical core-matrix order (ops.FusedTPWeights.prepare)
  const int64_t* row_ptr;
  const int64_t* src;
  float* out;            // [N, D_OUT]
  float* w_out;          // [E, W] or nullptr: the per-edge weights in instruction order (for an unfused backward)
  const int32_t* slice_cta0;  // [NSLICE + 1]: CTAs [cta0[s], cta0[s+1]) work on slice s
  int64_t N, E, ldh;
  int K;                 // hidden width, multiple of 8, <= FT_KMAX
};

struct FtSmem {
  float w[2][FT_ROWS * FT_KMAX];   // W2^T hi, lo
  float hraw[FT_TE * FT_KMAX];     // h tile (the fp32 values are the tf32 high operand: the tensor core truncates)
  float hlo[FT_TE * FT_KMAX];      // its tf32 low parts
  int slice, pad_;
  int64_t n0, n1;
};

// first n in [0, N] with row_ptr[n] >= t
__device__ __forceinline__ int64_t ft_lower_bound(const int64_t* __restrict__ row_ptr, int64_t N, int64_t t) {
  int64_t lo = 0, hi = N;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (row_ptr[mid] < t) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct FtNullPath {
  static constexpr bool ACTIVE = false;
  static constexpr int N1 = 1, N2 = 1, N3 = 0, XG_OFF = 0, Y_OFF = 0, W_OFF = 0, MUL = 32;
  static __device__ __forceinline__ void fma(const float2*, const float2*, float2, float2*) {}
  static __device__ __forceinline__ void store(float*, int, const float*) {}
  static __device__ __forceinline__ void store_zero(float*, int) {}
};

// ---------------------------------------------------------------------------------------------------------
// per-path pieces.  PathP (generated): N1/N2/N3 (= 2l+1), XG_OFF (float offset of the input chunk in an x row),
// Y_OFF, W_OFF, MUL, and  fma(x[N1], y[N2], w, acc[N3]) on edge pairs,  store(out_row, u, v),  store_zero(out_row, u)
// ---------------------------------------------------------------------------------------------------------
// one tile: this thread's edge pairs for channels u0 and u0 + 8 (accumulator rows r, r + 8)
template <class P, class Spec>
__device__ __forceinline__ void ft_tile(const FusedFwdArgs& a, int64_t t0, int cnt, int q, int u0, const float* hh,
                                        const float* xx, float2 (&acc)[2][FT_N3MAX]) {
  if constexpr (P::ACTIVE) {
#pragma unroll
    for (int j = 0; j < FT_TE / 8; ++j) {
      const int c = 8 * j + 2 * q;
      if (c < cnt) {
        // past the node's last edge the second edge of the pair repeats the first: its weights are exactly 0
        const int64_t e0 = t0 + c, e1 = (c + 1 < cnt) ? e0 + 1 : e0;
        const float2 w0 = make_float2(hh[4 * j] + xx[4 * j], hh[4 * j + 1] + xx[4 * j + 1]);
        const float2 w1 = make_float2(hh[4 * j + 2] + xx[4 * j + 2], hh[4 * j + 3] + xx[4 * j + 3]);
        const float* x0 = a.x + __ldg(a.src + e0) * Spec::D_IN + P::XG_OFF + u0;
        const float* x1 = a.x + __ldg(a.src + e1) * Spec::D_IN + P::XG_OFF + u0;
        const float* y0 = a.y + e0 * Spec::S + P::Y_OFF;
        const float* y1 = a.y + e1 * Spec::S + P::Y_OFF;
        float2 xa[P::N1], xb[P::N1], ya[P::N2];
#pragma unroll
        for (int i = 0; i < P::N1; ++i) {
          xa[i] = make_float2(__ldg(x0 + i * P::MUL), __ldg(x1 + i * P::MUL));
          xb[i] = make_float2(__ldg(x0 + i * P::MUL + 8), __ldg(x1 + i * P::MUL + 8));
        }
#pragma unroll
        for (int i = 0; i < P::N2; ++i) ya[i] = make_float2(__ldg(y0 + i), __ldg(y1 + i));
        P::fma(xa, ya, w0, acc[0]);
        P::fma(xb, ya, w1, acc[1]);
        if (a.w_out != nullptr) {
          float* wo = a.w_out + e0 * (int64_t)Spec::W + P::W_OFF + u0;
          wo[0] = w0.x;
          wo[8] = w1.x;
          if (c + 1 < cnt) { wo[Spec::W] = w0.y; wo[Spec::W + 8] = w1.y; }
        }
      }
    }
  }
}

// end of a node: the four lanes of a row add their sums (fixed order), lane q == 0 writes both channels
template <class P>
__device__ __forceinline__ void ft_finish(float* o, int q, int u0, float2 (&acc)[2][FT_N3MAX]) {
  if constexpr (P::ACTIVE) {
    float v0[P::N3], v1[P::N3];
#pragma unroll
    for (int k = 0; k < P::N3; ++k) {
      v0[k] = acc[0][k].x + acc[0][k].y;
      v1[k] = acc[1][k].x + acc[1][k].y;
      v0[k] += __shfl_xor_sync(0xffffffffu, v0[k], 1);
      v1[k] += __shfl_xor_sync(0xffffffffu, v1[k], 1);
      v0[k] += __shfl_xor_sync(0xffffffffu, v0[k], 2);
      v1[k] += __shfl_xor_sync(0xffffffffu, v1[k], 2);
    }
    if (q == 0) {
      P::store(o, u0, v0);
      P::store(o, u0 + 8, v1);
    }
  }
#pragma unroll
  for (int k = 0; k < FT_N3MAX; ++k) { acc[0][k] = make_float2(0.f, 0.f); acc[1][k] = make_float2(0.f, 0.f); }
}

// the per-path steps, called through Spec::dispatch<Op>(slice, block, args...) as Op::run<PathT>(first channel of the
// warp's 16-row block, args...)
struct FtZeroOp {
  template <class P>
  static __device__ __forceinline__ void run(int ub, float* const& orow, const int& lane) {
    if ((lane & 3) == 0) { P::store_zero(orow, ub + (lane >> 2)); P::store_zero(orow, ub + (lane >> 2) + 8); }
  }
};
template <class Spec>
struct FtTileOp {
  template <class P>
  static __device__ __forceinline__ void run(int ub, const FusedFwdArgs& a, const int64_t& t0, const int& cnt,
                                             const int& lane, float (&hh)[32], float (&xx)[32], float2 (&acc)[2][FT_N3MAX]) {
    ft_tile<P, Spec>(a, t0, cnt, lane & 3, ub + (lane >> 2), hh, xx, acc);
  }
};
struct FtFinishOp {
  template <class P>
  static __device__ __forceinline__ void run(int ub, float* const& orow, const int& lane, float2 (&acc)[2][FT_N3MAX]) {
    ft_finish<P>(orow, lane & 3, ub + (lane >> 2), acc);
  }
};

// ---------------------------------------------------------------------------------------------------------
// the kernel.  Spec (generated): S, D_IN, D_OUT, W, NSLICE, and dispatch<Op>(slice, block, args...) for the path that
// owns rows 16 block .. 16 block + 15 of the slice.
// The MMAs and barriers are outside the per-path code: every thread of a warpgroup runs the same instructions.
// ---------------------------------------------------------------------------------------------------------
template <class Spec>
__global__ void __launch_bounds__(FT_THREADS, 1) tp_fused_fwd_kernel(const FusedFwdArgs a) {
  extern __shared__ __align__(1024) uint8_t ft_smem_raw[];
  FtSmem& S = *reinterpret_cast<FtSmem*>(ft_smem_raw);
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;

  if (tid == 0) {
    int s = 0;
    while (s + 1 < Spec::NSLICE && (int)blockIdx.x >= a.slice_cta0[s + 1]) ++s;
    const int j = (int)blockIdx.x - a.slice_cta0[s], ns = a.slice_cta0[s + 1] - a.slice_cta0[s];
    S.slice = s;
    const int64_t t_lo = (a.E * (int64_t)j) / ns, t_hi = (a.E * (int64_t)(j + 1)) / ns;
    S.n0 = (j == 0) ? 0 : ft_lower_bound(a.row_ptr, a.N, t_lo);
    S.n1 = (j + 1 == ns) ? a.N : ft_lower_bound(a.row_ptr, a.N, t_hi);
  }
  __syncthreads();
  const int slice = S.slice;
  const int64_t n0 = S.n0, n1 = S.n1;
  {  // the slice's weights, once (waited for with the first h tile)
    const float4* src = reinterpret_cast<const float4*>(a.wprep + (int64_t)slice * 2 * FT_ROWS * FT_KMAX);
    float4* dst = reinterpret_cast<float4*>(&S.w[0][0]);
    for (int i = tid; i < 2 * FT_ROWS * FT_KMAX / 4; i += FT_THREADS) cp_async16(dst + i, src + i, 16u);
    cp_async_commit();
  }
  const int ksteps = a.K / 8;
  // h staging: thread -> rows 8 i + r8 (i < 8), k-group kg; a quarter warp writes one 128-byte core matrix
  const int r8 = tid & 7, kg = tid >> 3;
  const bool kin = kg < a.K / 4;  // k-groups beyond K are never read by the MMAs
  const int my_off = kg * 32 + r8 * 4;
  constexpr uint32_t LBO = 128, SBO = (FT_KMAX / 4) * 128;
  const uint32_t wg_rows = (uint32_t)wg * (64 / 8) * SBO;  // byte offset of row 64 wg in a weight block
  const uint64_t dWhi = make_desc(smem_u32(S.w[0]) + wg_rows, LBO, SBO);
  const uint64_t dWlo = make_desc(smem_u32(S.w[1]) + wg_rows, LBO, SBO);
  const uint64_t dH = make_desc(smem_u32(S.hraw), LBO, SBO);
  const uint64_t dL = make_desc(smem_u32(S.hlo), LBO, SBO);
  const int block = wg * 4 + warp;  // this warp's 16 rows of the slice
  float2 acc[2][FT_N3MAX];
#pragma unroll
  for (int k = 0; k < FT_N3MAX; ++k) { acc[0][k] = make_float2(0.f, 0.f); acc[1][k] = make_float2(0.f, 0.f); }
  float hh[32], xx[32];

  for (int64_t n = n0; n < n1; ++n) {
    const int64_t beg = a.row_ptr[n], end = a.row_ptr[n + 1];
    float* orow = a.out + n * Spec::D_OUT;
    if (beg == end) {
      Spec::template dispatch<FtZeroOp>(slice, block, orow, lane);
      continue;
    }
    for (int64_t t0 = beg; t0 < end; t0 += FT_TE) {
      const int cnt = (int)((end - t0 < FT_TE) ? (end - t0) : FT_TE);
      __syncthreads();  // both warpgroups' MMAs of the previous tile have completed: h may be overwritten
      if (kin) {
#pragma unroll
        for (int i = 0; i < FT_TE / 8; ++i) {
          const int row = 8 * i + r8;
          const bool in = row < cnt;
          cp_async16(S.hraw + i * (FT_KMAX / 4 * 32) + my_off, in ? a.h + (t0 + row) * a.ldh + kg * 4 : a.h, in ? 16u : 0u);
        }
      }
      cp_async_commit();
      cp_async_wait<0>();
      if (kin) {
#pragma unroll
        for (int i = 0; i < FT_TE / 8; ++i) {
          const float4 t = *reinterpret_cast<const float4*>(S.hraw + i * (FT_KMAX / 4 * 32) + my_off);
          *reinterpret_cast<float4*>(S.hlo + i * (FT_KMAX / 4 * 32) + my_off) =
              make_float4(tf32_lo(t.x), tf32_lo(t.y), tf32_lo(t.z), tf32_lo(t.w));
        }
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor core
      __syncthreads();
      wgmma_fence();
      // k-step advance = 2 core matrices = 256 bytes = 16 descriptor units
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) wgmma_tf32_m64n64(hh, dWhi + ks * 16, dH + ks * 16, ks > 0);
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) wgmma_tf32_m64n64(xx, dWlo + ks * 16, dH + ks * 16, ks > 0);
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) wgmma_tf32_m64n64(xx, dWhi + ks * 16, dL + ks * 16, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      Spec::template dispatch<FtTileOp<Spec>>(slice, block, a, t0, cnt, lane, hh, xx, acc);
    }
    Spec::template dispatch<FtFinishOp>(slice, block, orow, lane, acc);
  }
  cp_async_wait<0>();
}

template <class Spec>
inline size_t ft_smem_bytes() {
  return sizeof(FtSmem) + 1024;
}

}  // namespace
