// Radial-MLP hidden layer (K = 8) on CUDA cores, sm_90a.
//
// Reference op (paths under /root/reference):
//   edge_weight = ScalarMLPFunction(edge_embedding)            nequip/nn/mlp.py:80-195, 262-268
//   built with depth 1 by InteractionBlock                     nequip/nn/interaction_block.py:119-127, 196
//     h   = silu(emb @ (W1 * a1))          [E, NB] x [NB, H]   (NB = 8 Bessel functions, H = 128)   <- here
//     w   =      h   @ (W2 * a2)           [E, H ] x [H, W]    nqb_gemm.cu (unfused) / the fused TP kernels
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nqb.h"
#include "nqb_tc.cuh"

namespace {

constexpr int H = 128;       // hidden width == K of the second-layer GEMM
constexpr int NB = 8;        // Bessel functions

// ---------------------------------------------------------------------------------------------
// first radial layer on CUDA cores (K = 8): h = silu(emb @ W1s)  and its backward
//   gemb[e, k] = sum_m gh[e, m] * silu'(pre[e, m]) * W1s[k, m],  pre recomputed from emb
// (feeds / follows the grouped tensor-core GEMM of the second layer, nqb_gemm.cu)
//   * lane = 4 hidden units whose 8 x 4 first-layer weights live in registers for the whole kernel;
//   * a warp owns a BATCH of 32 consecutive edges; lane j fetches edge j's 8 basis values with two
//     coalesced 16-byte loads (1 KB per warp) and the batch after that is already in flight while the
//     current one is computed; inside the batch the values of edge j are broadcast with warp shuffles,
//     so no load sits on the critical path of an edge;
//   * float2 arithmetic on two hidden units at a time, sigmoid from ex2.approx / rcp.approx;
//   * backward: four edges per inner iteration -- their four grad_h rows are loaded up front and the
//     4 x 8 partial sums are reduced with one 32-value halving butterfly (31 shuffles) that leaves
//     element `lane` in lane `lane`: grad_emb is written as one 128-byte row.
// ---------------------------------------------------------------------------------------------
struct Basis8 { float4 a, b; };
__device__ __forceinline__ Basis8 load_basis(const float* __restrict__ emb, int64_t e, int64_t E) {
  Basis8 r;
  if (e < E) {
    r.a = __ldg(reinterpret_cast<const float4*>(emb + e * NB));
    r.b = __ldg(reinterpret_cast<const float4*>(emb + e * NB + 4));
  } else {
    r.a = make_float4(0.f, 0.f, 0.f, 0.f);
    r.b = r.a;
  }
  return r;
}
// the basis values of slot u < n: edge u itself, or with ROWS the edge rows[2 u]
template <bool ROWS>
__device__ __forceinline__ Basis8 load_slot(const float* __restrict__ emb, const int64_t* __restrict__ rows, int64_t u,
                                            int64_t n) {
  if constexpr (ROWS) {
    const int64_t e = u < n ? __ldg(rows + 2 * u) : 0;
    return load_basis(emb, e, u < n ? e + 1 : 0);
  } else {
    return load_basis(emb, u, n);
  }
}
// the 8 basis values of the batch's edge j (held by lane j), broadcast to every lane
__device__ __forceinline__ void bcast_basis(const Basis8& mine, int j, float (&x)[NB]) {
  x[0] = __shfl_sync(0xffffffffu, mine.a.x, j); x[1] = __shfl_sync(0xffffffffu, mine.a.y, j);
  x[2] = __shfl_sync(0xffffffffu, mine.a.z, j); x[3] = __shfl_sync(0xffffffffu, mine.a.w, j);
  x[4] = __shfl_sync(0xffffffffu, mine.b.x, j); x[5] = __shfl_sync(0xffffffffu, mine.b.y, j);
  x[6] = __shfl_sync(0xffffffffu, mine.b.z, j); x[7] = __shfl_sync(0xffffffffu, mine.b.w, j);
}
// pre-activations of this lane's 4 hidden units: p[q] = sum_k x[k] * W1s[k, m0 + q]  (k ascending)
__device__ __forceinline__ void preact4(const float (&x)[NB], const float2 (&w01)[NB], const float2 (&w23)[NB],
                                        float2& p01, float2& p23) {
  p01 = make_float2(0.f, 0.f);
  p23 = p01;
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    const float2 xx = make_float2(x[k], x[k]);
    p01 = fma2_rn(xx, w01[k], p01);
    p23 = fma2_rn(xx, w23[k], p23);
  }
}

// ROWS = true: h[u] = silu(emb[rows[2 u]] @ W1s) for u < min(E, *count) (the representative edges of the slots of
// nqb_edge_pairs); the grid is sized for E
template <bool ROWS = false>
__global__ void __launch_bounds__(256) k_hidden_fwd(const float* __restrict__ emb, const float* __restrict__ W1s,
                                                    int64_t E, float* __restrict__ h,
                                                    const int64_t* __restrict__ rows = nullptr,
                                                    const int64_t* __restrict__ count = nullptr) {
  const int lane = threadIdx.x & 31, m0 = lane * 4;
  if constexpr (ROWS) E = min(E, *count);
  float2 w01[NB], w23[NB];
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(W1s + k * H + m0));
    w01[k] = make_float2(t.x, t.y);
    w23[k] = make_float2(t.z, t.w);
  }
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t nbatch = (E + 31) >> 5;
  int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  Basis8 cur = load_slot<ROWS>(emb, rows, b * 32 + lane, b < nbatch ? E : 0);
  for (; b < nbatch; b += nwarps) {
    const int64_t bn = b + nwarps;
    const Basis8 nxt = load_slot<ROWS>(emb, rows, bn * 32 + lane, bn < nbatch ? E : 0);  // in flight during this batch
    const int64_t e0 = b * 32;
    const int cnt = (int)((E - e0) < 32 ? (E - e0) : 32);  // warp-uniform
    float* hrow = h + e0 * H + m0;
#pragma unroll 2
    for (int j = 0; j < cnt; ++j) {
      float x[NB];
      bcast_basis(cur, j, x);
      float2 p01, p23;
      preact4(x, w01, w23, p01, p23);
      float4 o;
      o.x = p01.x * sigmoid(p01.x);
      o.y = p01.y * sigmoid(p01.y);
      o.z = p23.x * sigmoid(p23.x);
      o.w = p23.y * sigmoid(p23.y);
      __stcs(reinterpret_cast<float4*>(hrow + (int64_t)j * H), o);
    }
    cur = nxt;
  }
}

// ROWS = true: the backward on the slots of nqb_edge_pairs, u < min(E, *count): grad_h row u is the slot's summed
// gradient, the pre-activation is recomputed from emb[rows[2 u]], and the slot writes its representative's grad_emb row
// and exact zeros to its partner's row (the grid is sized for E)
template <bool ROWS = false>
__global__ void __launch_bounds__(256) k_hidden_bwd(const float* __restrict__ emb, const float* __restrict__ W1s,
                                                    const float* __restrict__ gh, int64_t E, float* __restrict__ gemb,
                                                    const int64_t* __restrict__ rows = nullptr,
                                                    const int64_t* __restrict__ count = nullptr) {
  const int lane = threadIdx.x & 31, m0 = lane * 4;
  if constexpr (ROWS) E = min(E, *count);
  float2 w01[NB], w23[NB];
#pragma unroll
  for (int k = 0; k < NB; ++k) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(W1s + k * H + m0));
    w01[k] = make_float2(t.x, t.y);
    w23[k] = make_float2(t.z, t.w);
  }
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t nbatch = (E + 31) >> 5;
  int64_t b = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // ROWS: lane j also keeps the (representative, partner) edges of the batch's slot j
  [[maybe_unused]] longlong2 cur_pr, nxt_pr;
  auto load = [&](int64_t u, int64_t n, longlong2& pr) {
    if constexpr (ROWS) {
      pr = u < n ? __ldg(reinterpret_cast<const longlong2*>(rows) + u) : make_longlong2(0, -1);
      return load_basis(emb, pr.x, u < n ? pr.x + 1 : 0);
    } else {
      return load_basis(emb, u, n);
    }
  };
  Basis8 cur = load(b * 32 + lane, b < nbatch ? E : 0, cur_pr);
  for (; b < nbatch; b += nwarps) {
    const int64_t bn = b + nwarps;
    const Basis8 nxt = load(bn * 32 + lane, bn < nbatch ? E : 0, nxt_pr);
    const int64_t e0 = b * 32;
    const int cnt = (int)((E - e0) < 32 ? (E - e0) : 32);  // warp-uniform
    const float* grow = gh + e0 * H + m0;
#pragma unroll 1
    for (int j0 = 0; j0 < cnt; j0 += 4) {  // four edges per iteration
      float4 g[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        g[u] = (j0 + u < cnt) ? __ldcs(reinterpret_cast<const float4*>(grow + (int64_t)(j0 + u) * H))
                              : make_float4(0.f, 0.f, 0.f, 0.f);
      float v[32];  // v[u * 8 + k]: this lane's share of grad_emb[e0 + j0 + u, k]
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float x[NB];
        bcast_basis(cur, (j0 + u) & 31, x);
        float2 p01, p23;
        preact4(x, w01, w23, p01, p23);
        // gp[q] = grad_h[q] * silu'(p[q]),  silu'(p) = s (1 + p (1 - s))
        const float s0 = sigmoid(p01.x), s1 = sigmoid(p01.y), s2 = sigmoid(p23.x), s3 = sigmoid(p23.y);
        const float2 gp01 = make_float2(g[u].x * (s0 * fmaf(p01.x, 1.0f - s0, 1.0f)), g[u].y * (s1 * fmaf(p01.y, 1.0f - s1, 1.0f)));
        const float2 gp23 = make_float2(g[u].z * (s2 * fmaf(p23.x, 1.0f - s2, 1.0f)), g[u].w * (s3 * fmaf(p23.y, 1.0f - s3, 1.0f)));
#pragma unroll
        for (int k = 0; k < NB; ++k) {
          const float2 t = fma2_rn(gp23, w23[k], fmul2_rn(gp01, w01[k]));
          v[u * 8 + k] = t.x + t.y;
        }
      }
      // halving butterfly over the 32 lanes: after the step with offset o a lane keeps the half of its values
      // whose element index has bit o equal to its own lane bit o; after five steps lane l holds element l
#define NQB_HALVE(O, C)                                                        \
  {                                                                            \
    const bool up = (lane & (O)) != 0;                                         \
    _Pragma("unroll") for (int j = 0; j < (C); ++j) {                          \
      const float mine = up ? v[j + (C)] : v[j];                               \
      const float theirs = up ? v[j] : v[j + (C)];                             \
      v[j] = mine + __shfl_xor_sync(0xffffffffu, theirs, (O));                 \
    }                                                                          \
  }
      NQB_HALVE(16, 16)
      NQB_HALVE(8, 8)
      NQB_HALVE(4, 4)
      NQB_HALVE(2, 2)
      NQB_HALVE(1, 1)
#undef NQB_HALVE
      // element `lane` = (edge j0 + lane / 8, component lane % 8): 128 contiguous bytes per warp
      if constexpr (ROWS) {
        const int src = (j0 + (lane >> 3)) & 31;
        const int64_t rep = __shfl_sync(0xffffffffu, cur_pr.x, src), par = __shfl_sync(0xffffffffu, cur_pr.y, src);
        if (j0 + (lane >> 3) < cnt) {
          gemb[rep * NB + (lane & 7)] = v[0];
          if (par >= 0) gemb[par * NB + (lane & 7)] = 0.f;
        }
      } else {
        if (j0 + (lane >> 3) < cnt) gemb[(e0 + j0) * NB + lane] = v[0];
      }
    }
    cur = nxt;
    if constexpr (ROWS) cur_pr = nxt_pr;
  }
}

// ---------------------------------------------------------------------------------------------
// reverse-edge pair map (nqb_edge_pairs): the radial MLP's input is the edge embedding alone, so an edge and its
// reverse edge with a bitwise-equal embedding row get bitwise-equal MLP outputs and share one row of work.
//   k_pair_candidates: cand[e] = the first edge f != e, in CSR order of the row idx1[e], with idx1[f] = idx0[e],
//     shift[f] = -shift[e] (as values) and emb[f] bitwise emb[e]; -1 if none.  Eight lanes scan one row, eight
//     slots per step (coalesced loads), and stop at the first step with a hit;
//   an edge's partner is cand[e] when the relation is mutual (cand[cand[e]] = e); it represents a slot when it has
//     no partner or is the smaller of the two.  Slots are numbered by an exclusive scan over the edge ids:
//   k_pair_block_counts: representatives per tile of PT edges;
//   k_pair_write: each tile adds the counts of the tiles before it, scans its own edges and writes its slots; the
//     last tile writes the total.
// ---------------------------------------------------------------------------------------------
constexpr int PT = 1024;  // edges per tile of the slot scan (256 threads x 4)

__global__ void __launch_bounds__(256) k_pair_candidates(const int64_t* __restrict__ ei, int64_t E, int64_t N,
                                                         const double* __restrict__ shift,
                                                         const uint32_t* __restrict__ emb, int words,
                                                         const int64_t* __restrict__ row_ptr,
                                                         const int64_t* __restrict__ perm, int64_t* __restrict__ cand) {
  const int lane = threadIdx.x & 31, g = lane >> 3, r = lane & 7;
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t wv = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); wv * 4 < E; wv += nwarps) {
    const int64_t e = wv * 4 + g;  // four edges per warp, one per group of eight lanes
    int64_t a = -1, s = 0, s1 = 0;
    if (e < E) {
      a = ei[e];
      const int64_t b = ei[E + e];
      if (b >= 0 && b < N) {
        s = row_ptr[b];
        s1 = row_ptr[b + 1];
      }
    }
    int64_t found = -1;
    bool done = s >= s1;
    while (__any_sync(0xffffffffu, !done)) {
      int64_t f = -1;
      bool hit = false;
      if (!done && s + r < s1) {
        f = perm ? perm[s + r] : s + r;
        hit = f != e && ei[E + f] == a;
        if (hit && shift)
          hit = shift[3 * f] == -shift[3 * e] && shift[3 * f + 1] == -shift[3 * e + 1] &&
                shift[3 * f + 2] == -shift[3 * e + 2];
        for (int k = 0; hit && k < words; ++k) hit = emb[f * words + k] == emb[e * words + k];
      }
      const uint32_t grp = (__ballot_sync(0xffffffffu, hit) >> (8 * g)) & 0xffu;
      const int64_t first = __shfl_sync(0xffffffffu, f, 8 * g + (grp ? __ffs(grp) - 1 : 0));
      if (!done && grp) {
        found = first;
        done = true;
      }
      s += 8;
      if (s >= s1) done = true;
    }
    if (r == 0 && e < E) cand[e] = found;
  }
}

// 1 when edge e represents a slot; its partner (or -1) in *partner
__device__ __forceinline__ int pair_rep(const int64_t* __restrict__ cand, int64_t e, int64_t* partner) {
  const int64_t c = cand[e];
  const int64_t p = (c >= 0 && cand[c] == e) ? c : -1;
  *partner = p;
  return (p < 0 || e < p) ? 1 : 0;
}

// inclusive sum over the 256 threads of the block (scratch: 8 ints), returned to every thread together with the total
__device__ __forceinline__ int block_scan256(int v, int* scratch, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) scratch[warp] = v;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const int x = scratch[w];
    before += (w < warp) ? x : 0;
    all += x;
  }
  __syncthreads();
  *total = all;
  return v + before;
}

__global__ void __launch_bounds__(256) k_pair_block_counts(const int64_t* __restrict__ cand, int64_t E,
                                                           int64_t* __restrict__ counts) {
  __shared__ int scratch[8];
  const int64_t e0 = (int64_t)blockIdx.x * PT + threadIdx.x * 4;
  int n = 0;
  int64_t p;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (e0 + k < E) n += pair_rep(cand, e0 + k, &p);
  int total;
  block_scan256(n, scratch, &total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(256) k_pair_write(const int64_t* __restrict__ cand, int64_t E,
                                                    const int64_t* __restrict__ counts, int64_t* __restrict__ pair_rows,
                                                    int64_t* __restrict__ count) {
  __shared__ int scratch[8];
  __shared__ int64_t base_part[8];
  // slots of the tiles before this one
  int64_t before = 0;
  for (int64_t t = threadIdx.x; t < blockIdx.x; t += blockDim.x) before += counts[t];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
  if ((threadIdx.x & 31) == 0) base_part[threadIdx.x >> 5] = before;
  __syncthreads();
  int64_t base = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) base += base_part[w];
  const int64_t e0 = (int64_t)blockIdx.x * PT + threadIdx.x * 4;
  int rep[4], n = 0;
  int64_t partner[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    rep[k] = (e0 + k < E) ? pair_rep(cand, e0 + k, &partner[k]) : 0;
    n += rep[k];
  }
  int total;
  int64_t u = base + block_scan256(n, scratch, &total) - n;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (rep[k]) {
      reinterpret_cast<longlong2*>(pair_rows)[u] = make_longlong2(e0 + k, partner[k]);
      ++u;
    }
  if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) *count = base + total;
}

}  // namespace

extern "C" int nqb_set_error(const char* msg);  // defined in nqb_runtime.cu
extern "C" void nqb_count_launch(void);

// persistent grid of exactly the resident CTAs (occupancy x SMs), so that a warp sees several batches and
// its next batch is always prefetched; fewer CTAs when there are fewer batches than warps
template <typename K>
static unsigned hidden_grid(K kernel, int which, int64_t E) {
  static int ctas_dev[4][64] = {{0}, {0}, {0}, {0}};
  int dev = 0;
  cudaGetDevice(&dev);
  dev &= 63;
  if (ctas_dev[which][dev] == 0) {
    int sms = 0, occ = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, 256, 0) != cudaSuccess || occ <= 0) occ = 2;
    ctas_dev[which][dev] = (sms > 0 ? sms : 132) * occ;
  }
  const int64_t need = (((E + 31) >> 5) + 7) / 8;  // 8 warps per CTA, one batch of 32 edges per warp
  return (unsigned)(need < ctas_dev[which][dev] ? need : ctas_dev[which][dev]);
}

extern "C" int nqb_mlp_hidden_fwd(const float* emb, const float* W1s, int64_t E, int num_bessel, int hidden, float* h,
                                  nqb_stream_t st) {
  if (num_bessel != NB || hidden != H) return nqb_set_error("nqb_mlp_hidden_fwd: only num_bessel=8, hidden=128 is built");
  if (E < 0) return nqb_set_error("nqb_mlp_hidden_fwd: negative size");
  if (E == 0) return 0;
  if (!emb || !W1s || !h) return nqb_set_error("nqb_mlp_hidden_fwd: null pointer");
  k_hidden_fwd<<<hidden_grid(k_hidden_fwd<false>, 0, E), 256, 0, (cudaStream_t)st>>>(emb, W1s, E, h);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_mlp_hidden_fwd_rows(const float* emb, const float* W1s, const int64_t* pair_rows,
                                       const int64_t* count, int64_t capacity, int num_bessel, int hidden, float* h,
                                       nqb_stream_t st) {
  if (num_bessel != NB || hidden != H)
    return nqb_set_error("nqb_mlp_hidden_fwd_rows: only num_bessel=8, hidden=128 is built");
  if (capacity < 0) return nqb_set_error("nqb_mlp_hidden_fwd_rows: negative size");
  if (capacity == 0) return 0;
  if (!emb || !W1s || !pair_rows || !count || !h) return nqb_set_error("nqb_mlp_hidden_fwd_rows: null pointer");
  k_hidden_fwd<true><<<hidden_grid(k_hidden_fwd<true>, 2, capacity), 256, 0, (cudaStream_t)st>>>(emb, W1s, capacity, h,
                                                                                                 pair_rows, count);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_mlp_hidden_bwd(const float* emb, const float* W1s, const float* grad_h, int64_t E, int num_bessel,
                                  int hidden, float* grad_emb, nqb_stream_t st) {
  if (num_bessel != NB || hidden != H) return nqb_set_error("nqb_mlp_hidden_bwd: only num_bessel=8, hidden=128 is built");
  if (E < 0) return nqb_set_error("nqb_mlp_hidden_bwd: negative size");
  if (E == 0) return 0;
  if (!emb || !W1s || !grad_h || !grad_emb) return nqb_set_error("nqb_mlp_hidden_bwd: null pointer");
  k_hidden_bwd<<<hidden_grid(k_hidden_bwd<false>, 1, E), 256, 0, (cudaStream_t)st>>>(emb, W1s, grad_h, E, grad_emb);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_mlp_hidden_bwd_rows(const float* emb, const float* W1s, const float* grad_h,
                                       const int64_t* pair_rows, const int64_t* count, int64_t capacity,
                                       int num_bessel, int hidden, float* grad_emb, nqb_stream_t st) {
  if (num_bessel != NB || hidden != H)
    return nqb_set_error("nqb_mlp_hidden_bwd_rows: only num_bessel=8, hidden=128 is built");
  if (capacity < 0) return nqb_set_error("nqb_mlp_hidden_bwd_rows: negative size");
  if (capacity == 0) return 0;
  if (!emb || !W1s || !grad_h || !pair_rows || !count || !grad_emb)
    return nqb_set_error("nqb_mlp_hidden_bwd_rows: null pointer");
  if ((uintptr_t)pair_rows & 15) return nqb_set_error("nqb_mlp_hidden_bwd_rows: pair_rows must be 16-byte aligned");
  k_hidden_bwd<true><<<hidden_grid(k_hidden_bwd<true>, 3, capacity), 256, 0, (cudaStream_t)st>>>(
      emb, W1s, grad_h, capacity, grad_emb, pair_rows, count);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int64_t nqb_edge_pairs_work_size(int64_t E) { return E > 0 ? E + (E + PT - 1) / PT : 0; }

extern "C" int nqb_edge_pairs(const int64_t* edge_index, int64_t E, int64_t N, const double* shift, const float* emb,
                              int num_bessel, const int64_t* row_ptr, const int64_t* perm, int64_t* work,
                              int64_t* pair_rows, int64_t* count, nqb_stream_t st) {
  if (E < 0 || N < 0 || num_bessel <= 0) return nqb_set_error("nqb_edge_pairs: bad size");
  if (!count) return nqb_set_error("nqb_edge_pairs: null pointer");
  if (E == 0) {
    cudaError_t e = cudaMemsetAsync(count, 0, sizeof(int64_t), (cudaStream_t)st);
    return e == cudaSuccess ? 0 : nqb_set_error(cudaGetErrorString(e));
  }
  if (!edge_index || !emb || !row_ptr || !work || !pair_rows) return nqb_set_error("nqb_edge_pairs: null pointer");
  if ((uintptr_t)pair_rows & 15) return nqb_set_error("nqb_edge_pairs: pair_rows must be 16-byte aligned");
  const int64_t tiles = (E + PT - 1) / PT;
  int sms = 0, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t warps = (E + 3) / 4, cap = (int64_t)(sms > 0 ? sms : 132) * 8;  // 8 CTAs of 8 warps per SM
  const unsigned cblocks = (unsigned)((warps + 7) / 8 < cap ? (warps + 7) / 8 : cap);
  k_pair_candidates<<<cblocks, 256, 0, (cudaStream_t)st>>>(edge_index, E, N, shift,
                                                            reinterpret_cast<const uint32_t*>(emb), num_bessel, row_ptr,
                                                            perm, work);
  nqb_count_launch();
  k_pair_block_counts<<<(unsigned)tiles, 256, 0, (cudaStream_t)st>>>(work, E, work + E);
  nqb_count_launch();
  k_pair_write<<<(unsigned)tiles, 256, 0, (cudaStream_t)st>>>(work, E, work + E, pair_rows, count);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}
