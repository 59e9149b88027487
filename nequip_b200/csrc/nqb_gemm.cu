// Grouped fp32-accurate GEMM on the Hopper tensor cores (wgmma tf32, 3xTF32 split), sm_90a.
//
//   C_p[M, N_p] (ldc)  (+)=  rowscale_p[m] * ( A_p[M, K_p] (lda, fp32 row-major) @ B_p[K_p, N_p] )
//
// for a list of problems p that share M (number of edges or atoms) -- one launch per dense layer:
//   * radial MLP second layer and its backward         nequip/nn/mlp.py:262-268 (torch.mm)
//   * o3.Linear per-irrep channel mixing (linear_1/2)   nequip/nn/interaction_block.py:82-87,129-138
//   * self-connection FullyConnectedTensorProduct       nequip/nn/interaction_block.py:140-146
//     (per-type effective weights; rowscale = one-hot column of the atom type)
// in the channel-contiguous (ir_mul) node layout every (irrep component, chunk pair) is a plain
// strided GEMM, so no transposes/copies are needed around these calls.
//
// fp32 parity on a TF32 pipe: a = hi + lo (hi = a with the low 13 mantissa bits ignored by the tensor core),
// D = A_hi B_hi + (A_lo B_hi + A_hi B_lo).  The two cross terms go to their own accumulator and long reductions
// are cut into segments of SEG * 32 = 320 in K whose partial sums are added in registers (round-to-nearest), so
// that no accumulator sees more than 40 accumulation steps.
//
// CTA = 2 warpgroups, persistent over (M-tile, N-tile) work items of 128 x 128; the CTAs working on one A tile
// run together and share it in L2.  Warpgroup g owns rows 64 g .. 64 g + 63 of the tile:
//   * it stages its own A rows, one 32-wide K chunk at a time, with 16-byte cp.async (DEPTH chunks ahead across
//     work-item boundaries) into the canonical K-major core-matrix layout, and writes their tf32 low parts;
//   * it issues wgmma m64n128k8 from shared memory (4 k-steps x 3 terms per chunk) into two register
//     accumulators (hi*hi and cross terms), keeps one chunk's MMAs in flight while it stages the next chunk of
//     the same accumulation segment, and stores C straight from the accumulators.
// Thread 0 streams the pre-split weight chunks [hi | lo] x [128 x 32] with cp.async.bulk into a ring of BSLOTS
// slots (mbarrier complete_tx); a problem with K <= 128 keeps its chunks resident for all of the CTA's M-tiles.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/nqb.h"
#include "nqb_tc.cuh"

namespace {

constexpr int TM = 128;          // rows per tile
constexpr int TN = 128;          // max columns per tile (= wgmma N)
constexpr int KC = 32;           // K chunk (one weight block, one staged A piece)
constexpr int MW = 64;           // rows per warpgroup (= wgmma M)
constexpr int NWG = TM / MW;     // consumer warpgroups
constexpr int DEPTH = 2;         // A chunks in flight per warpgroup
constexpr int RAW = DEPTH + 1;   // ring of raw A chunks: the one being multiplied + DEPTH loading
constexpr int NLO = 2;           // ring of A low-part chunks
constexpr int BSLOTS = 4;        // B slots: a ring when K > 128, resident per N-tile when K <= 128
constexpr int SEG = 320 / KC;    // chunks per accumulation segment
constexpr int NTHREADS = NWG * 128;
constexpr int BLOCK_FLOATS = 2 * TN * KC;  // one prepared weight block: [hi | lo] x [128 x 32]

struct GemmDesc {  // mirrored by nequip_b200/ops.py (int64 fields)
  int64_t a_off, c_off, b_off, rs_off;  // element offsets from the base pointers; rs_off = ROW of the
                                        // [R, rs_ld] row-scale matrix (< 0: no row scale)
  int64_t lda, ldc, K, N;
  int64_t kchunks, ntiles, tile0, flags;  // flags: see the epilogue
};

struct Smem {
  float b[BSLOTS][BLOCK_FLOATS];     // 4 x 32 KB
  float araw[NWG][RAW][MW * KC];     // 2 x 3 x 8 KB: fp32 A chunks, canonical K-major core-matrix layout
  float alo[NWG][NLO][MW * KC];      // 2 x 2 x 8 KB: their tf32 low parts
  uint64_t b_full[BSLOTS], b_empty[BSLOTS];
};

// the gathered-sum A operand (ROWS = PAIRS_A) lands each partner chunk in the low-part slot of its chunk, so the
// low-part ring has RAW slots instead of NLO: 128 + 48 + 48 KB
struct SmemPairsA {
  float b[BSLOTS][BLOCK_FLOATS];
  float araw[NWG][RAW][MW * KC];  // representative rows; the low-part pass overwrites them with the sums
  float alo[NWG][RAW][MW * KC];   // partner rows (zero-filled when a slot has none); overwritten with the low parts
  uint64_t b_full[BSLOTS], b_empty[BSLOTS];
};

// how A rows and C rows map to M (nqb_gemm_grouped / _pairs / _pair_sum)
constexpr int ROWS_PLAIN = 0;  // row m of A and of C
constexpr int PAIRS_C = 1;     // A row m; C rows pair_rows[m][0] and, when >= 0, pair_rows[m][1]
constexpr int PAIRS_A = 2;     // A row pair_rows[m][0] + A row pair_rows[m][1] (when >= 0); C row m
template <int ROWS>
using SmemFor = std::conditional_t<ROWS == PAIRS_A, SmemPairsA, Smem>;

__device__ __forceinline__ const GemmDesc* find_desc(const GemmDesc* d, int nd, int q) {
  int i = 0;
  while (i + 1 < nd && d[i + 1].tile0 <= q) ++i;
  return d + i;
}

// Work schedule.  T = N-tiles over all problems, G = CTAs.
//   T <= G: CTA b owns ONE N-tile q = b % T and the M-tiles r, r+R, r+2R, ... (r = b / T, R = G / T):
//           the T CTAs that share r sweep the same M-tiles in lockstep (A tiles are shared in L2)
//           and the weight tile of a K <= 128 problem stays resident in shared memory;
//   T >  G: CTA b owns N-tiles b, b+G, ... and sweeps all M-tiles for each.
struct Sched {
  int q, q_step, nq_total;
  int64_t m_start, m_step;
  // tile_ctas (nullable): per N-tile {first CTA, number of CTAs} of a cost-weighted split computed by the
  // host for a grid of exactly sched_ctas CTAs (problems of one launch differ in K, N and store mode, so
  // an even split leaves most CTAs idle while the expensive tiles finish)
  __device__ Sched(int b, int G, int T, const int32_t* tile_ctas, int sched_ctas) {
    nq_total = T;
    if (tile_ctas != nullptr && G == sched_ctas) {
      q = T; q_step = T; m_start = 0; m_step = 1;
      for (int t = 0; t < T; ++t) {
        const int c0 = tile_ctas[2 * t], n = tile_ctas[2 * t + 1];
        if (b >= c0 && b < c0 + n) { q = t; m_start = b - c0; m_step = n; break; }
      }
    } else if (T <= G) {
      const int R = G / T;
      q = (b < T * R) ? (b % T) : T;  // T = no work
      q_step = T;
      m_start = b / T;
      m_step = R;
    } else {
      q = b; q_step = G; m_start = 0; m_step = 1;
    }
  }
};

struct WorkQ {  // one N-tile of one problem
  const GemmDesc* d;
  int nt, kchunks, K, ncols;
  bool resident;
};
__device__ __forceinline__ void decode_q(const GemmDesc* descs, int ndesc, int q, WorkQ& w) {
  w.d = find_desc(descs, ndesc, q);
  w.nt = q - (int)w.d->tile0;
  w.kchunks = (int)w.d->kchunks;
  w.K = (int)w.d->K;
  w.ncols = min(TN, (int)w.d->N - w.nt * TN);
  w.resident = w.kchunks <= BSLOTS;
}

__device__ __forceinline__ void bar_wg(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

// ACT = false: the plain GEMM.  ACT = true also honours the activation bits 3-5 of a problem's flags in the
// epilogue, with the auxiliary matrix at aux_base (addressed with C's c_off and ldc); see nqb.h.
// ROWS = PAIRS_C / PAIRS_A (plain problems only): M = min(M, *m_dev) is read on the device, and
//   PAIRS_C: result row m is stored to the C rows pair_rows[m][0] and, when it is >= 0, pair_rows[m][1]
//            (nqb_gemm_grouped_pairs);
//   PAIRS_A: row m of the product is (A[pair_rows[m][0]] + A[pair_rows[m][1]]) @ B, the second term only when
//            pair_rows[m][1] >= 0, stored to C row m (nqb_gemm_grouped_pair_sum).  Both rows are staged with cp.async;
//            the low-part pass forms the fp32 sum, writes it over the staged representative chunk (the hi operand)
//            and writes its low part.
template <bool ACT, int ROWS = ROWS_PLAIN>
__global__ void __launch_bounds__(NTHREADS, 1)
k_gemm3x(const GemmDesc* __restrict__ descs, int ndesc, int ntiles_total, const int32_t* __restrict__ tile_ctas,
         int sched_ctas, const float* __restrict__ a_base, const float* __restrict__ b_base, float* __restrict__ c_base,
         const float* __restrict__ rs_base, int64_t rs_ld, int64_t M, float* __restrict__ aux_base,
         const int64_t* __restrict__ m_dev, const int64_t* __restrict__ pair_rows) {
  constexpr bool SUMA = ROWS == PAIRS_A;
  constexpr int NLON = SUMA ? RAW : NLO;  // low-part slots
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  SmemFor<ROWS>& S = *reinterpret_cast<SmemFor<ROWS>*>(smem_raw);
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  if constexpr (ROWS != ROWS_PLAIN) M = min(M, *m_dev);  // the schedule does not depend on M, only the M-tiles and row guards
  const int64_t mtiles = (M + TM - 1) / TM;

  if (tid == 0) {
    for (int s = 0; s < BSLOTS; ++s) { mbar_init(&S.b_full[s], 1); mbar_init(&S.b_empty[s], NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();
  const Sched sch(blockIdx.x, gridDim.x, ntiles_total, tile_ctas, sched_ctas);

  // ---- A staging: a cursor over this CTA's flat chunk sequence (N-tile q, M-tile pmt, chunk ph_) -------------
  // thread -> rows 16 warp + 8 g + r8 (g < 2) of the warpgroup's 64, k-groups 4 kh + kq (kh < 2): a quarter warp
  // writes one contiguous 128-byte core matrix
  const int r8 = lane & 7, kq = lane >> 3;
  const int my_off = (2 * warp) * (KC / 4 * 32) + kq * 32 + r8 * 4;
  int pq = sch.q, ph_ = 0, pnh = 1, pK = 0;
  int64_t pmt = sch.m_start, plda = 0;
  const float* pA = nullptr;
  bool pvalid = pq < sch.nq_total && sch.m_start < mtiles;
  auto open_q = [&]() {
    WorkQ w;
    decode_q(descs, ndesc, pq, w);
    pA = a_base + w.d->a_off;
    plda = w.d->lda;
    pK = w.K;
    pnh = w.kchunks;
  };
  if (pvalid) open_q();
  uint32_t n_issued = 0;
  // PAIRS_A: (representative, partner) A rows of this thread's two rows of the cursor's M-tile; -1 = none
  [[maybe_unused]] int32_t prow[2][2];
  // cp.async the cursor's chunk into raw stage n_issued % RAW (PAIRS_A: its partner rows into low-part stage
  // n_issued % RAW, whose last reader, chunk n_issued - RAW, has retired), advance, commit
  auto issue = [&]() {
    if (pvalid) {
      float* dst = S.araw[wg][n_issued % RAW] + my_off;
      if constexpr (SUMA) {
        if (ph_ == 0) {  // the first chunk of an M-tile: read its rows' slots once
#pragma unroll
          for (int g = 0; g < 2; ++g) {
            const int64_t m = pmt * TM + wg * MW + warp * 16 + g * 8 + r8;
            const longlong2 pr = m < M ? __ldg(reinterpret_cast<const longlong2*>(pair_rows) + m) : make_longlong2(-1, -1);
            prow[g][0] = (int32_t)pr.x;
            prow[g][1] = (int32_t)pr.y;
          }
        }
      }
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const int64_t m = pmt * TM + wg * MW + warp * 16 + g * 8 + r8;
#pragma unroll
        for (int kh = 0; kh < 2; ++kh) {
          const int k = ph_ * KC + (kh * 4 + kq) * 4;
          if constexpr (SUMA) {
            const bool in = prow[g][0] >= 0 && k < pK, pin = in && prow[g][1] >= 0;
            cp_async16(dst + g * (KC / 4 * 32) + kh * 128, pA + (in ? (int64_t)prow[g][0] * plda + k : 0), in ? 16u : 0u);
            cp_async16(S.alo[wg][n_issued % RAW] + my_off + g * (KC / 4 * 32) + kh * 128,
                       pA + (pin ? (int64_t)prow[g][1] * plda + k : 0), pin ? 16u : 0u);
          } else {
            const bool in = m < M && k < pK;
            const int64_t off = in ? m * plda + k : 0;
            cp_async16(dst + g * (KC / 4 * 32) + kh * 128, pA + off, in ? 16u : 0u);
          }
        }
      }
      if (++ph_ == pnh) {
        ph_ = 0;
        pmt += sch.m_step;
        if (pmt >= mtiles) {
          pmt = sch.m_start;
          pq += sch.q_step;
          pvalid = pq < sch.nq_total;
          if (pvalid) open_q();
        }
      }
    }
    ++n_issued;
    cp_async_commit();
  };
#pragma unroll 1
  for (int j = 0; j < DEPTH; ++j) issue();

  // ---- weight chunks (thread 0) ------------------------------------------------------------------------------
  uint32_t bused = 0, bpar_ld = 0;  // per-slot bit: slot loaded before / parity of its load count
  auto load_slot = [&](int slot, const float* src, uint32_t bytes) {
    if ((bused >> slot) & 1) mbar_wait(&S.b_empty[slot], ((bpar_ld >> slot) & 1) ^ 1);
    mbar_expect_tx(&S.b_full[slot], 2 * bytes);
    bulk_g2s(S.b[slot], src, bytes, &S.b_full[slot]);
    bulk_g2s(S.b[slot] + TN * KC, src + TN * KC, bytes, &S.b_full[slot]);
    bused |= 1u << slot;
    bpar_ld ^= 1u << slot;
  };
  uint32_t bpar = 0;  // per-slot bit: parity of the loads consumed (waited for)

  constexpr uint32_t SBO = (KC / 4) * 128, LBO = 128;
  constexpr uint32_t A_STAGE = (MW * KC * sizeof(float)) >> 4;
  constexpr uint32_t B_SLOT = (BLOCK_FLOATS * sizeof(float)) >> 4, B_LO = (TN * KC * sizeof(float)) >> 4;
  const uint64_t dR0 = make_desc(smem_u32(S.araw[wg][0]), LBO, SBO);
  const uint64_t dL0 = make_desc(smem_u32(S.alo[wg][0]), LBO, SBO);
  const uint64_t dB0 = make_desc(smem_u32(S.b[0]), LBO, SBO);
  const int r0 = warp * 16 + (lane >> 2), c0 = 2 * (lane & 3);  // accumulator rows r0, r0 + 8; columns 8 j + c0 (+1)
  float hh[64], xx[64], acc[64];
  uint32_t i = 0;  // chunks consumed by this warpgroup

  for (int q = sch.q; q < sch.nq_total; q += sch.q_step) {
    WorkQ w;
    decode_q(descs, ndesc, q, w);
    if (sch.m_start >= mtiles) continue;
    const GemmDesc* d = w.d;
    const int nseg = (w.kchunks + SEG - 1) / SEG;
    const int64_t nmt = (mtiles - 1 - sch.m_start) / sch.m_step + 1;
    const int64_t nload = w.resident ? w.kchunks : nmt * w.kchunks;  // chunk loads of this N-tile
    const uint32_t bytes = (uint32_t)TN * KC * sizeof(float);
    const float* B = b_base + d->b_off + (int64_t)w.nt * w.kchunks * BLOCK_FLOATS;
    if (tid == 0)
      for (int64_t c = 0; c < min((int64_t)BSLOTS, nload); ++c) load_slot((int)c, B + (c % w.kchunks) * BLOCK_FLOATS, bytes);
    int64_t x = 0, xr = 0;  // streaming mode: chunk loads of this N-tile consumed / given back to the loader
    // chunk y's MMAs have retired: its slot is free for chunk y + BSLOTS
    auto release = [&](int64_t y) {
      const int slot = (int)(y % BSLOTS);
      if (lane == 0) mbar_arrive(&S.b_empty[slot]);
      if (tid == 0 && y + BSLOTS < nload) load_slot(slot, B + ((y + BSLOTS) % w.kchunks) * BLOCK_FLOATS, bytes);
    };
    // flags: bit0 read-modify-write accumulate (single writer per element within the launch),
    //        bit1 rows whose row scale is zero are not touched (disjoint row-masked writers),
    //        bit2 accumulate with red.global.add (several problems of this launch add into the same C)
    // both accumulate modes add with red.global (performed at L2)
    // ACT only (never with bit0 / bit2): bit3 store silu(v), bit4 also store v to aux, bit5 store v * silu'(aux)
    const bool reduce = (d->flags & 5) != 0, skipz = (d->flags & 2) != 0;
    const int64_t ldc = d->ldc;
    float* C = c_base + d->c_off + (int64_t)w.nt * TN;
    [[maybe_unused]] const int act = ACT ? (int)(d->flags >> 3) & 7 : 0;
    [[maybe_unused]] float* X = ACT && (act & 6) ? aux_base + d->c_off + (int64_t)w.nt * TN : nullptr;
    bool first_mt = true;
    for (int64_t mt = sch.m_start; mt < mtiles; mt += sch.m_step) {
      for (int seg = 0; seg < nseg; ++seg) {
        const int h1 = min(w.kchunks, (seg + 1) * SEG);
        for (int h = seg * SEG; h < h1; ++h, ++i) {
          // chunk i - 1's MMAs (if any) run during everything up to this chunk's first wgmma; chunk i - NLON, the
          // last reader of low-part slot i % NLON, has retired
          cp_async_wait<DEPTH - 1>();  // my parts of chunk i have landed
          float* raw = S.araw[wg][i % RAW] + my_off;
          float* lo = S.alo[wg][i % NLON] + my_off;
#pragma unroll
          for (int g = 0; g < 2; ++g)
#pragma unroll
            for (int kh = 0; kh < 2; ++kh) {
              float4 t = *reinterpret_cast<const float4*>(raw + g * (KC / 4 * 32) + kh * 128);
              if constexpr (SUMA) {  // this thread's own cp.async pieces: the representative + the partner
                const float4 p = *reinterpret_cast<const float4*>(lo + g * (KC / 4 * 32) + kh * 128);
                t = make_float4(t.x + p.x, t.y + p.y, t.z + p.z, t.w + p.w);
                *reinterpret_cast<float4*>(raw + g * (KC / 4 * 32) + kh * 128) = t;
              }
              *reinterpret_cast<float4*>(lo + g * (KC / 4 * 32) + kh * 128) =
                  make_float4(tf32_lo(t.x), tf32_lo(t.y), tf32_lo(t.z), tf32_lo(t.w));
            }
          fence_proxy_async();  // generic-proxy writes -> visible to the tensor core
          bar_wg(wg);
          uint32_t slot;
          if (w.resident) {
            slot = h;
            if (first_mt) { mbar_wait(&S.b_full[slot], (bpar >> slot) & 1); bpar ^= 1u << slot; }
          } else {
            slot = (uint32_t)(x++ % BSLOTS);
            mbar_wait(&S.b_full[slot], (bpar >> slot) & 1);
            bpar ^= 1u << slot;
          }
          const uint64_t a_hi = dR0 + (uint64_t)((i % RAW) * A_STAGE), a_lo = dL0 + (uint64_t)((i % NLON) * A_STAGE);
          const uint64_t b_hi = dB0 + (uint64_t)(slot * B_SLOT), b_lo = b_hi + B_LO;
          const uint32_t fresh = (h == seg * SEG);  // the first chunk of a segment overwrites the accumulators
          wgmma_fence();
          // k-step advance = 2 core matrices = 256 bytes = 16 descriptor units
#pragma unroll
          for (int ks = 0; ks < KC / 8; ++ks) wgmma_tf32_m64n128(hh, a_hi + ks * 16, b_hi + ks * 16, !(fresh && ks == 0));
#pragma unroll
          for (int ks = 0; ks < KC / 8; ++ks) wgmma_tf32_m64n128(xx, a_lo + ks * 16, b_hi + ks * 16, !(fresh && ks == 0));
#pragma unroll
          for (int ks = 0; ks < KC / 8; ++ks) wgmma_tf32_m64n128(xx, a_hi + ks * 16, b_lo + ks * 16, 1u);
          wgmma_commit();
          wgmma_wait<1>();  // chunk i - 1 has retired, chunk i stays in flight
          if (xr + 1 < x) release(xr++);
          issue();  // chunk i + DEPTH into the stage of chunk i - 1
        }
        wgmma_wait<0>();  // the sums below and the epilogue read the accumulators
        if (xr < x) release(xr++);
        // segment sums in registers; the last segment leaves the result in hh
        if (seg + 1 < nseg) {
#pragma unroll
          for (int j = 0; j < 64; ++j) acc[j] = (seg == 0 ? 0.f : acc[j]) + (hh[j] + xx[j]);
        } else {
#pragma unroll
          for (int j = 0; j < 64; ++j) hh[j] = (seg == 0) ? hh[j] + xx[j] : acc[j] + (hh[j] + xx[j]);
        }
      }
      // ---- epilogue: C rows r0 and r0 + 8 of this warpgroup, two adjacent columns per store --------------------
      const int64_t m0 = mt * TM + wg * MW + r0;
      if constexpr (ROWS == PAIRS_C) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int64_t m = m0 + half * 8;
          if (m >= M) continue;
          const longlong2 pr = __ldg(reinterpret_cast<const longlong2*>(pair_rows) + m);
          float* crow0 = C + pr.x * ldc + c0;
          float* crow1 = C + pr.y * ldc + c0;  // stored to only when pr.y >= 0
#pragma unroll
          for (int j = 0; j < TN / 8; ++j) {
            if (j * 8 + c0 < w.ncols) {
              const float2 v = make_float2(hh[4 * j + 2 * half], hh[4 * j + 2 * half + 1]);
              *reinterpret_cast<float2*>(crow0 + j * 8) = v;
              if (pr.y >= 0) *reinterpret_cast<float2*>(crow1 + j * 8) = v;
            }
          }
        }
      } else
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int64_t m = m0 + half * 8;
        float rs = 1.0f;
        if (d->rs_off >= 0) rs = (m < M) ? __ldg(rs_base + d->rs_off * rs_ld + m) : 0.f;
        if (m >= M || (skipz && rs == 0.f)) continue;
        float* crow = C + m * ldc + c0;
#pragma unroll
        for (int j = 0; j < TN / 8; ++j) {
          if (j * 8 + c0 < w.ncols) {
            float v0 = hh[4 * j + 2 * half] * rs, v1 = hh[4 * j + 2 * half + 1] * rs;
            if constexpr (ACT) {
              if (act != 0) {
                float* xp = X + m * ldc + c0 + j * 8;
                if (act & 4) {  // gradient through the activation: silu'(p) = s (1 + p (1 - s))
                  const float2 p = *reinterpret_cast<const float2*>(xp);
                  const float s0 = sigmoid(p.x), s1 = sigmoid(p.y);
                  v0 *= s0 * fmaf(p.x, 1.0f - s0, 1.0f);
                  v1 *= s1 * fmaf(p.y, 1.0f - s1, 1.0f);
                } else {
                  if (act & 2) *reinterpret_cast<float2*>(xp) = make_float2(v0, v1);
                  if (act & 1) {
                    v0 *= sigmoid(v0);
                    v1 *= sigmoid(v1);
                  }
                }
              }
            }
            if (reduce)
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(crow + j * 8), "f"(v0), "f"(v1) : "memory");
            else
              *reinterpret_cast<float2*>(crow + j * 8) = make_float2(v0, v1);
          }
        }
      }
      first_mt = false;
    }
    // resident weights: release the slots once every MMA of this N-tile has retired
    if (w.resident && lane == 0)
      for (int c = 0; c < w.kchunks; ++c) mbar_arrive(&S.b_empty[c]);
  }
  cp_async_wait<0>();
}

// prepared layout: for n-tile j, k-chunk c: block (j * kchunks + c) of BLOCK_FLOATS floats = [hi | lo],
// each [128 rows (n) x 32 (k)] K-major canonical; rows >= N and k >= K are zero.
__global__ void k_gemm_prepare(const float* __restrict__ B, int64_t ldb, int K, int N, int transposed, float scale,
                               float* __restrict__ out, int kchunks, int ntiles) {
  const int64_t total = (int64_t)ntiles * kchunks * TN * KC;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int kk = (int)(idx % KC);
    const int nn = (int)((idx / KC) % TN);
    const int64_t blk = idx / (KC * TN);
    const int c = (int)(blk % kchunks), j = (int)(blk / kchunks);
    const int k = c * KC + kk, n = j * TN + nn;
    float v = 0.f;
    if (k < K && n < N) v = (transposed ? B[(int64_t)n * ldb + k] : B[(int64_t)k * ldb + n]) * scale;
    const float hi = tf32_rn(v), lo = v - hi;
    float* tile = out + blk * BLOCK_FLOATS;
    const int off = canon_off(nn, kk, KC / 4);
    tile[off] = hi;
    tile[TN * KC + off] = lo;
  }
}

}  // namespace

extern "C" int nqb_set_error(const char* msg);
extern "C" void nqb_count_launch(void);

// per-device state (one process may drive several GPUs: attributes and SM counts are per device)
static int gemm_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev & 63;
}
static int gemm_sm_count() {
  static int n[64] = {0};
  const int dev = gemm_device();
  if (n[dev] == 0) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

extern "C" int64_t nqb_gemm_prepared_floats(int K, int N) {
  const int64_t kchunks = (K + KC - 1) / KC, ntiles = (N + TN - 1) / TN;
  return kchunks * ntiles * BLOCK_FLOATS;
}

extern "C" int nqb_gemm_prepare(const float* B, int64_t ldb, int K, int N, int transposed, float scale, float* prepared,
                                nqb_stream_t st) {
  if (!B || !prepared) return nqb_set_error("nqb_gemm_prepare: null pointer");
  if (K <= 0 || N <= 0) return nqb_set_error("nqb_gemm_prepare: bad shape");
  const int kchunks = (K + KC - 1) / KC, ntiles = (N + TN - 1) / TN;
  const int64_t total = (int64_t)ntiles * kchunks * TN * KC;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  k_gemm_prepare<<<blocks, 256, 0, (cudaStream_t)st>>>(B, ldb, K, N, transposed, scale, prepared, kchunks, ntiles);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// the launcher of the entry points; errors are reported under the entry point's name
template <bool ACT, int ROWS = ROWS_PLAIN>
static int gemm_grouped_launch(const char* who, const void* descs_dev, int ndesc, int ntiles_total,
                               const int32_t* tile_ctas_dev, int sched_ctas, const float* a_base,
                               const float* prepared_base, float* c_base, float* aux_base, const float* rowscale_base,
                               int64_t rs_ld, int64_t M, nqb_stream_t st, const int64_t* m_dev = nullptr,
                               const int64_t* pair_rows = nullptr) {
  auto fail = [&](const char* what) {
    char msg[160];  // nqb_set_error copies it
    snprintf(msg, sizeof(msg), "%s: %s", who, what);
    return nqb_set_error(msg);
  };
  if (ndesc <= 0 || ntiles_total <= 0) return fail("empty problem list");
  if (M < 0) return fail("negative M");
  if (M == 0) return 0;
  if (!descs_dev || !a_base || !prepared_base || !c_base) return fail("null pointer");
  // the device descriptors cannot be read here: an activation launch always takes an aux matrix
  if (ACT && !aux_base) return fail("aux_base is null (bit4 / bit5 problems store to or read from it)");
  if (ROWS != ROWS_PLAIN && (!m_dev || !pair_rows)) return fail("pair_rows or count is null");
  if (ROWS != ROWS_PLAIN && ((uintptr_t)pair_rows & 15)) return fail("pair_rows must be 16-byte aligned");
  if (ROWS == PAIRS_A && M > INT32_MAX) return fail("capacity must be < 2^31 (A rows are held as int32)");
  // A is staged with 16-byte cp.async, the weights with bulk copies, C and aux are stored in float2 pairs
  if (((uintptr_t)a_base | (uintptr_t)prepared_base | (uintptr_t)c_base | (uintptr_t)aux_base) & 15)
    return fail(ACT ? "a_base, prepared_base, c_base and aux_base must be 16-byte aligned"
                    : "a_base, prepared_base and c_base must be 16-byte aligned");
  static bool attr_set[64] = {false};
  const int dev = gemm_device();
  if (!attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(k_gemm3x<ACT, ROWS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)sizeof(SmemFor<ROWS>) + 1024);
    if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
    attr_set[dev] = true;
  }
  const int64_t nwork = ((M + TM - 1) / TM) * (int64_t)ntiles_total;
  int grid = (int)(nwork < gemm_sm_count() ? nwork : gemm_sm_count());
  if (tile_ctas_dev != nullptr && sched_ctas > 0 && sched_ctas <= gemm_sm_count()) grid = sched_ctas;
  else tile_ctas_dev = nullptr;
  k_gemm3x<ACT, ROWS><<<grid, NTHREADS, sizeof(SmemFor<ROWS>) + 1024, (cudaStream_t)st>>>(
      (const GemmDesc*)descs_dev, ndesc, ntiles_total, tile_ctas_dev, sched_ctas, a_base, prepared_base, c_base,
      rowscale_base, rs_ld, M, aux_base, m_dev, pair_rows);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_gemm_grouped(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                                int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                                const float* rowscale_base, int64_t rs_ld, int64_t M, nqb_stream_t st) {
  return gemm_grouped_launch<false>("nqb_gemm_grouped", descs_dev, ndesc, ntiles_total, tile_ctas_dev, sched_ctas,
                                    a_base, prepared_base, c_base, nullptr, rowscale_base, rs_ld, M, st);
}

extern "C" int nqb_gemm_grouped_act(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                                    int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                                    const float* rowscale_base, int64_t rs_ld, int64_t M, float* aux_base,
                                    nqb_stream_t st) {
  return gemm_grouped_launch<true>("nqb_gemm_grouped_act", descs_dev, ndesc, ntiles_total, tile_ctas_dev, sched_ctas,
                                   a_base, prepared_base, c_base, aux_base, rowscale_base, rs_ld, M, st);
}

extern "C" int nqb_gemm_grouped_pairs(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                                      int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                                      const int64_t* pair_rows, const int64_t* count_dev, int64_t capacity,
                                      nqb_stream_t st) {
  return gemm_grouped_launch<false, PAIRS_C>("nqb_gemm_grouped_pairs", descs_dev, ndesc, ntiles_total, tile_ctas_dev,
                                          sched_ctas, a_base, prepared_base, c_base, nullptr, nullptr, 0, capacity,
                                          st, count_dev, pair_rows);
}

extern "C" int nqb_gemm_grouped_pair_sum(const void* descs_dev, int ndesc, int ntiles_total,
                                         const int32_t* tile_ctas_dev, int sched_ctas, const float* a_base,
                                         const float* prepared_base, float* c_base, const int64_t* pair_rows,
                                         const int64_t* count_dev, int64_t capacity, nqb_stream_t st) {
  return gemm_grouped_launch<false, PAIRS_A>("nqb_gemm_grouped_pair_sum", descs_dev, ndesc, ntiles_total,
                                             tile_ctas_dev, sched_ctas, a_base, prepared_base, c_base, nullptr,
                                             nullptr, 0, capacity, st, count_dev, pair_rows);
}
