// Neighbour list on the GPU (cell list, full list, periodic images), sm_90a.         SURVEY.md section 8(f)-2
//
// Reference contract (paths under /root/reference):
//   compute_neighborlist_ / backends            nequip/data/_nl.py:60-152, 292-361 -- full list (both directions), no
//     self interaction in the home image, edge vector = pos[j] - pos[i] + shift @ cell, shifts integer-valued;
//     the reference builds it on the host from pos.detach().cpu().numpy() (a serial bottleneck at >= 10k atoms)
//   SortedNeighborListTransform                 nequip/data/transforms/neighborlist.py:120-157 -- edges sorted by
//     (centre, neighbour) and the permutation to the (neighbour, centre) order
// Output here: edges grouped by centre i (= edge_index[0], the scatter destination of the convolution) and sorted
// by neighbour j inside a row -- i.e. the destination CSR the TP kernels want, written directly in device memory.
//
// Two passes over the 27 (or more, for small cells) neighbouring bins of every atom: count, exclusive scan (host
// side: torch.cumsum), fill + in-row sort.  All arithmetic that decides membership (wrapped coordinates, image
// offsets, squared distance) is done in the same order as the host reference list (nequip_b200/data.py) with
// explicitly rounded operations (no FMA contraction), so the edge set is bit-identical.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/nqb.h"

extern "C" int nqb_set_error(const char* msg);
extern "C" void nqb_count_launch(void);

namespace {

struct NlParams {
  double cell[9];     // rows = lattice vectors
  double inv[9];      // inverse (columns give fractional coordinates: frac = pos @ inv)
  double diag[3];     // diagonal of an orthorhombic cell (frac = pos / diag, exactly as the host list does)
  int orthorhombic;
  int pbc[3];
  int nb[3];          // bins per direction
  int sr[3];          // bin search range per direction
  double lo[3], width[3];  // non-periodic directions: bounding box origin / extent in fractional units
  double r2;
};

// Where the kernels read NlParams from (template argument PS): the by-value kernel parameter NlParams (host-built
// per launch) or a block in device memory, NlBlock* (variable cell: nqb_nl_params_pack fills it on the host and the
// caller copies it in before a launch or a graph replay).  The block also holds the null-edge shift of the capacity
// fill, which follows the cell.  One kernel body per kernel reads its parameters through nl_p / nl_pad_shift.
// Open directions (nqb_nl_params_pack_open): the trailing fields are read by nqb_nl_bbox only, which writes the
// bounding box (p.lo, p.width) and the grid (p.nb, p.sr) of every open direction into the block before the bins.
struct NlBlock {
  NlParams p;
  double pad_shift[3];
  int open[3];         // 1: the bounding box of this direction is found on the device
  int cap;             // most bins along an open direction (the caller's scratch grid)
  double perp[3];      // distance between opposite faces of the cell along each lattice direction
  double r_max;
};
typedef const NlBlock* __restrict__ NlBlockPtr;

// A batch of independent frames (PS = NlFrames, nqb_nl_*_frames): one block per frame, and atom i reads its
// parameters from blocks[batch[i]].  The bins of all frames lie in one global range: frame f owns
// [bin_base[f], bin_base[f + 1]), and nl_bin0 offsets atom i's bins by its frame's base, so the atoms of a frame only
// ever meet the atoms of that frame.  For the other parameter sources nl_bin0 is 0.
struct NlFrames {
  const NlBlock* blocks;    // [F]
  const int64_t* batch;     // [N] frame of each atom
  const int64_t* bin_base;  // [F + 1]
};

__device__ __forceinline__ const NlParams& nl_p(const NlParams& p, int64_t) { return p; }
__device__ __forceinline__ const NlParams& nl_p(NlBlockPtr b, int64_t) { return b->p; }
__device__ __forceinline__ const NlParams& nl_p(const NlFrames& f, int64_t i) { return f.blocks[f.batch[i]].p; }
__device__ __forceinline__ int64_t nl_bin0(const NlParams&, int64_t) { return 0; }
__device__ __forceinline__ int64_t nl_bin0(NlBlockPtr, int64_t) { return 0; }
__device__ __forceinline__ int64_t nl_bin0(const NlFrames& f, int64_t i) { return f.bin_base[f.batch[i]]; }
__device__ __forceinline__ double3 nl_pad_shift(const NlParams&, int64_t, double3 pad_shift) { return pad_shift; }
__device__ __forceinline__ double3 nl_pad_shift(NlBlockPtr b, int64_t, double3) {
  return make_double3(b->pad_shift[0], b->pad_shift[1], b->pad_shift[2]);
}
// a null edge of atom i takes the shift of its own frame: one shift for every frame could be short in another cell
__device__ __forceinline__ double3 nl_pad_shift(const NlFrames& f, int64_t i, double3) {
  const NlBlock& b = f.blocks[f.batch[i]];
  return make_double3(b.pad_shift[0], b.pad_shift[1], b.pad_shift[2]);
}

// Per-edge-type cutoffs (kTyped): the pair (i, j) is a neighbour when d2 < rc2[T * types[i] + types[j]] instead of
// d2 < r2.  rc2 = rc * rc is computed on the host in float64; the bins stay sized by the global r_max >= every rc.
// The untyped kernels take this parameter last and never read it, so their code is unchanged.
struct NlTypes {
  const int64_t* types;  // [N]
  const double* rc2;     // [T * T]
  int T;
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

// fractional coordinates of one position: x / diag for an orthorhombic cell (as the host list), otherwise
// pos @ inv with explicitly rounded operations; k_nl_bin and k_nl_bbox both call this, so the bounding box is that
// of the coordinates that get binned
__device__ __forceinline__ void nl_frac(const NlParams& p, double x, double y, double z, double f[3]) {
  if (p.orthorhombic) {
    f[0] = __ddiv_rn(x, p.diag[0]); f[1] = __ddiv_rn(y, p.diag[1]); f[2] = __ddiv_rn(z, p.diag[2]);
  } else {
    for (int d = 0; d < 3; ++d) f[d] = dadd(dadd(dmul(x, p.inv[d]), dmul(y, p.inv[3 + d])), dmul(z, p.inv[6 + d]));
  }
}

// wrapped cartesian position, integer base shift (pos + base @ cell is the wrapped position) and bin of one atom
template <class PS>
__global__ void k_nl_bin(PS ps, const double* __restrict__ pos, int64_t N, double* __restrict__ wpos,
                         int32_t* __restrict__ base, int64_t* __restrict__ bin, int32_t* __restrict__ cidx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const NlParams& p = nl_p(ps, i);
  double f[3];
  nl_frac(p, pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], f);
  double w[3];
  int c[3];
  for (int d = 0; d < 3; ++d) {
    if (p.pbc[d]) {
      const double fl = floor(f[d]);
      w[d] = dadd(f[d], -fl);
      base[3 * i + d] = (int32_t)(-fl);
      int q = (int)dmul(w[d], (double)p.nb[d]);
      c[d] = q < p.nb[d] - 1 ? q : p.nb[d] - 1;
    } else {
      w[d] = f[d];
      base[3 * i + d] = 0;
      int q = (int)floor(dmul(__ddiv_rn(dadd(f[d], -p.lo[d]), p.width[d]), (double)p.nb[d]));
      c[d] = q < 0 ? 0 : (q < p.nb[d] - 1 ? q : p.nb[d] - 1);
    }
    cidx[3 * i + d] = c[d];
  }
  if (p.orthorhombic) {
    wpos[3 * i] = dmul(w[0], p.diag[0]); wpos[3 * i + 1] = dmul(w[1], p.diag[1]); wpos[3 * i + 2] = dmul(w[2], p.diag[2]);
  } else {
    for (int d = 0; d < 3; ++d)
      wpos[3 * i + d] = dadd(dadd(dmul(w[0], p.cell[d]), dmul(w[1], p.cell[3 + d])), dmul(w[2], p.cell[6 + d]));
  }
  bin[i] = nl_bin0(ps, i) + ((int64_t)c[2] * p.nb[1] + c[1]) * p.nb[0] + c[0];
}

// visit every (neighbour atom j, image) candidate of atom i; F(j, img[3], within cutoff)
template <bool kTyped, class F>
__device__ __forceinline__ void nl_visit(const NlParams& p, const NlTypes& ty, int64_t i, const double* __restrict__ wpos,
                                         const int32_t* __restrict__ cidx, const int64_t* __restrict__ order,
                                         const int64_t* __restrict__ bin_start, F&& f) {
  const double xi = wpos[3 * i], yi = wpos[3 * i + 1], zi = wpos[3 * i + 2];
  const double* rc2_i = kTyped ? ty.rc2 + (int64_t)ty.T * ty.types[i] : nullptr;
  const int c0 = cidx[3 * i], c1 = cidx[3 * i + 1], c2 = cidx[3 * i + 2];
  for (int oz = -p.sr[2]; oz <= p.sr[2]; ++oz) {
    int bz = c2 + oz, iz = 0;
    if (p.pbc[2]) { iz = (bz >= 0) ? bz / p.nb[2] : -((-bz + p.nb[2] - 1) / p.nb[2]); bz -= iz * p.nb[2]; }
    else if (bz < 0 || bz >= p.nb[2]) continue;
    for (int oy = -p.sr[1]; oy <= p.sr[1]; ++oy) {
      int by = c1 + oy, iy = 0;
      if (p.pbc[1]) { iy = (by >= 0) ? by / p.nb[1] : -((-by + p.nb[1] - 1) / p.nb[1]); by -= iy * p.nb[1]; }
      else if (by < 0 || by >= p.nb[1]) continue;
      for (int ox = -p.sr[0]; ox <= p.sr[0]; ++ox) {
        int bx = c0 + ox, ix = 0;
        if (p.pbc[0]) { ix = (bx >= 0) ? bx / p.nb[0] : -((-bx + p.nb[0] - 1) / p.nb[0]); bx -= ix * p.nb[0]; }
        else if (bx < 0 || bx >= p.nb[0]) continue;
        // image offset in cartesian coordinates: img @ cell (exact for an orthorhombic cell)
        double sx, sy, sz;
        if (p.orthorhombic) {
          sx = dmul((double)ix, p.diag[0]); sy = dmul((double)iy, p.diag[1]); sz = dmul((double)iz, p.diag[2]);
        } else {
          sx = dadd(dadd(dmul((double)ix, p.cell[0]), dmul((double)iy, p.cell[3])), dmul((double)iz, p.cell[6]));
          sy = dadd(dadd(dmul((double)ix, p.cell[1]), dmul((double)iy, p.cell[4])), dmul((double)iz, p.cell[7]));
          sz = dadd(dadd(dmul((double)ix, p.cell[2]), dmul((double)iy, p.cell[5])), dmul((double)iz, p.cell[8]));
        }
        const int64_t b = ((int64_t)bz * p.nb[1] + by) * p.nb[0] + bx;
        const bool home = (ix == 0) && (iy == 0) && (iz == 0);
        for (int64_t q = bin_start[b]; q < bin_start[b + 1]; ++q) {
          const int64_t j = order[q];
          if (home && j == i) continue;
          const double dx = dadd(dadd(wpos[3 * j], sx), -xi), dy = dadd(dadd(wpos[3 * j + 1], sy), -yi),
                       dz = dadd(dadd(wpos[3 * j + 2], sz), -zi);
          const double d2 = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
          if (kTyped ? d2 < rc2_i[ty.types[j]] : d2 < p.r2) f(j, ix, iy, iz);
        }
      }
    }
  }
}

template <class PS, bool kTyped = false>
__global__ void k_nl_count(PS ps, int64_t N, const double* __restrict__ wpos, const int32_t* __restrict__ cidx,
                           const int64_t* __restrict__ order, const int64_t* __restrict__ bin_start,
                           int64_t* __restrict__ counts, NlTypes ty) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int64_t n = 0;
  nl_visit<kTyped>(nl_p(ps, i), ty, i, wpos, cidx, order, bin_start + nl_bin0(ps, i),
                   [&](int64_t, int, int, int) { ++n; });
  counts[i] = n;
}

__device__ __forceinline__ bool nl_less(int64_t ja, const double* sa, int64_t jb, const double* sb) {
  if (ja != jb) return ja < jb;
  if (sa[0] != sb[0]) return sa[0] < sb[0];
  if (sa[1] != sb[1]) return sa[1] < sb[1];
  return sa[2] < sb[2];
}

// kCapacity = false: the row's edges go to [row_ptr[i], row_ptr[i + 1]) of an exactly sized list (nqb_nl_fill).
// kCapacity = true (nqb_nl_fill_capacity): the row owns [row_ptr_pad[i], row_ptr_pad[i + 1]) of a list of E = capacity
// slots; its real edges come first (same order and shifts as above, none when *overflow is set) and the remaining slots
// hold null edges (i, i, pad_shift).  The trailing parameters are appended so the unpadded variant's code is unchanged.
// With PS = NlBlockPtr or NlFrames (only with kCapacity) the null-edge shift comes from the block (of atom i's frame)
// and the pad_shift argument is not read.
template <bool kCapacity, class PS, bool kTyped = false>
__global__ void k_nl_fill(PS ps, int64_t N, const double* __restrict__ wpos, const int32_t* __restrict__ cidx,
                          const int32_t* __restrict__ base, const int64_t* __restrict__ order,
                          const int64_t* __restrict__ bin_start, const int64_t* __restrict__ row_ptr, int64_t E,
                          int64_t* __restrict__ edge_index, double* __restrict__ shifts,
                          const int32_t* __restrict__ overflow, double3 pad_shift, NlTypes ty) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int64_t beg = row_ptr[i];
  int64_t n = 0;
  int64_t* ej = edge_index + E;  // neighbours (row 1)
  if (!kCapacity || *overflow == 0) {
    nl_visit<kTyped>(nl_p(ps, i), ty, i, wpos, cidx, order, bin_start + nl_bin0(ps, i),
                     [&](int64_t j, int ix, int iy, int iz) {
      // insertion into the sorted prefix of the row (rows hold a few dozen neighbours)
      double s[3] = {(double)(ix + base[3 * j] - base[3 * i]), (double)(iy + base[3 * j + 1] - base[3 * i + 1]),
                     (double)(iz + base[3 * j + 2] - base[3 * i + 2])};
      int64_t q = beg + n;
      while (q > beg && nl_less(j, s, ej[q - 1], shifts + 3 * (q - 1))) {
        ej[q] = ej[q - 1];
        shifts[3 * q] = shifts[3 * (q - 1)]; shifts[3 * q + 1] = shifts[3 * (q - 1) + 1]; shifts[3 * q + 2] = shifts[3 * (q - 1) + 2];
        --q;
      }
      ej[q] = j;
      shifts[3 * q] = s[0]; shifts[3 * q + 1] = s[1]; shifts[3 * q + 2] = s[2];
      edge_index[beg + n] = i;
      ++n;
    });
  }
  if (kCapacity) {
    const int64_t end = row_ptr[i + 1];
    const double3 ps3 = nl_pad_shift(ps, i, pad_shift);
    for (int64_t q = beg + n; q < end; ++q) {
      edge_index[q] = i;
      ej[q] = i;
      shifts[3 * q] = ps3.x; shifts[3 * q + 1] = ps3.y; shifts[3 * q + 2] = ps3.z;
    }
  }
}

// Padded row pointer of the capacity mode (one thread per entry of [0, N]).  E = row_ptr[N] real edges; each row gets
// floor or ceil of (capacity - E) / N null edges: row_ptr_pad[i] = row_ptr[i] + floor((capacity - E) i / N).  When
// E > capacity, every row holds only null edges: row_ptr_pad[i] = floor(capacity i / N).
__global__ void k_nl_pad(int64_t N, int64_t capacity, const int64_t* __restrict__ row_ptr,
                         int64_t* __restrict__ row_ptr_pad, int64_t* __restrict__ num_edges,
                         int32_t* __restrict__ overflow) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > N) return;
  const int64_t E = row_ptr[N];
  const bool over = E > capacity;
  row_ptr_pad[i] = over ? capacity * i / N : row_ptr[i] + (capacity - E) * i / N;
  if (i == 0) {
    *num_edges = E;
    *overflow = over ? 1 : 0;
  }
}

// Bounding box of the open directions (nqb_nl_bbox).  Min / max of the fractional coordinates (nl_frac, the
// arithmetic of k_nl_bin) per CTA, then one atomicMax per CTA and value into work[0..5] on an order-preserving 64-bit
// key: work[d] = max of ~key(fmin_d), work[3 + d] = max of key(fmax_d), so 0 is the identity of all six.  fmin / fmax
// skip NaN coordinates.  The CTA that takes the last ticket (work[6]) reads the six keys back with atomicExch(0),
// writes lo / width / nb / sr of every open direction into the block, as ops.neighbor_list computes them on the host,
// and resets the ticket: the work words are zero again for the next call or graph replay.  Min and max are exact, so
// the result does not depend on the order in which CTAs arrive.
constexpr int kBboxThreads = 256;
constexpr int64_t kBboxMaxBlocks = 264;

__device__ __forceinline__ unsigned long long nl_key(double v) {  // monotone: v < w => key(v) < key(w), -0 < +0
  const unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double nl_unkey(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}

__global__ void __launch_bounds__(kBboxThreads)
k_nl_bbox(NlBlock* __restrict__ b, const double* __restrict__ pos, int64_t N, unsigned long long* __restrict__ acc,
          unsigned int* __restrict__ ticket) {
  const NlParams& p = b->p;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    double f[3];
    nl_frac(p, pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], f);
    for (int d = 0; d < 3; ++d) { lo[d] = fmin(lo[d], f[d]); hi[d] = fmax(hi[d], f[d]); }
  }
  for (int o = 16; o > 0; o >>= 1)
    for (int d = 0; d < 3; ++d) {
      lo[d] = fmin(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmax(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  __shared__ double s[kBboxThreads / 32][6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
    for (int d = 0; d < 3; ++d) { s[warp][d] = lo[d]; s[warp][3 + d] = hi[d]; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kBboxThreads / 32; ++w)
    for (int d = 0; d < 3; ++d) { lo[d] = fmin(lo[d], s[w][d]); hi[d] = fmax(hi[d], s[w][3 + d]); }
  for (int d = 0; d < 3; ++d) {
    atomicMax(acc + d, ~nl_key(lo[d]));
    atomicMax(acc + 3 + d, nl_key(hi[d]));
  }
  __threadfence();
  if (atomicAdd(ticket, 1u) != gridDim.x - 1) return;
  __threadfence();
  for (int d = 0; d < 3; ++d) {
    const double fmin_d = nl_unkey(~atomicExch(acc + d, 0ull)), fmax_d = nl_unkey(atomicExch(acc + 3 + d, 0ull));
    if (!b->open[d]) continue;
    // width = max(fmax - fmin, 1e-9) (1 + 1e-9); a NaN or -inf difference (no finite coordinate) takes 1e-9
    double w = dadd(fmax_d, -fmin_d);
    w = dmul(w > 1e-9 ? w : 1e-9, 1.0 + 1e-9);
    // nb = min(cap, max(1, floor(perp * width / r_max))), in [1, cap] for any width (NaN gives 1, inf gives cap)
    const double t = floor(__ddiv_rn(dmul(b->perp[d], w), b->r_max));
    b->p.lo[d] = fmin_d;
    b->p.width[d] = w;
    b->p.nb[d] = t >= 1.0 ? (t < (double)b->cap ? (int)t : b->cap) : 1;
    b->p.sr[d] = 1;
  }
  atomicExch(ticket, 0u);
}

// Bounding boxes of a batch of frames (nqb_nl_bbox_frames): CTA f reduces the fractional coordinates (nl_frac) of its
// frame's atoms [atom_ptr[f], atom_ptr[f + 1]) and writes lo / width / nb / sr of every open direction of blocks[f]
// with the formulas of k_nl_bbox.  One CTA owns one block, so there are no atomics and no work words, and the grid
// depends on F only (capturable).  A frame without open directions or without atoms keeps its packed block.
__global__ void __launch_bounds__(kBboxThreads)
k_nl_bbox_frames(NlBlock* __restrict__ blocks, const double* __restrict__ pos, const int64_t* __restrict__ atom_ptr) {
  NlBlock* b = blocks + blockIdx.x;
  const int64_t beg = atom_ptr[blockIdx.x], end = atom_ptr[blockIdx.x + 1];
  if (!(b->open[0] || b->open[1] || b->open[2]) || end <= beg) return;
  const NlParams& p = b->p;
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t i = beg + threadIdx.x; i < end; i += blockDim.x) {
    double f[3];
    nl_frac(p, pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], f);
    for (int d = 0; d < 3; ++d) { lo[d] = fmin(lo[d], f[d]); hi[d] = fmax(hi[d], f[d]); }
  }
  for (int o = 16; o > 0; o >>= 1)
    for (int d = 0; d < 3; ++d) {
      lo[d] = fmin(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmax(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  __shared__ double s[kBboxThreads / 32][6];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
    for (int d = 0; d < 3; ++d) { s[warp][d] = lo[d]; s[warp][3 + d] = hi[d]; }
  __syncthreads();  // every thread's reads of the block precede thread 0's writes
  if (threadIdx.x != 0) return;
  for (int w = 1; w < kBboxThreads / 32; ++w)
    for (int d = 0; d < 3; ++d) { lo[d] = fmin(lo[d], s[w][d]); hi[d] = fmax(hi[d], s[w][3 + d]); }
  for (int d = 0; d < 3; ++d) {
    if (!b->open[d]) continue;
    double w = dadd(hi[d], -lo[d]);
    w = dmul(w > 1e-9 ? w : 1e-9, 1.0 + 1e-9);
    const double t = floor(__ddiv_rn(dmul(b->perp[d], w), b->r_max));
    b->p.lo[d] = lo[d];
    b->p.width[d] = w;
    b->p.nb[d] = t >= 1.0 ? (t < (double)b->cap ? (int)t : b->cap) : 1;
    b->p.sr[d] = 1;
  }
}

// Cells of a batched variable-cell plan packed on the device (nqb_nl_frames_set_cells): thread f rewrites the fields of
// blocks[f] that the host pack derives from the cell -- cell, inverse, diag / orthorhombic, perp, the search range on
// the block's fixed grid and the null-edge shift -- with the host's formulas in the host's order of operations
// (ops._NlArgs, ops.null_edge_shift; explicitly rounded, no FMA).  The inverse is the adjugate over the determinant,
// so it may differ from the host's LU inverse by a few ulp.  A non-finite or singular cell (ops._nl_check_cell:
// |det| <= 1e-12 |a_0| |a_1| |a_2|) leaves the block untouched and sets bad[f] = 1.
__global__ void k_nl_frames_set_cells(int F, const double* __restrict__ cells, NlBlock* __restrict__ blocks,
                                      int32_t* __restrict__ bad) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double c[9];
  bool finite = true;
  for (int k = 0; k < 9; ++k) {
    c[k] = cells[9 * (int64_t)f + k];
    finite = finite && isfinite(c[k]);
  }
  double len[3];
  for (int d = 0; d < 3; ++d)
    len[d] = sqrt(dadd(dadd(dmul(c[3 * d], c[3 * d]), dmul(c[3 * d + 1], c[3 * d + 1])), dmul(c[3 * d + 2], c[3 * d + 2])));
  // adjugate (transposed cofactors) and determinant
  double adj[9];
  adj[0] = dadd(dmul(c[4], c[8]), -dmul(c[5], c[7]));
  adj[1] = dadd(dmul(c[2], c[7]), -dmul(c[1], c[8]));
  adj[2] = dadd(dmul(c[1], c[5]), -dmul(c[2], c[4]));
  adj[3] = dadd(dmul(c[5], c[6]), -dmul(c[3], c[8]));
  adj[4] = dadd(dmul(c[0], c[8]), -dmul(c[2], c[6]));
  adj[5] = dadd(dmul(c[2], c[3]), -dmul(c[0], c[5]));
  adj[6] = dadd(dmul(c[3], c[7]), -dmul(c[4], c[6]));
  adj[7] = dadd(dmul(c[1], c[6]), -dmul(c[0], c[7]));
  adj[8] = dadd(dmul(c[0], c[4]), -dmul(c[1], c[3]));
  const double det = dadd(dadd(dmul(c[0], adj[0]), dmul(c[1], adj[3])), dmul(c[2], adj[6]));
  if (!finite || !(fabs(det) > dmul(1e-12, dmul(dmul(len[0], len[1]), len[2])))) {
    bad[f] = 1;
    return;
  }
  NlBlock* b = blocks + f;
  NlParams& p = b->p;
  bool ortho = true;
  for (int k = 0; k < 9; ++k) {
    p.cell[k] = c[k];
    p.inv[k] = __ddiv_rn(adj[k], det);
    if ((k % 4) != 0 && c[k] != 0.0) ortho = false;
  }
  p.orthorhombic = ortho ? 1 : 0;
  int dmax = 0;
  double lmax = len[0];
  for (int d = 0; d < 3; ++d) {
    p.diag[d] = c[4 * d];
    const double* inv = p.inv;
    const double nrm = sqrt(dadd(dadd(dmul(inv[d], inv[d]), dmul(inv[3 + d], inv[3 + d])), dmul(inv[6 + d], inv[6 + d])));
    b->perp[d] = __ddiv_rn(1.0, nrm);
    const double sr = ceil(dadd(__ddiv_rn(b->r_max, __ddiv_rn(b->perp[d], (double)p.nb[d])), -1e-12));
    p.sr[d] = sr > 1.0 ? (int)sr : 1;
    if (len[d] > lmax) {  // the first longest, as numpy's argmax
      dmax = d;
      lmax = len[d];
    }
  }
  for (int d = 0; d < 3; ++d) b->pad_shift[d] = d == dmax ? floor(__ddiv_rn(b->r_max, lmax)) + 2.0 : 0.0;
}

}  // namespace

// Step 1: bins.  cell/inv: row-major 3x3 on the HOST (9 doubles each); nbins/search: per direction.
extern "C" int nqb_nl_bin(const double* pos, int64_t N, const double* cell_host, const double* inv_host, const int* pbc,
                          const int* nbins, const int* search, const double* lo, const double* width, double r_max,
                          double* wpos, int32_t* base, int64_t* bin, int32_t* cidx, nqb_stream_t st) {
  if (N < 0) return nqb_set_error("nqb_nl_bin: negative size");
  if (N == 0) return 0;
  if (!pos || !cell_host || !inv_host || !pbc || !nbins || !search || !wpos || !base || !bin || !cidx)
    return nqb_set_error("nqb_nl_bin: null pointer");
  NlParams p;
  bool ortho = true;
  for (int k = 0; k < 9; ++k) { p.cell[k] = cell_host[k]; p.inv[k] = inv_host[k]; if ((k % 4) != 0 && cell_host[k] != 0.0) ortho = false; }
  p.orthorhombic = ortho ? 1 : 0;
  for (int d = 0; d < 3; ++d) {
    p.diag[d] = cell_host[4 * d]; p.pbc[d] = pbc[d]; p.nb[d] = nbins[d]; p.sr[d] = search[d];
    p.lo[d] = lo ? lo[d] : 0.0; p.width[d] = width ? width[d] : 1.0;
    if (nbins[d] < 1 || search[d] < 0) return nqb_set_error("nqb_nl_bin: bad bin grid");
  }
  p.r2 = r_max * r_max;
  k_nl_bin<NlParams><<<(unsigned)((N + 127) / 128), 128, 0, (cudaStream_t)st>>>(p, pos, N, wpos, base, bin, cidx);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

static int nl_params(const double* cell_host, const double* inv_host, const int* pbc, const int* nbins, const int* search,
                     double r_max, NlParams& p) {
  bool ortho = true;
  for (int k = 0; k < 9; ++k) { p.cell[k] = cell_host[k]; p.inv[k] = inv_host[k]; if ((k % 4) != 0 && cell_host[k] != 0.0) ortho = false; }
  p.orthorhombic = ortho ? 1 : 0;
  for (int d = 0; d < 3; ++d) {
    p.diag[d] = cell_host[4 * d]; p.pbc[d] = pbc[d]; p.nb[d] = nbins[d]; p.sr[d] = search[d]; p.lo[d] = 0.0; p.width[d] = 1.0;
  }
  p.r2 = r_max * r_max;
  return 0;
}

// Step 2: neighbours per atom.  order = atom ids sorted by bin, bin_start [nbins + 1].
extern "C" int nqb_nl_count(int64_t N, const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                            const int* search, double r_max, const double* wpos, const int32_t* cidx,
                            const int64_t* order, const int64_t* bin_start, int64_t* counts, nqb_stream_t st) {
  if (N <= 0) return 0;
  if (!wpos || !cidx || !order || !bin_start || !counts) return nqb_set_error("nqb_nl_count: null pointer");
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  k_nl_count<NlParams><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(p, N, wpos, cidx, order, bin_start, counts,
                                                                                NlTypes{});
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Step 3: fill.  row_ptr [N + 1] = exclusive scan of counts; edge_index [2, E] (row 0 = centre i, row 1 = neighbour j,
// sorted by (i, j, shift)); shifts [E, 3] (integer-valued doubles): pos[j] - pos[i] + shifts @ cell is the edge vector.
extern "C" int nqb_nl_fill(int64_t N, int64_t E, const double* cell_host, const double* inv_host, const int* pbc,
                           const int* nbins, const int* search, double r_max, const double* wpos, const int32_t* cidx,
                           const int32_t* base, const int64_t* order, const int64_t* bin_start, const int64_t* row_ptr,
                           int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || E <= 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr || !edge_index || !shifts)
    return nqb_set_error("nqb_nl_fill: null pointer");
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  k_nl_fill<false, NlParams><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      p, N, wpos, cidx, base, order, bin_start, row_ptr, E, edge_index, shifts, nullptr, make_double3(0.0, 0.0, 0.0),
      NlTypes{});
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Capacity mode, step 3a: padded row pointer, true edge count and overflow flag from the exact row pointer.
extern "C" int nqb_nl_pad(int64_t N, int64_t capacity, const int64_t* row_ptr, int64_t* row_ptr_pad, int64_t* num_edges,
                          int32_t* overflow, nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_pad: needs N > 0 and capacity >= 0");
  if (!row_ptr || !row_ptr_pad || !num_edges || !overflow) return nqb_set_error("nqb_nl_pad: null pointer");
  k_nl_pad<<<(unsigned)((N + 1 + 127) / 128), 128, 0, (cudaStream_t)st>>>(N, capacity, row_ptr, row_ptr_pad, num_edges,
                                                                          overflow);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Capacity mode, step 3b: fill a [2, capacity] list along row_ptr_pad (from nqb_nl_pad); pad_shift: 3 doubles on the HOST.
extern "C" int nqb_nl_fill_capacity(int64_t N, int64_t capacity, const double* cell_host, const double* inv_host,
                                    const int* pbc, const int* nbins, const int* search, double r_max, const double* wpos,
                                    const int32_t* cidx, const int32_t* base, const int64_t* order,
                                    const int64_t* bin_start, const int64_t* row_ptr_pad, const int32_t* overflow,
                                    const double* pad_shift_host, int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_fill_capacity: needs N > 0 and capacity >= 0");
  if (capacity == 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr_pad || !overflow || !pad_shift_host || !edge_index ||
      !shifts)
    return nqb_set_error("nqb_nl_fill_capacity: null pointer");
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  const double3 ps = make_double3(pad_shift_host[0], pad_shift_host[1], pad_shift_host[2]);
  k_nl_fill<true, NlParams><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      p, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts, overflow, ps, NlTypes{});
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Variable cell: the same three kernels reading their parameters from a block in device memory, so that a captured
// graph follows a cell that changes between replays.  The block is built on the host by nqb_nl_params_pack (the
// helper above, so the orthorhombic test and every field match the by-value path) and copied in by the caller.
extern "C" int64_t nqb_nl_params_bytes(void) { return (int64_t)sizeof(NlBlock); }

extern "C" int nqb_nl_params_pack(const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                                  const int* search, double r_max, const double* pad_shift_host, void* out_host) {
  if (!cell_host || !inv_host || !pbc || !nbins || !search || !pad_shift_host || !out_host)
    return nqb_set_error("nqb_nl_params_pack: null pointer");
  for (int d = 0; d < 3; ++d) {
    if (!pbc[d]) return nqb_set_error("nqb_nl_params_pack: every direction must be periodic");
    if (nbins[d] < 1 || search[d] < 0) return nqb_set_error("nqb_nl_params_pack: bad bin grid");
  }
  NlBlock b;
  memset(&b, 0, sizeof(b));
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, b.p);
  for (int d = 0; d < 3; ++d) b.pad_shift[d] = pad_shift_host[d];
  memcpy(out_host, &b, sizeof(b));
  return 0;
}

static int nl_launch_done();

// Open directions: the block of nqb_nl_params_pack with the directions where pbc[d] == 0 marked open.  Their
// lo / width / nb / sr are left for nqb_nl_bbox (a valid one-bin grid until then); cap, perp and r_max are what it
// derives the grid from.
extern "C" int nqb_nl_params_pack_open(const double* cell_host, const double* inv_host, const int* pbc,
                                       const int* nbins, const int* search, double r_max, const double* pad_shift_host,
                                       int cap, const double* perp_host, void* out_host) {
  if (!cell_host || !inv_host || !pbc || !nbins || !search || !pad_shift_host || !perp_host || !out_host)
    return nqb_set_error("nqb_nl_params_pack_open: null pointer");
  if (cap < 1 || !(r_max > 0.0) || !isfinite(r_max))
    return nqb_set_error("nqb_nl_params_pack_open: needs cap >= 1 and a finite r_max > 0");
  for (int d = 0; d < 3; ++d) {
    if (pbc[d] && (nbins[d] < 1 || search[d] < 0)) return nqb_set_error("nqb_nl_params_pack_open: bad bin grid");
    if (!(perp_host[d] > 0.0) || !isfinite(perp_host[d]))
      return nqb_set_error("nqb_nl_params_pack_open: perpendicular widths must be finite and positive");
  }
  NlBlock b;
  memset(&b, 0, sizeof(b));
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, b.p);
  for (int d = 0; d < 3; ++d) {
    b.pad_shift[d] = pad_shift_host[d];
    b.open[d] = pbc[d] ? 0 : 1;
    if (!pbc[d]) { b.p.nb[d] = 1; b.p.sr[d] = 1; }
    b.perp[d] = perp_host[d];
  }
  b.cap = cap;
  b.r_max = r_max;
  memcpy(out_host, &b, sizeof(b));
  return 0;
}

extern "C" int nqb_nl_bbox(const double* pos, int64_t N, void* params_dev, uint64_t* work, nqb_stream_t st) {
  if (N < 0) return nqb_set_error("nqb_nl_bbox: negative size");
  if (N == 0) return 0;
  if (!pos || !params_dev || !work) return nqb_set_error("nqb_nl_bbox: null pointer");
  int64_t blocks = (N + kBboxThreads - 1) / kBboxThreads;
  if (blocks > kBboxMaxBlocks) blocks = kBboxMaxBlocks;
  k_nl_bbox<<<(unsigned)blocks, kBboxThreads, 0, (cudaStream_t)st>>>(
      (NlBlock*)params_dev, pos, N, (unsigned long long*)work, (unsigned int*)(work + 6));
  return nl_launch_done();
}

extern "C" int nqb_nl_bin_dp(const double* pos, int64_t N, const void* params_dev, double* wpos, int32_t* base,
                             int64_t* bin, int32_t* cidx, nqb_stream_t st) {
  if (N < 0) return nqb_set_error("nqb_nl_bin_dp: negative size");
  if (N == 0) return 0;
  if (!pos || !params_dev || !wpos || !base || !bin || !cidx) return nqb_set_error("nqb_nl_bin_dp: null pointer");
  k_nl_bin<NlBlockPtr><<<(unsigned)((N + 127) / 128), 128, 0, (cudaStream_t)st>>>(
      (const NlBlock*)params_dev, pos, N, wpos, base, bin, cidx);
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_nl_count_dp(int64_t N, const void* params_dev, const double* wpos, const int32_t* cidx,
                               const int64_t* order, const int64_t* bin_start, int64_t* counts, nqb_stream_t st) {
  if (N <= 0) return 0;
  if (!params_dev || !wpos || !cidx || !order || !bin_start || !counts)
    return nqb_set_error("nqb_nl_count_dp: null pointer");
  k_nl_count<NlBlockPtr><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      (const NlBlock*)params_dev, N, wpos, cidx, order, bin_start, counts, NlTypes{});
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_nl_fill_capacity_dp(int64_t N, int64_t capacity, const void* params_dev, const double* wpos,
                                       const int32_t* cidx, const int32_t* base, const int64_t* order,
                                       const int64_t* bin_start, const int64_t* row_ptr_pad, const int32_t* overflow,
                                       int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_fill_capacity_dp: needs N > 0 and capacity >= 0");
  if (capacity == 0) return 0;
  if (!params_dev || !wpos || !cidx || !base || !order || !bin_start || !row_ptr_pad || !overflow || !edge_index ||
      !shifts)
    return nqb_set_error("nqb_nl_fill_capacity_dp: null pointer");
  k_nl_fill<true, NlBlockPtr><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      (const NlBlock*)params_dev, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts,
      overflow, make_double3(0.0, 0.0, 0.0), NlTypes{});
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

// Per-edge-type cutoffs: nqb_nl_count, nqb_nl_fill, nqb_nl_fill_capacity and their _dp forms with the membership test
// d2 < rc2[T * types[i] + types[j]].  types [N] i64 in [0, T) and rc2 [T * T] f64 (rc * rc, every rc <= r_max) are
// device arrays; the bins, search ranges and parameter blocks are those of r_max.
static int nl_types(const char* what, const int64_t* types, const double* rc2, int T, NlTypes& ty) {
  if (T < 1 || !types || !rc2) {
    static thread_local char msg[160];
    snprintf(msg, sizeof(msg), "%s: needs types, rc2 and T >= 1", what);
    return nqb_set_error(msg);
  }
  ty = NlTypes{types, rc2, T};
  return 0;
}

static int nl_launch_done() {
  nqb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return nqb_set_error(cudaGetErrorString(e));
  return 0;
}

extern "C" int nqb_nl_count_typed(int64_t N, const double* cell_host, const double* inv_host, const int* pbc,
                                  const int* nbins, const int* search, double r_max, const double* wpos,
                                  const int32_t* cidx, const int64_t* order, const int64_t* bin_start,
                                  const int64_t* types, const double* rc2, int T, int64_t* counts, nqb_stream_t st) {
  if (N <= 0) return 0;
  if (!wpos || !cidx || !order || !bin_start || !counts) return nqb_set_error("nqb_nl_count_typed: null pointer");
  NlTypes ty;
  if (int rc = nl_types("nqb_nl_count_typed", types, rc2, T, ty)) return rc;
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  k_nl_count<NlParams, true><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(p, N, wpos, cidx, order, bin_start,
                                                                                      counts, ty);
  return nl_launch_done();
}

extern "C" int nqb_nl_fill_typed(int64_t N, int64_t E, const double* cell_host, const double* inv_host, const int* pbc,
                                 const int* nbins, const int* search, double r_max, const double* wpos,
                                 const int32_t* cidx, const int32_t* base, const int64_t* order,
                                 const int64_t* bin_start, const int64_t* row_ptr, const int64_t* types,
                                 const double* rc2, int T, int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || E <= 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr || !edge_index || !shifts)
    return nqb_set_error("nqb_nl_fill_typed: null pointer");
  NlTypes ty;
  if (int rc = nl_types("nqb_nl_fill_typed", types, rc2, T, ty)) return rc;
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  k_nl_fill<false, NlParams, true><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      p, N, wpos, cidx, base, order, bin_start, row_ptr, E, edge_index, shifts, nullptr, make_double3(0.0, 0.0, 0.0), ty);
  return nl_launch_done();
}

extern "C" int nqb_nl_fill_capacity_typed(int64_t N, int64_t capacity, const double* cell_host, const double* inv_host,
                                          const int* pbc, const int* nbins, const int* search, double r_max,
                                          const double* wpos, const int32_t* cidx, const int32_t* base,
                                          const int64_t* order, const int64_t* bin_start, const int64_t* row_ptr_pad,
                                          const int32_t* overflow, const double* pad_shift_host, const int64_t* types,
                                          const double* rc2, int T, int64_t* edge_index, double* shifts,
                                          nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_fill_capacity_typed: needs N > 0 and capacity >= 0");
  if (capacity == 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr_pad || !overflow || !pad_shift_host || !edge_index ||
      !shifts)
    return nqb_set_error("nqb_nl_fill_capacity_typed: null pointer");
  NlTypes ty;
  if (int rc = nl_types("nqb_nl_fill_capacity_typed", types, rc2, T, ty)) return rc;
  NlParams p;
  nl_params(cell_host, inv_host, pbc, nbins, search, r_max, p);
  const double3 ps = make_double3(pad_shift_host[0], pad_shift_host[1], pad_shift_host[2]);
  k_nl_fill<true, NlParams, true><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      p, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts, overflow, ps, ty);
  return nl_launch_done();
}

extern "C" int nqb_nl_count_dp_typed(int64_t N, const void* params_dev, const double* wpos, const int32_t* cidx,
                                     const int64_t* order, const int64_t* bin_start, const int64_t* types,
                                     const double* rc2, int T, int64_t* counts, nqb_stream_t st) {
  if (N <= 0) return 0;
  if (!params_dev || !wpos || !cidx || !order || !bin_start || !counts)
    return nqb_set_error("nqb_nl_count_dp_typed: null pointer");
  NlTypes ty;
  if (int rc = nl_types("nqb_nl_count_dp_typed", types, rc2, T, ty)) return rc;
  k_nl_count<NlBlockPtr, true><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      (const NlBlock*)params_dev, N, wpos, cidx, order, bin_start, counts, ty);
  return nl_launch_done();
}

extern "C" int nqb_nl_fill_capacity_dp_typed(int64_t N, int64_t capacity, const void* params_dev, const double* wpos,
                                             const int32_t* cidx, const int32_t* base, const int64_t* order,
                                             const int64_t* bin_start, const int64_t* row_ptr_pad,
                                             const int32_t* overflow, const int64_t* types, const double* rc2, int T,
                                             int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_fill_capacity_dp_typed: needs N > 0 and capacity >= 0");
  if (capacity == 0) return 0;
  if (!params_dev || !wpos || !cidx || !base || !order || !bin_start || !row_ptr_pad || !overflow || !edge_index ||
      !shifts)
    return nqb_set_error("nqb_nl_fill_capacity_dp_typed: null pointer");
  NlTypes ty;
  if (int rc = nl_types("nqb_nl_fill_capacity_dp_typed", types, rc2, T, ty)) return rc;
  k_nl_fill<true, NlBlockPtr, true><<<(unsigned)((N + 63) / 64), 64, 0, (cudaStream_t)st>>>(
      (const NlBlock*)params_dev, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts,
      overflow, make_double3(0.0, 0.0, 0.0), ty);
  return nl_launch_done();
}

// A batch of frames: bin, count and fill of the exact list with the parameters of atom i read from
// blocks[batch[i]] and its bins offset by bin_base[batch[i]] (NlFrames).  batch [N] i64 is non-decreasing in [0, F),
// bin_base [F + 1] i64 the exclusive scan of the frames' bin counts; the sort, searchsorted and scan between the
// steps run once over the global bin range.  Per-edge-type cutoffs when types / rc2 are given (T >= 1), none when
// both are NULL.  The blocks come from nqb_nl_frames_pack and are copied to the device by the caller.
extern "C" int nqb_nl_frames_pack(int F, const double* cell_host, const double* inv_host, const int* pbc,
                                  const int* nbins, const int* search, const double* lo, const double* width,
                                  double r_max, void* out_host) {
  if (F < 0) return nqb_set_error("nqb_nl_frames_pack: negative frame count");
  if (F > 0 && (!cell_host || !inv_host || !pbc || !nbins || !search || !lo || !width || !out_host))
    return nqb_set_error("nqb_nl_frames_pack: null pointer");
  for (int f = 0; f < F; ++f) {
    NlBlock b;
    memset(&b, 0, sizeof(b));
    for (int d = 0; d < 3; ++d)
      if (nbins[3 * f + d] < 1 || search[3 * f + d] < 0) return nqb_set_error("nqb_nl_frames_pack: bad bin grid");
    // the fields nqb_nl_bin (lo / width) and nqb_nl_count / nqb_nl_fill (the rest) build for this frame
    nl_params(cell_host + 9 * f, inv_host + 9 * f, pbc + 3 * f, nbins + 3 * f, search + 3 * f, r_max, b.p);
    for (int d = 0; d < 3; ++d) { b.p.lo[d] = lo[3 * f + d]; b.p.width[d] = width[3 * f + d]; }
    memcpy((char*)out_host + (size_t)f * sizeof(NlBlock), &b, sizeof(b));
  }
  return 0;
}

static int nl_frames(const char* what, const void* blocks_dev, const int64_t* batch, const int64_t* bin_base,
                     NlFrames& fr) {
  if (!blocks_dev || !batch || !bin_base) {
    static thread_local char msg[160];
    snprintf(msg, sizeof(msg), "%s: null blocks / batch / bin_base", what);
    return nqb_set_error(msg);
  }
  fr = NlFrames{(const NlBlock*)blocks_dev, batch, bin_base};
  return 0;
}

static int nl_types_opt(const char* what, const int64_t* types, const double* rc2, int T, NlTypes& ty) {
  if (!types && !rc2) { ty = NlTypes{}; return 0; }
  return nl_types(what, types, rc2, T, ty);
}

extern "C" int nqb_nl_bin_frames(const double* pos, int64_t N, const void* blocks_dev, const int64_t* batch,
                                 const int64_t* bin_base, double* wpos, int32_t* base, int64_t* bin, int32_t* cidx,
                                 nqb_stream_t st) {
  if (N < 0) return nqb_set_error("nqb_nl_bin_frames: negative size");
  if (N == 0) return 0;
  if (!pos || !wpos || !base || !bin || !cidx) return nqb_set_error("nqb_nl_bin_frames: null pointer");
  NlFrames fr;
  if (int rc = nl_frames("nqb_nl_bin_frames", blocks_dev, batch, bin_base, fr)) return rc;
  k_nl_bin<NlFrames><<<(unsigned)((N + 127) / 128), 128, 0, (cudaStream_t)st>>>(fr, pos, N, wpos, base, bin, cidx);
  return nl_launch_done();
}

extern "C" int nqb_nl_count_frames(int64_t N, const void* blocks_dev, const int64_t* batch, const int64_t* bin_base,
                                   const double* wpos, const int32_t* cidx, const int64_t* order,
                                   const int64_t* bin_start, const int64_t* types, const double* rc2, int T,
                                   int64_t* counts, nqb_stream_t st) {
  if (N <= 0) return 0;
  if (!wpos || !cidx || !order || !bin_start || !counts) return nqb_set_error("nqb_nl_count_frames: null pointer");
  NlFrames fr;
  if (int rc = nl_frames("nqb_nl_count_frames", blocks_dev, batch, bin_base, fr)) return rc;
  NlTypes ty;
  if (int rc = nl_types_opt("nqb_nl_count_frames", types, rc2, T, ty)) return rc;
  const unsigned blocks = (unsigned)((N + 63) / 64);
  if (ty.types)
    k_nl_count<NlFrames, true><<<blocks, 64, 0, (cudaStream_t)st>>>(fr, N, wpos, cidx, order, bin_start, counts, ty);
  else
    k_nl_count<NlFrames><<<blocks, 64, 0, (cudaStream_t)st>>>(fr, N, wpos, cidx, order, bin_start, counts, ty);
  return nl_launch_done();
}

extern "C" int nqb_nl_fill_frames(int64_t N, int64_t E, const void* blocks_dev, const int64_t* batch,
                                  const int64_t* bin_base, const double* wpos, const int32_t* cidx,
                                  const int32_t* base, const int64_t* order, const int64_t* bin_start,
                                  const int64_t* row_ptr, const int64_t* types, const double* rc2, int T,
                                  int64_t* edge_index, double* shifts, nqb_stream_t st) {
  if (N <= 0 || E <= 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr || !edge_index || !shifts)
    return nqb_set_error("nqb_nl_fill_frames: null pointer");
  NlFrames fr;
  if (int rc = nl_frames("nqb_nl_fill_frames", blocks_dev, batch, bin_base, fr)) return rc;
  NlTypes ty;
  if (int rc = nl_types_opt("nqb_nl_fill_frames", types, rc2, T, ty)) return rc;
  const unsigned blocks = (unsigned)((N + 63) / 64);
  const double3 zero = make_double3(0.0, 0.0, 0.0);
  if (ty.types)
    k_nl_fill<false, NlFrames, true><<<blocks, 64, 0, (cudaStream_t)st>>>(
        fr, N, wpos, cidx, base, order, bin_start, row_ptr, E, edge_index, shifts, nullptr, zero, ty);
  else
    k_nl_fill<false, NlFrames><<<blocks, 64, 0, (cudaStream_t)st>>>(
        fr, N, wpos, cidx, base, order, bin_start, row_ptr, E, edge_index, shifts, nullptr, zero, ty);
  return nl_launch_done();
}

// Capacity mode for a batch of frames (NeighborListPlan with batch=).  nqb_nl_frames_pack_capacity: the blocks of
// nqb_nl_frames_pack, plus each frame's null-edge shift (pad_shift [F,3]) and the fields of nqb_nl_params_pack_open:
// open[d] = !pbc[3f + d], cap [F] (most bins along frame f's open directions), perp [F,3], r_max.
extern "C" int nqb_nl_frames_pack_capacity(int F, const double* cell_host, const double* inv_host, const int* pbc,
                                           const int* nbins, const int* search, const double* lo, const double* width,
                                           double r_max, const double* pad_shift_host, const int* cap,
                                           const double* perp_host, void* out_host) {
  if (F < 0) return nqb_set_error("nqb_nl_frames_pack_capacity: negative frame count");
  if (F > 0 && (!pad_shift_host || !cap || !perp_host)) return nqb_set_error("nqb_nl_frames_pack_capacity: null pointer");
  if (!(r_max > 0.0) || !isfinite(r_max)) return nqb_set_error("nqb_nl_frames_pack_capacity: needs a finite r_max > 0");
  for (int f = 0; f < F; ++f) {
    if (cap[f] < 1) return nqb_set_error("nqb_nl_frames_pack_capacity: needs cap >= 1");
    for (int d = 0; d < 3; ++d)
      if (!(perp_host[3 * f + d] > 0.0) || !isfinite(perp_host[3 * f + d]))
        return nqb_set_error("nqb_nl_frames_pack_capacity: perpendicular widths must be finite and positive");
  }
  if (int rc = nqb_nl_frames_pack(F, cell_host, inv_host, pbc, nbins, search, lo, width, r_max, out_host)) return rc;
  for (int f = 0; f < F; ++f) {
    NlBlock* b = (NlBlock*)((char*)out_host + (size_t)f * sizeof(NlBlock));
    for (int d = 0; d < 3; ++d) {
      b->pad_shift[d] = pad_shift_host[3 * f + d];
      b->open[d] = pbc[3 * f + d] ? 0 : 1;
      b->perp[d] = perp_host[3 * f + d];
    }
    b->cap = cap[f];
    b->r_max = r_max;
  }
  return 0;
}

extern "C" int nqb_nl_bbox_frames(const double* pos, int F, const int64_t* atom_ptr, void* blocks_dev,
                                  nqb_stream_t st) {
  if (F < 0) return nqb_set_error("nqb_nl_bbox_frames: negative frame count");
  if (F == 0) return 0;
  if (!pos || !atom_ptr || !blocks_dev) return nqb_set_error("nqb_nl_bbox_frames: null pointer");
  k_nl_bbox_frames<<<(unsigned)F, kBboxThreads, 0, (cudaStream_t)st>>>((NlBlock*)blocks_dev, pos, atom_ptr);
  return nl_launch_done();
}

extern "C" int nqb_nl_frames_set_cells(int F, const double* cells, void* blocks_dev, int32_t* bad, nqb_stream_t st) {
  if (F < 0) return nqb_set_error("nqb_nl_frames_set_cells: negative frame count");
  if (F == 0) return 0;
  if (!cells || !blocks_dev || !bad) return nqb_set_error("nqb_nl_frames_set_cells: null pointer");
  k_nl_frames_set_cells<<<(unsigned)((F + 127) / 128), 128, 0, (cudaStream_t)st>>>(F, cells, (NlBlock*)blocks_dev, bad);
  return nl_launch_done();
}

extern "C" int nqb_nl_fill_capacity_frames(int64_t N, int64_t capacity, const void* blocks_dev, const int64_t* batch,
                                           const int64_t* bin_base, const double* wpos, const int32_t* cidx,
                                           const int32_t* base, const int64_t* order, const int64_t* bin_start,
                                           const int64_t* row_ptr_pad, const int32_t* overflow, const int64_t* types,
                                           const double* rc2, int T, int64_t* edge_index, double* shifts,
                                           nqb_stream_t st) {
  if (N <= 0 || capacity < 0) return nqb_set_error("nqb_nl_fill_capacity_frames: needs N > 0 and capacity >= 0");
  if (capacity == 0) return 0;
  if (!wpos || !cidx || !base || !order || !bin_start || !row_ptr_pad || !overflow || !edge_index || !shifts)
    return nqb_set_error("nqb_nl_fill_capacity_frames: null pointer");
  NlFrames fr;
  if (int rc = nl_frames("nqb_nl_fill_capacity_frames", blocks_dev, batch, bin_base, fr)) return rc;
  NlTypes ty;
  if (int rc = nl_types_opt("nqb_nl_fill_capacity_frames", types, rc2, T, ty)) return rc;
  const unsigned blocks = (unsigned)((N + 63) / 64);
  const double3 zero = make_double3(0.0, 0.0, 0.0);
  if (ty.types)
    k_nl_fill<true, NlFrames, true><<<blocks, 64, 0, (cudaStream_t)st>>>(
        fr, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts, overflow, zero, ty);
  else
    k_nl_fill<true, NlFrames><<<blocks, 64, 0, (cudaStream_t)st>>>(
        fr, N, wpos, cidx, base, order, bin_start, row_ptr_pad, capacity, edge_index, shifts, overflow, zero, ty);
  return nl_launch_done();
}
