// Device-side vocabulary shared by every generated tensor-product kernel
// (nequip_b200/codegen.py).  fp32 kernels work on channel PAIRS held in a float2 so
// that every operation covers two channels (fma2_rn / fmul2_rn); fp64 kernels are scalar.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

// ---- lane geometry traits are emitted per signature: VT<T>::{V, CPT, LPE, EPW, CB}
template <typename T> struct VT;

// ---- construction ---------------------------------------------------------------
__device__ __forceinline__ float2 vsplat(float a) { return make_float2(a, a); }
__device__ __forceinline__ double vsplat(double a) { return a; }
template <typename T> __device__ __forceinline__ typename VT<T>::V vzero();
template <> __device__ __forceinline__ float2 vzero<float>() { return make_float2(0.f, 0.f); }
template <> __device__ __forceinline__ double vzero<double>() { return 0.0; }

// ---- arithmetic -----------------------------------------------------------------
__device__ __forceinline__ float2 vmul(float2 a, float2 b) { return fmul2_rn(a, b); }
__device__ __forceinline__ float2 vfma(float2 a, float2 b, float2 c) { return fma2_rn(a, b, c); }
// immediate forms: the constant is broadcast to both halves
__device__ __forceinline__ float2 vmuli(float2 a, float c) { return fmul2_rn(a, make_float2(c, c)); }
__device__ __forceinline__ float2 vfmai(float2 a, float c, float2 b) { return fma2_rn(a, make_float2(c, c), b); }
__device__ __forceinline__ double vmul(double a, double b) { return a * b; }
__device__ __forceinline__ double vfma(double a, double b, double c) { return fma(a, b, c); }
__device__ __forceinline__ double vmuli(double a, double c) { return a * c; }
__device__ __forceinline__ double vfmai(double a, double c, double b) { return fma(a, c, b); }
__device__ __forceinline__ float vhsum(float2 a) { return a.x + a.y; }
__device__ __forceinline__ double vhsum(double a) { return a; }

// A chunk of MUL channels is "full" when no lane's channels fall past its end: MUL fills whole channel blocks and
// reaches every channel block its path group is given.  GMUL is the group's largest multiplicity (its work items
// cover ceil(GMUL / block) blocks); 0 stands for every channel block of the signature.  Accesses to a chunk that is
// not full are masked per channel.
template <typename T, int MUL, int GMUL = 0> __device__ constexpr bool vfull() {
  constexpr int B = VT<T>::LPE * VT<T>::CPT;
  return MUL % B == 0 && MUL >= (GMUL > 0 ? (GMUL + B - 1) / B : VT<T>::CB) * B;
}

// ---- strided channel loads: component i of CPT adjacent channels ---------------------
// p points at (channel ch0, component i); the next channel is N elements further.
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ float2 vload(const float* __restrict__ p, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full) return make_float2(__ldg(p), __ldg(p + N));
  return make_float2(ch0 < MUL ? __ldg(p) : 0.f, ch0 + 1 < MUL ? __ldg(p + N) : 0.f);
}
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ double vload(const double* __restrict__ p, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  if (full) return __ldg(p);
  return ch0 < MUL ? __ldg(p) : 0.0;
}
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ void vstore(float* __restrict__ p, float2 v, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full || ch0 < MUL) p[0] = v.x;
  if (full || ch0 + 1 < MUL) p[N] = v.y;
}
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ void vstore(double* __restrict__ p, double v, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  if (full || ch0 < MUL) p[0] = v;
}
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ void vatomic(float* p, float2 v, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full || ch0 < MUL) atomicAdd(p, v.x);
  if (full || ch0 + 1 < MUL) atomicAdd(p + N, v.y);
}
template <int N, int MUL, int GMUL = 0> __device__ __forceinline__ void vatomic(double* p, double v, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  if (full || ch0 < MUL) atomicAdd(p, v);
}

// ---- channel-contiguous (ir_mul) accesses: the CPT channels of one component are adjacent ----------
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ float2 vloadc(const float* __restrict__ p, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full && AL2) return __ldg(reinterpret_cast<const float2*>(p));
  return make_float2((full || ch0 < MUL) ? __ldg(p) : 0.f, (full || ch0 + 1 < MUL) ? __ldg(p + 1) : 0.f);
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ double vloadc(const double* __restrict__ p, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  return (full || ch0 < MUL) ? __ldg(p) : 0.0;
}
__device__ __forceinline__ void red_v2(float* p, float a, float b);
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ void vatomicc(float* p, float2 v, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full && AL2) {
    red_v2(p, v.x, v.y);
  } else {
    if (full || ch0 < MUL) atomicAdd(p, v.x);
    if (full || ch0 + 1 < MUL) atomicAdd(p + 1, v.y);
  }
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ void vatomicc(double* p, double v, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  if (full || ch0 < MUL) atomicAdd(p, v);
}

// whole row of a channel pair: 2*N adjacent floats starting at p (8-byte aligned) -> N vector
// reductions red.global.add.v2.f32 instead of 2*N scalar ones
__device__ __forceinline__ void red_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
template <int N, int MUL, int GMUL = 0, typename... Vs> __device__ __forceinline__ void vatomic_row(float* p, int ch0, Vs... vs) {
  static_assert(sizeof...(Vs) == N, "one value per component");
  constexpr bool full = vfull<float, MUL, GMUL>();
  const float2 v[N] = {vs...};
  if (full) {
    float flat[2 * N];
#pragma unroll
    for (int i = 0; i < N; ++i) { flat[i] = v[i].x; flat[N + i] = v[i].y; }
#pragma unroll
    for (int q = 0; q < N; ++q) red_v2(p + 2 * q, flat[2 * q], flat[2 * q + 1]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) {
      if (ch0 < MUL) atomicAdd(p + i, v[i].x);
      if (ch0 + 1 < MUL) atomicAdd(p + N + i, v[i].y);
    }
  }
}
template <int N, int MUL, int GMUL = 0, typename... Vs> __device__ __forceinline__ void vatomic_row(double* p, int ch0, Vs... vs) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  const double v[N] = {vs...};
#pragma unroll
  for (int i = 0; i < N; ++i)
    if (full || ch0 < MUL) atomicAdd(p + i, v[i]);
}

// ---- contiguous per-channel scalars (the radial weights): streamed, never re-read -------
__device__ __forceinline__ float2 ld_stream2(const float* p) {
  float2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ float ld_stream(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ double ld_stream(const double* p) {
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  return r;
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ float2 vloadw(const float* __restrict__ p, int ch0, bool valid) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  float2 r;
  if (full && AL2) {
    r = ld_stream2(p);
  } else {
    r.x = (full || ch0 < MUL) ? ld_stream(p) : 0.f;
    r.y = (full || ch0 + 1 < MUL) ? ld_stream(p + 1) : 0.f;
  }
  if (!valid) r = make_float2(0.f, 0.f);
  return r;
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ double vloadw(const double* __restrict__ p, int ch0, bool valid) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  double r = (full || ch0 < MUL) ? ld_stream(p) : 0.0;
  return valid ? r : 0.0;
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ void vstorew(float* __restrict__ p, float2 v, int ch0) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  if (full && AL2) {
    *reinterpret_cast<float2*>(p) = v;
  } else {
    if (full || ch0 < MUL) p[0] = v.x;
    if (full || ch0 + 1 < MUL) p[1] = v.y;
  }
}
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ void vstorew(double* __restrict__ p, double v, int ch0) {
  constexpr bool full = vfull<double, MUL, GMUL>();
  if (full || ch0 < MUL) p[0] = v;
}

#ifndef NQB_TC_HELPERS
// ---- shared-memory weight ring (forward v2): mbarrier + cp.async.bulk ---------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
#endif  // NQB_TC_HELPERS
// weights of the channel pair from the shared-memory ring
template <int MUL, bool AL2, int GMUL = 0> __device__ __forceinline__ float2 vloadws(const float* p, int ch0, bool valid) {
  constexpr bool full = vfull<float, MUL, GMUL>();
  float2 r = make_float2(0.f, 0.f);
  if (valid) {
    if (full && AL2) {
      r = *reinterpret_cast<const float2*>(p);
    } else {
      if (full || ch0 < MUL) r.x = p[0];
      if (full || ch0 + 1 < MUL) r.y = p[1];
    }
  }
  return r;
}

// ---- cross-lane -----------------------------------------------------------------------
// sum the partial accumulators of the EPW edge sub-groups (lanes l, l+LPE, l+2LPE, ...)
template <int LPE> __device__ __forceinline__ float2 vfold(float2 a) {
#pragma unroll
  for (int o = LPE; o < 32; o <<= 1) {
    a.x += __shfl_xor_sync(0xffffffffu, a.x, o);
    a.y += __shfl_xor_sync(0xffffffffu, a.y, o);
  }
  return a;
}
template <int LPE> __device__ __forceinline__ double vfold(double a) {
#pragma unroll
  for (int o = LPE; o < 32; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
}
// sum over the LPE lanes that share one edge
template <int LPE, typename T> __device__ __forceinline__ T lane_sum(T v) {
#pragma unroll
  for (int o = LPE / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// reduce-scatter of P per-lane partial sums over the LPE lanes that share one edge: halving
// butterfly (P-1 shuffles instead of P*log2(LPE)).  Afterwards v[0..C) (C = max(1, P/LPE)) hold
// the edge totals of components er_base(cl) .. er_base(cl)+C; er_leader(cl) picks one lane per
// component when LPE > P.
template <int O, int C, typename T> struct EdgeReduce {
  static __device__ __forceinline__ void run(T* v, int cl) {
    if constexpr (O >= 1) {
      if constexpr (C > 1) {
        constexpr int Hh = C / 2;
        const bool up = (cl & O) != 0;
#pragma unroll
        for (int j = 0; j < Hh; ++j) {
          const T mine = up ? v[j + Hh] : v[j];
          const T theirs = up ? v[j] : v[j + Hh];
          v[j] = mine + __shfl_xor_sync(0xffffffffu, theirs, O);
        }
        EdgeReduce<O / 2, Hh, T>::run(v, cl);
      } else {
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], O);
        EdgeReduce<O / 2, 1, T>::run(v, cl);
      }
    }
  }
};
template <int LPE, int P> __device__ __forceinline__ int er_base(int cl) {
  int base = 0, c = P;
#pragma unroll
  for (int o = LPE / 2; o >= 1; o >>= 1) {
    if (c > 1) { c >>= 1; if (cl & o) base += c; }
  }
  return base;
}
template <int LPE, int P> __device__ __forceinline__ bool er_leader(int cl) {
  int c = P; bool lead = true;
#pragma unroll
  for (int o = LPE / 2; o >= 1; o >>= 1) {
    if (c > 1) c >>= 1; else lead = lead && ((cl & o) == 0);
  }
  return lead;
}

}  // namespace
