// libnqb.so -- C-ABI runtime of the H100-native NequIP hot path (see include/nqb.h).
//
//  * plan registry: binds a TensorProductScatter signature to the specialised kernel
//    library generated for it (nequip_b200/codegen.py) via dlopen;
//  * destination-CSR helpers;
//  * edge geometry + real spherical harmonics + Bessel/cutoff radial embedding
//    kernels (forward and analytic backward).
//
// Reference semantics (paths under /root/reference):
//   with_edge_vectors_              nequip/nn/utils.py:68-118
//   SphericalHarmonicEdgeAttrs      nequip/nn/embedding/_edge.py:153-198  (e3nn SphericalHarmonics,
//                                   normalize=True, normalization="component")
//   EdgeLengthNormalizer            nequip/nn/embedding/_edge.py:65-80
//   BesselEdgeLengthEncoding        nequip/nn/embedding/_edge.py:136-150
//   PolynomialCutoff                nequip/nn/embedding/cutoffs.py:17-27
//   ApplyFactor                     nequip/nn/misc.py:46-48
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <string>
#include <vector>

#include "../../include/nqb.h"

// ------------------------------------------------------------------------------------------
// errors / accounting
// ------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};

static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
static int cuda_fail(cudaError_t e, const char* what) {
  return fail("%s: %s", what, cudaGetErrorString(e));
}
#define NQB_LAUNCH_CHECK(what)                                   \
  do {                                                           \
    g_launches.fetch_add(1, std::memory_order_relaxed);          \
    cudaError_t e__ = cudaGetLastError();                        \
    if (e__ != cudaSuccess) return cuda_fail(e__, what);         \
  } while (0)

extern "C" int nqb_abi_version(void) { return 2; }
// internal helpers shared with the other translation units of libnqb.so (not part of nqb.h)
extern "C" int nqb_set_error(const char* msg) { return fail("%s", msg); }
extern "C" void nqb_count_launch(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" const char* nqb_last_error(void) { return g_err; }
extern "C" int64_t nqb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

// ------------------------------------------------------------------------------------------
// plan
// ------------------------------------------------------------------------------------------
typedef const char* (*spec_signature_fn)();
typedef int (*spec_version_fn)();
typedef int (*spec_dims_fn)(int*, int*, int*, int*);
typedef int (*spec_fwd_fn)(int, const void*, const void*, const void*, const int64_t*, const int64_t*,
                           const int64_t*, int64_t, int64_t, void*, cudaStream_t);
typedef int (*spec_gy_slices_fn)(int);
typedef int (*spec_bwd_fn)(int, const void*, const void*, const void*, const int64_t*, const int64_t*,
                           const int64_t*, const void*, int64_t, int64_t, void*, void*, void*, int, cudaStream_t);

typedef int (*spec_fused_info_fn)(int*, int*, int*);
typedef int (*spec_fused_fwd_fn)(const float*, const float*, const float*, int64_t, int, const float*, const int64_t*,
                                 const int64_t*, int64_t, int64_t, float*, float*, const int32_t*, int, cudaStream_t);

struct nqb_plan {
  std::string signature;
  void* lib;
  spec_fwd_fn fwd;
  spec_bwd_fn bwd;
  spec_gy_slices_fn gy_slices = nullptr;
  spec_fused_fwd_fn fused_fwd = nullptr;  // null: the signature has no fused radial-MLP + TP kernel
  int fused_nslice = 0;
  int d_in, s_dim, w_numel, d_out;
  // {first column, columns} of the irreps_in1 chunks no instruction reads: the kernels never touch them, so the
  // deterministic backward zero-fills them in its per-edge grad_x buffer
  std::vector<std::pair<int, int>> unread_in1;
};

static void append_irreps(std::string& s, const nqb_irrep* ir, int n) {
  char buf[64];
  for (int i = 0; i < n; ++i) {
    snprintf(buf, sizeof(buf), "%s%dx%d%c", i ? "+" : "", ir[i].mul, ir[i].l, ir[i].p == 1 ? 'e' : 'o');
    s += buf;
  }
}

extern "C" int nqb_plan_create(const nqb_irrep* in1, int n_in1, const nqb_irrep* in2, int n_in2,
                               const nqb_irrep* out, int n_out, const nqb_instruction* ins, int n_ins,
                               const char* spec_lib_path, nqb_plan** plan) {
  if (!in1 || !in2 || !out || !ins || !plan) return fail("nqb_plan_create: null argument");
  if (n_ins <= 0) return fail("nqb_plan_create: empty instruction list");
  if (!spec_lib_path) return fail("nqb_plan_create: no specialised kernel library given");
  for (int i = 0; i < n_ins; ++i) {
    const nqb_instruction& q = ins[i];
    if (q.i_in1 < 0 || q.i_in1 >= n_in1 || q.i_in2 < 0 || q.i_in2 >= n_in2 || q.i_out < 0 || q.i_out >= n_out)
      return fail("nqb_plan_create: instruction %d indexes outside the irreps", i);
    const nqb_irrep &a = in1[q.i_in1], &b = in2[q.i_in2], &c = out[q.i_out];
    if (b.mul != 1) return fail("nqb_plan_create: edge-attribute multiplicity %d != 1 unsupported", b.mul);
    if (a.mul != c.mul) return fail("nqb_plan_create: 'uvu' needs mul_out == mul_in1 (instruction %d)", i);
    if (c.p != a.p * b.p || c.l < abs(a.l - b.l) || c.l > a.l + b.l)
      return fail("nqb_plan_create: instruction %d violates the selection rules", i);
  }
  std::string sig = "in1=";
  append_irreps(sig, in1, n_in1);
  sig += "|in2=";
  append_irreps(sig, in2, n_in2);
  sig += "|out=";
  append_irreps(sig, out, n_out);
  sig += "|ins=";
  char buf[64];
  for (int i = 0; i < n_ins; ++i) {
    snprintf(buf, sizeof(buf), "%s%d,%d,%d", i ? ";" : "", ins[i].i_in1, ins[i].i_in2, ins[i].i_out);
    sig += buf;
  }
  void* lib = dlopen(spec_lib_path, RTLD_NOW | RTLD_LOCAL);
  if (!lib) return fail("nqb_plan_create: dlopen(%s) failed: %s", spec_lib_path, dlerror());
  spec_signature_fn fsig = (spec_signature_fn)dlsym(lib, "nqb_spec_signature");
  spec_dims_fn fdims = (spec_dims_fn)dlsym(lib, "nqb_spec_dims");
  spec_fwd_fn ffwd = (spec_fwd_fn)dlsym(lib, "nqb_spec_fwd");
  spec_bwd_fn fbwd = (spec_bwd_fn)dlsym(lib, "nqb_spec_bwd");
  if (!fsig || !fdims || !ffwd || !fbwd) {
    dlclose(lib);
    return fail("nqb_plan_create: %s does not export the nqb_spec_* entry points", spec_lib_path);
  }
  if (sig != fsig()) {
    std::string have = fsig();
    dlclose(lib);
    return fail("nqb_plan_create: kernel library was generated for a different signature\n  want %s\n  have %s",
                sig.c_str(), have.c_str());
  }
  nqb_plan* p = new nqb_plan();
  p->signature = sig;
  p->lib = lib;
  p->fwd = ffwd;
  p->bwd = fbwd;
  fdims(&p->d_in, &p->s_dim, &p->w_numel, &p->d_out);
  for (int i = 0, off = 0; i < n_in1; off += in1[i].mul * (2 * in1[i].l + 1), ++i) {
    bool read = false;
    for (int k = 0; k < n_ins; ++k) read |= ins[k].i_in1 == i;
    if (!read) p->unread_in1.push_back({off, in1[i].mul * (2 * in1[i].l + 1)});
  }
  p->gy_slices = (spec_gy_slices_fn)dlsym(lib, "nqb_spec_gy_slices");
  spec_fused_info_fn finfo = (spec_fused_info_fn)dlsym(lib, "nqb_spec_fused_info");
  spec_fused_fwd_fn ffused = (spec_fused_fwd_fn)dlsym(lib, "nqb_spec_fused_fwd");
  int nxs = 0, xrow = 0;
  if (finfo && ffused && finfo(&p->fused_nslice, &nxs, &xrow) == 0 && p->fused_nslice > 0) p->fused_fwd = ffused;
  *plan = p;
  return 0;
}

extern "C" void nqb_plan_destroy(nqb_plan* plan) {
  if (!plan) return;
  // the kernel library stays mapped: other plans may share it and unloading CUDA modules
  // from a destructor thread is not worth the risk
  delete plan;
}

extern "C" int nqb_plan_dims(const nqb_plan* plan, int* d_in, int* s_dim, int* weight_numel, int* d_out) {
  if (!plan) return fail("nqb_plan_dims: null plan");
  if (d_in) *d_in = plan->d_in;
  if (s_dim) *s_dim = plan->s_dim;
  if (weight_numel) *weight_numel = plan->w_numel;
  if (d_out) *d_out = plan->d_out;
  return 0;
}

extern "C" int nqb_plan_signature(const nqb_plan* plan, char* buf, int buflen) {
  if (!plan) return -1;
  int need = (int)plan->signature.size() + 1;
  if (buf && buflen > 0) {
    strncpy(buf, plan->signature.c_str(), buflen - 1);
    buf[buflen - 1] = 0;
  }
  return need;
}

extern "C" int nqb_tp_scatter_fwd(const nqb_plan* plan, int dtype, const void* x, const void* y, const void* w,
                                  const int64_t* row_ptr, const int64_t* perm, const int64_t* src, int64_t N,
                                  int64_t E, void* out, nqb_stream_t st) {
  if (!plan) return fail("nqb_tp_scatter_fwd: null plan");
  if (dtype != NQB_F32 && dtype != NQB_F64) return fail("nqb_tp_scatter_fwd: bad dtype %d", dtype);
  if (N < 0 || E < 0) return fail("nqb_tp_scatter_fwd: negative size");
  if (N == 0) return 0;
  if (!row_ptr || !out || (E > 0 && (!x || !y || !w || !src)))
    return fail("nqb_tp_scatter_fwd: null pointer argument");
  int rc = plan->fwd(dtype, x, y, w, row_ptr, perm, src, N, E, out, (cudaStream_t)st);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (rc) return cuda_fail((cudaError_t)rc, "nqb_tp_scatter_fwd launch");
  return 0;
}

extern "C" int nqb_tp_scatter_bwd(const nqb_plan* plan, int dtype, const void* x, const void* y, const void* w,
                                  const int64_t* row_ptr, const int64_t* perm, const int64_t* src,
                                  const void* grad_out, int64_t N, int64_t E, void* grad_x, void* grad_y,
                                  void* grad_w, int deterministic, nqb_stream_t st) {
  if (!plan) return fail("nqb_tp_scatter_bwd: null plan");
  if (dtype != NQB_F32 && dtype != NQB_F64) return fail("nqb_tp_scatter_bwd: bad dtype %d", dtype);
  if (N < 0 || E < 0) return fail("nqb_tp_scatter_bwd: negative size");
  if (N == 0 || E == 0) return 0;
  if (!row_ptr || !x || !y || !w || !src || !grad_out || !grad_y || !grad_w)
    return fail("nqb_tp_scatter_bwd: null pointer argument");
  if (deterministic && !plan->gy_slices) return fail("nqb_tp_scatter_bwd: kernel library has no deterministic mode");
  if (deterministic && grad_x) {
    // the per-edge grad_x buffer is fully written: zeros in the columns of chunks no instruction reads
    const size_t esz = dtype == NQB_F32 ? sizeof(float) : sizeof(double);
    for (const auto& c : plan->unread_in1) {
      cudaError_t e = cudaMemset2DAsync((char*)grad_x + c.first * esz, plan->d_in * esz, 0, c.second * esz, (size_t)E,
                                        (cudaStream_t)st);
      if (e != cudaSuccess) return cuda_fail(e, "nqb_tp_scatter_bwd: zero fill of unread grad_x columns");
    }
  }
  int rc = plan->bwd(dtype, x, y, w, row_ptr, perm, src, grad_out, N, E, grad_x, grad_y, grad_w, deterministic ? 1 : 0,
                     (cudaStream_t)st);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (rc) return cuda_fail((cudaError_t)rc, "nqb_tp_scatter_bwd launch");
  return 0;
}

extern "C" int nqb_tp_scatter_gy_slices(const nqb_plan* plan, int dtype) {
  if (!plan || !plan->gy_slices) return 0;
  return plan->gy_slices(dtype);
}

// out[n, :] = sum over the rows perm[q], q in [seg_ptr[n], seg_ptr[n+1]), of rows[., :]   (fixed order: deterministic)
template <typename T>
__global__ void k_segment_sum(const T* __restrict__ rows, int D, const int64_t* __restrict__ perm,
                              const int64_t* __restrict__ seg_ptr, int64_t N, T* __restrict__ out) {
  const int64_t n = blockIdx.x;
  if (n >= N) return;
  const int64_t beg = seg_ptr[n], end = seg_ptr[n + 1];
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    T acc = (T)0;
    for (int64_t q = beg; q < end; ++q) acc += rows[perm[q] * (int64_t)D + c];
    out[n * (int64_t)D + c] = acc;
  }
}

extern "C" int nqb_segment_sum(int dtype, const void* rows, int D, const int64_t* perm, const int64_t* seg_ptr, int64_t N,
                               void* out, nqb_stream_t st) {
  if (dtype != NQB_F32 && dtype != NQB_F64) return fail("nqb_segment_sum: bad dtype %d", dtype);
  if (N < 0 || D <= 0) return fail("nqb_segment_sum: bad size");
  if (N == 0) return 0;
  if (!rows || !perm || !seg_ptr || !out) return fail("nqb_segment_sum: null pointer");
  const int threads = D >= 256 ? 256 : (D >= 128 ? 128 : 64);
  if (dtype == NQB_F32)
    k_segment_sum<float><<<(unsigned)N, threads, 0, (cudaStream_t)st>>>((const float*)rows, D, perm, seg_ptr, N, (float*)out);
  else
    k_segment_sum<double><<<(unsigned)N, threads, 0, (cudaStream_t)st>>>((const double*)rows, D, perm, seg_ptr, N, (double*)out);
  NQB_LAUNCH_CHECK("nqb_segment_sum");
  return 0;
}

extern "C" int nqb_tp_fused_slices(const nqb_plan* plan) {
  if (!plan || !plan->fused_fwd) return 0;
  return plan->fused_nslice;
}

extern "C" int nqb_tp_fused_fwd(const nqb_plan* plan, const float* x, const float* y, const float* h, int64_t ldh, int K,
                                const float* w2_prepared, const int64_t* row_ptr, const int64_t* src, int64_t N, int64_t E,
                                float* out, float* w_out, const int32_t* slice_cta0, int nctas, nqb_stream_t st) {
  if (!plan) return fail("nqb_tp_fused_fwd: null plan");
  if (!plan->fused_fwd) return fail("nqb_tp_fused_fwd: this signature has no fused kernel (nqb_tp_fused_slices() == 0)");
  if (N < 0 || E < 0) return fail("nqb_tp_fused_fwd: negative size");
  if (N == 0) return 0;
  if (!row_ptr || !out || !w2_prepared || !slice_cta0 || (E > 0 && (!x || !y || !h || !src)))
    return fail("nqb_tp_fused_fwd: null pointer argument");
  if (K <= 0 || K > 128 || (K % 8) || (ldh % 4) || ldh < K) return fail("nqb_tp_fused_fwd: needs 0 < K <= 128, K %% 8 == 0, ldh %% 4 == 0");
  // h rows are staged with 16-byte cp.async
  if (E > 0 && ((uintptr_t)h & 15)) return fail("nqb_tp_fused_fwd: h must be 16-byte aligned");
  if (nctas <= 0) return fail("nqb_tp_fused_fwd: empty grid");
  int rc = plan->fused_fwd(x, y, h, ldh, K, w2_prepared, row_ptr, src, N, E, out, w_out, slice_cta0, nctas, (cudaStream_t)st);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (rc) return cuda_fail((cudaError_t)rc, "nqb_tp_fused_fwd launch");
  return 0;
}

// ------------------------------------------------------------------------------------------
// CSR helpers
// ------------------------------------------------------------------------------------------
__global__ void k_check_sorted(const int64_t* __restrict__ keys, int64_t E, int32_t* flag) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  bool bad = false;
  for (; i + 1 < E; i += stride) bad |= keys[i] > keys[i + 1];
  if (bad) *flag = 0;
}
__global__ void k_set_flag(int32_t* flag, int32_t v) { *flag = v; }

extern "C" int nqb_csr_check_sorted(const int64_t* keys, int64_t E, int32_t* flag_dev, nqb_stream_t st) {
  if (!flag_dev) return fail("nqb_csr_check_sorted: null flag");
  k_set_flag<<<1, 1, 0, (cudaStream_t)st>>>(flag_dev, 1);
  NQB_LAUNCH_CHECK("nqb_csr_check_sorted");
  if (E > 1) {
    if (!keys) return fail("nqb_csr_check_sorted: null keys");
    int blocks = (int)((E + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    k_check_sorted<<<blocks, 256, 0, (cudaStream_t)st>>>(keys, E, flag_dev);
    NQB_LAUNCH_CHECK("nqb_csr_check_sorted");
  }
  return 0;
}

// row_ptr[n] = first slot whose key >= n (lower bound), n = 0..N
__global__ void k_csr_from_sorted(const int64_t* __restrict__ keys, int64_t E, int64_t N, int64_t* __restrict__ row_ptr) {
  int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n > N) return;
  int64_t lo = 0, hi = E;
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < n) lo = mid + 1; else hi = mid;
  }
  row_ptr[n] = lo;
}

extern "C" int nqb_csr_from_sorted(const int64_t* sorted_keys, int64_t E, int64_t N, int64_t* row_ptr,
                                   nqb_stream_t st) {
  if (N < 0 || E < 0) return fail("nqb_csr_from_sorted: negative size");
  if (!row_ptr) return fail("nqb_csr_from_sorted: null row_ptr");
  if (E > 0 && !sorted_keys) return fail("nqb_csr_from_sorted: null keys");
  int64_t blocks = (N + 1 + 255) / 256;
  k_csr_from_sorted<<<(unsigned)blocks, 256, 0, (cudaStream_t)st>>>(sorted_keys, E, N, row_ptr);
  NQB_LAUNCH_CHECK("nqb_csr_from_sorted");
  return 0;
}

// ------------------------------------------------------------------------------------------
// spherical harmonics (lmax <= 4), y is the polar axis, m = -l..l, component normalisation
// ------------------------------------------------------------------------------------------
#define NQB_MAX_S 25

// degree 4: the block Y_4 = c * C^{4,1,3} : (Y_1, Y_3) of the w3j recursion (SURVEY App. A.3, oracle/sh.py
// sh_recurrence), multiplied out into quartic polynomials of the unit vector.  Coefficients:
//   a4 = 3 sqrt(35) / 2, b4 = 3 sqrt(70) / 4, c4 = 3 sqrt(5) / 2, d4 = 3 sqrt(10) / 4, e4 = 3 sqrt(5) / 4,
//   f4 = 3 sqrt(35) / 8
#define NQB_SH4_CONSTS                                                                                  \
  const double a4 = 8.874119674649425, b4 = 6.274950199005566, c4 = 3.3541019662496847;               \
  const double d4 = 2.3717082451262845, e4 = 1.6770509831248424, f4 = 2.218529918662356;

template <int LMAX>
__device__ __forceinline__ void sh_eval(double x, double y, double z, double* Y) {
  Y[0] = 1.0;
  if (LMAX >= 1) {
    const double s3 = 1.7320508075688772;
    Y[1] = s3 * x; Y[2] = s3 * y; Y[3] = s3 * z;
  }
  if (LMAX >= 2) {
    const double s15 = 3.872983346207417, s5 = 2.23606797749979;
    const double x2 = x * x, y2 = y * y, z2 = z * z;
    Y[4] = s15 * x * z;
    Y[5] = s15 * x * y;
    Y[6] = s5 * (y2 - 0.5 * (x2 + z2));
    Y[7] = s15 * y * z;
    Y[8] = 0.5 * s15 * (z2 - x2);
  }
  if (LMAX >= 3) {
    const double a3 = 2.091650066335189;   // sqrt(35/8)
    const double b3 = 1.6201851746019651;  // sqrt(21/8)
    const double c3 = 1.3228756555322954;  // sqrt(7)/2
    const double s105 = 10.246950765959598;
    const double x2 = x * x, y2 = y * y, z2 = z * z;
    Y[9] = a3 * x * (3.0 * z2 - x2);
    Y[10] = s105 * x * y * z;
    Y[11] = b3 * x * (4.0 * y2 - x2 - z2);
    Y[12] = c3 * y * (2.0 * y2 - 3.0 * x2 - 3.0 * z2);
    Y[13] = b3 * z * (4.0 * y2 - x2 - z2);
    Y[14] = 0.5 * s105 * y * (z2 - x2);
    Y[15] = a3 * z * (z2 - 3.0 * x2);
  }
  if (LMAX >= 4) {
    NQB_SH4_CONSTS
    const double x2 = x * x, y2 = y * y, z2 = z * z;
    Y[16] = a4 * x * z * (z2 - x2);
    Y[17] = b4 * x * y * (3.0 * z2 - x2);
    Y[18] = c4 * x * z * (6.0 * y2 - x2 - z2);
    Y[19] = d4 * x * y * (4.0 * y2 - 3.0 * x2 - 3.0 * z2);
    Y[20] = 0.375 * (3.0 * x2 * x2 - 24.0 * x2 * y2 + 6.0 * x2 * z2 + 8.0 * y2 * y2 - 24.0 * y2 * z2 + 3.0 * z2 * z2);
    Y[21] = d4 * y * z * (4.0 * y2 - 3.0 * x2 - 3.0 * z2);
    Y[22] = e4 * (x2 - z2) * (x2 - 6.0 * y2 + z2);
    Y[23] = b4 * y * z * (z2 - 3.0 * x2);
    Y[24] = f4 * (x2 * x2 - 6.0 * x2 * z2 + z2 * z2);
  }
}

// gradient of the homogeneous polynomials P_lm at the unit vector u, contracted with g:
//   G = sum_m g_m grad P_lm(u),   D = sum_m g_m l P_lm(u)
// then dL/dr = (G - D u) / |r|   (Y(r) = P_l(r)/|r|^l).
template <int LMAX>
__device__ __forceinline__ void sh_vjp(double x, double y, double z, const double* g, double& Gx, double& Gy,
                                       double& Gz, double& D) {
  Gx = Gy = Gz = D = 0.0;
  double Y[NQB_MAX_S];
  sh_eval<LMAX>(x, y, z, Y);
  if (LMAX >= 1) {
    const double s3 = 1.7320508075688772;
    Gx += s3 * g[1]; Gy += s3 * g[2]; Gz += s3 * g[3];
    D += g[1] * Y[1] + g[2] * Y[2] + g[3] * Y[3];
  }
  if (LMAX >= 2) {
    const double s15 = 3.872983346207417, s5 = 2.23606797749979;
    Gx += g[4] * s15 * z + g[5] * s15 * y - g[6] * s5 * x - g[8] * s15 * x;
    Gy += g[5] * s15 * x + g[6] * 2.0 * s5 * y + g[7] * s15 * z;
    Gz += g[4] * s15 * x - g[6] * s5 * z + g[7] * s15 * y + g[8] * s15 * z;
    D += 2.0 * (g[4] * Y[4] + g[5] * Y[5] + g[6] * Y[6] + g[7] * Y[7] + g[8] * Y[8]);
  }
  if (LMAX >= 3) {
    const double a3 = 2.091650066335189, b3 = 1.6201851746019651, c3 = 1.3228756555322954;
    const double s105 = 10.246950765959598;
    const double x2 = x * x, y2 = y * y, z2 = z * z;
    Gx += g[9] * a3 * (3.0 * z2 - 3.0 * x2) + g[10] * s105 * y * z + g[11] * b3 * (4.0 * y2 - 3.0 * x2 - z2)
        + g[12] * c3 * (-6.0 * x * y) + g[13] * b3 * (-2.0 * x * z) + g[14] * 0.5 * s105 * (-2.0 * x * y)
        + g[15] * a3 * (-6.0 * x * z);
    Gy += g[10] * s105 * x * z + g[11] * b3 * 8.0 * x * y + g[12] * c3 * (6.0 * y2 - 3.0 * x2 - 3.0 * z2)
        + g[13] * b3 * 8.0 * y * z + g[14] * 0.5 * s105 * (z2 - x2);
    Gz += g[9] * a3 * 6.0 * x * z + g[10] * s105 * x * y + g[11] * b3 * (-2.0 * x * z) + g[12] * c3 * (-6.0 * y * z)
        + g[13] * b3 * (4.0 * y2 - x2 - 3.0 * z2) + g[14] * 0.5 * s105 * 2.0 * y * z + g[15] * a3 * (3.0 * z2 - 3.0 * x2);
    D += 3.0 * (g[9] * Y[9] + g[10] * Y[10] + g[11] * Y[11] + g[12] * Y[12] + g[13] * Y[13] + g[14] * Y[14] + g[15] * Y[15]);
  }
  if (LMAX >= 4) {
    NQB_SH4_CONSTS
    const double x2 = x * x, y2 = y * y, z2 = z * z, xyz = x * y * z;
    Gx += g[16] * a4 * z * (z2 - 3.0 * x2) + g[17] * 3.0 * b4 * y * (z2 - x2) + g[18] * c4 * z * (6.0 * y2 - 3.0 * x2 - z2)
        + g[19] * d4 * y * (4.0 * y2 - 9.0 * x2 - 3.0 * z2) + g[20] * 4.5 * x * (x2 - 4.0 * y2 + z2)
        - g[21] * 6.0 * d4 * xyz + g[22] * 4.0 * e4 * x * (x2 - 3.0 * y2) - g[23] * 6.0 * b4 * xyz
        + g[24] * 4.0 * f4 * x * (x2 - 3.0 * z2);
    Gy += g[17] * b4 * x * (3.0 * z2 - x2) + g[18] * 12.0 * c4 * xyz + g[19] * 3.0 * d4 * x * (4.0 * y2 - x2 - z2)
        + g[20] * 6.0 * y * (2.0 * y2 - 3.0 * x2 - 3.0 * z2) + g[21] * 3.0 * d4 * z * (4.0 * y2 - x2 - z2)
        - g[22] * 12.0 * e4 * y * (x2 - z2) + g[23] * b4 * z * (z2 - 3.0 * x2);
    Gz += g[16] * a4 * x * (3.0 * z2 - x2) + g[17] * 6.0 * b4 * xyz + g[18] * c4 * x * (6.0 * y2 - x2 - 3.0 * z2)
        - g[19] * 6.0 * d4 * xyz + g[20] * 4.5 * z * (x2 - 4.0 * y2 + z2) + g[21] * d4 * y * (4.0 * y2 - 3.0 * x2 - 9.0 * z2)
        + g[22] * 4.0 * e4 * z * (3.0 * y2 - z2) + g[23] * 3.0 * b4 * y * (z2 - x2) + g[24] * 4.0 * f4 * z * (z2 - 3.0 * x2);
    D += 4.0 * (g[16] * Y[16] + g[17] * Y[17] + g[18] * Y[18] + g[19] * Y[19] + g[20] * Y[20] + g[21] * Y[21]
                + g[22] * Y[22] + g[23] * Y[23] + g[24] * Y[24]);
  }
}

template <typename T> __device__ __forceinline__ double to_d(T v) { return (double)v; }

template <int LMAX, typename TO>
__global__ void k_sh_fwd(const double* __restrict__ vec, int64_t E, TO* __restrict__ out) {
  constexpr int S = (LMAX + 1) * (LMAX + 1);
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double x = vec[3 * e], y = vec[3 * e + 1], z = vec[3 * e + 2];
  double r = sqrt(x * x + y * y + z * z);
  double inv = 1.0 / fmax(r, 1e-12);  // torch.nn.functional.normalize eps
  x *= inv; y *= inv; z *= inv;
  double Y[NQB_MAX_S];
  sh_eval<LMAX>(x, y, z, Y);
#pragma unroll
  for (int q = 0; q < S; ++q) out[e * S + q] = (TO)Y[q];
}

template <int LMAX, typename TO>
__global__ void k_sh_bwd(const double* __restrict__ vec, int64_t E, const TO* __restrict__ gy, double* __restrict__ gvec) {
  constexpr int S = (LMAX + 1) * (LMAX + 1);
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  double x = vec[3 * e], y = vec[3 * e + 1], z = vec[3 * e + 2];
  double r = sqrt(x * x + y * y + z * z);
  double inv = 1.0 / fmax(r, 1e-12);
  x *= inv; y *= inv; z *= inv;
  double g[NQB_MAX_S];
#pragma unroll
  for (int q = 0; q < S; ++q) g[q] = (double)gy[e * S + q];
  double Gx, Gy, Gz, D;
  sh_vjp<LMAX>(x, y, z, g, Gx, Gy, Gz, D);
  gvec[3 * e] = (Gx - D * x) * inv;
  gvec[3 * e + 1] = (Gy - D * y) * inv;
  gvec[3 * e + 2] = (Gz - D * z) * inv;
}

extern "C" int nqb_sh_fwd(int lmax, const double* vec, int64_t E, int out_dtype, void* y, nqb_stream_t st) {
  if (lmax < 0 || lmax > 4) return fail("nqb_sh_fwd: lmax=%d unsupported (0..4)", lmax);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_sh_fwd: bad dtype");
  if (E < 0) return fail("nqb_sh_fwd: negative size");
  if (E == 0) return 0;
  if (!vec || !y) return fail("nqb_sh_fwd: null pointer");
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
  if (out_dtype == NQB_F32) {
    switch (lmax) {
      case 0: k_sh_fwd<0, float><<<blocks, 128, 0, s>>>(vec, E, (float*)y); break;
      case 1: k_sh_fwd<1, float><<<blocks, 128, 0, s>>>(vec, E, (float*)y); break;
      case 2: k_sh_fwd<2, float><<<blocks, 128, 0, s>>>(vec, E, (float*)y); break;
      case 3: k_sh_fwd<3, float><<<blocks, 128, 0, s>>>(vec, E, (float*)y); break;
      default: k_sh_fwd<4, float><<<blocks, 128, 0, s>>>(vec, E, (float*)y); break;
    }
  } else {
    switch (lmax) {
      case 0: k_sh_fwd<0, double><<<blocks, 128, 0, s>>>(vec, E, (double*)y); break;
      case 1: k_sh_fwd<1, double><<<blocks, 128, 0, s>>>(vec, E, (double*)y); break;
      case 2: k_sh_fwd<2, double><<<blocks, 128, 0, s>>>(vec, E, (double*)y); break;
      case 3: k_sh_fwd<3, double><<<blocks, 128, 0, s>>>(vec, E, (double*)y); break;
      default: k_sh_fwd<4, double><<<blocks, 128, 0, s>>>(vec, E, (double*)y); break;
    }
  }
  NQB_LAUNCH_CHECK("nqb_sh_fwd");
  return 0;
}

extern "C" int nqb_sh_bwd(int lmax, const double* vec, int64_t E, int out_dtype, const void* grad_y,
                          double* grad_vec, nqb_stream_t st) {
  if (lmax < 0 || lmax > 4) return fail("nqb_sh_bwd: lmax=%d unsupported (0..4)", lmax);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_sh_bwd: bad dtype");
  if (E < 0) return fail("nqb_sh_bwd: negative size");
  if (E == 0) return 0;
  if (!vec || !grad_y || !grad_vec) return fail("nqb_sh_bwd: null pointer");
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
  if (out_dtype == NQB_F32) {
    switch (lmax) {
      case 0: k_sh_bwd<0, float><<<blocks, 128, 0, s>>>(vec, E, (const float*)grad_y, grad_vec); break;
      case 1: k_sh_bwd<1, float><<<blocks, 128, 0, s>>>(vec, E, (const float*)grad_y, grad_vec); break;
      case 2: k_sh_bwd<2, float><<<blocks, 128, 0, s>>>(vec, E, (const float*)grad_y, grad_vec); break;
      case 3: k_sh_bwd<3, float><<<blocks, 128, 0, s>>>(vec, E, (const float*)grad_y, grad_vec); break;
      default: k_sh_bwd<4, float><<<blocks, 128, 0, s>>>(vec, E, (const float*)grad_y, grad_vec); break;
    }
  } else {
    switch (lmax) {
      case 0: k_sh_bwd<0, double><<<blocks, 128, 0, s>>>(vec, E, (const double*)grad_y, grad_vec); break;
      case 1: k_sh_bwd<1, double><<<blocks, 128, 0, s>>>(vec, E, (const double*)grad_y, grad_vec); break;
      case 2: k_sh_bwd<2, double><<<blocks, 128, 0, s>>>(vec, E, (const double*)grad_y, grad_vec); break;
      case 3: k_sh_bwd<3, double><<<blocks, 128, 0, s>>>(vec, E, (const double*)grad_y, grad_vec); break;
      default: k_sh_bwd<4, double><<<blocks, 128, 0, s>>>(vec, E, (const double*)grad_y, grad_vec); break;
    }
  }
  NQB_LAUNCH_CHECK("nqb_sh_bwd");
  return 0;
}

// ------------------------------------------------------------------------------------------
// fused edge geometry + SH + radial embedding
// ------------------------------------------------------------------------------------------
#define NQB_MAX_BESSEL 32

struct EmbedParams {
  int num_bessel;
  double r_max, poly_p, prefactor;
};

__device__ __forceinline__ double poly_cutoff(double x, double p) {
  if (!(x < 1.0)) return 0.0;
  double xp = pow(x, p);
  double out = 1.0;
  out = out - ((p + 1.0) * (p + 2.0) / 2.0) * xp;
  out = out + (p * (p + 2.0)) * (xp * x);
  out = out - (p * (p + 1.0) / 2.0) * (xp * x * x);
  return out;
}
__device__ __forceinline__ double poly_cutoff_deriv(double x, double p) {
  if (!(x < 1.0)) return 0.0;
  double xpm1 = pow(x, p - 1.0);
  return 0.5 * p * (p + 1.0) * (p + 2.0) * (-xpm1 + 2.0 * xpm1 * x - xpm1 * x * x);
}

// Per-edge-type cutoffs (nequip/nn/embedding/_edge.py:65-80 with per_edge_type_cutoff): the normalised length is
// x = r * recip[T * type(tidx[0][e]) + type(tidx[1][e])] instead of r / r_max.  tidx names the edge's atoms for the
// type lookup; it is the geometry's eidx except in the edge-vector branch, whose eidx indexes made-up positions.
struct EdgeTypes {
  const int64_t* types;  // [N'] atom types of the atoms tidx names
  const int64_t* tidx;   // [2, E]
  const double* recip;   // [T * T] 1 / rc[source, target]
  int T;
};

// kTyped = false: x = r / r_max, and the trailing EdgeTypes parameter is not read (appended, so the code of the
// untyped variants is unchanged)
__device__ __forceinline__ double edge_recip(const EdgeTypes& et, int64_t E, int64_t e) {
  return et.recip[et.T * et.types[et.tidx[e]] + et.types[et.tidx[E + e]]];
}

// kFramed (nqb_edge_embed_fwd_frames): a batch of frames, cell [F, 3, 3]; edge e takes the cell of its centre's
// frame, cell + 9 * frame[eidx[0][e]], in the same shift expression.  Unframed variants do not read the trailing frame
// parameter (appended, so their code is unchanged).  The backward reads the stored edge vectors only and needs no
// framed variant.
template <int LMAX, typename TO, bool kTyped = false, bool kFramed = false>
__global__ void k_edge_embed_fwd(EmbedParams prm, const double* __restrict__ pos, const int64_t* __restrict__ eidx,
                                 const double* __restrict__ shift, const double* __restrict__ cell, int64_t E,
                                 double* __restrict__ vec, TO* __restrict__ yout, TO* __restrict__ emb, EdgeTypes et,
                                 const int64_t* __restrict__ frame) {
  constexpr int S = (LMAX + 1) * (LMAX + 1);
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int64_t i0 = eidx[e], i1 = eidx[E + e];
  double vx = pos[3 * i1] - pos[3 * i0];
  double vy = pos[3 * i1 + 1] - pos[3 * i0 + 1];
  double vz = pos[3 * i1 + 2] - pos[3 * i0 + 2];
  if (shift != nullptr && cell != nullptr) {
    const double s0 = shift[3 * e], s1 = shift[3 * e + 1], s2 = shift[3 * e + 2];
    const double* c = kFramed ? cell + 9 * frame[i0] : cell;
    vx += s0 * c[0] + s1 * c[3] + s2 * c[6];
    vy += s0 * c[1] + s1 * c[4] + s2 * c[7];
    vz += s0 * c[2] + s1 * c[5] + s2 * c[8];
  }
  vec[3 * e] = vx; vec[3 * e + 1] = vy; vec[3 * e + 2] = vz;
  const double r = sqrt(vx * vx + vy * vy + vz * vz);
  const double inv = 1.0 / fmax(r, 1e-12);
  double Y[NQB_MAX_S];
  sh_eval<LMAX>(vx * inv, vy * inv, vz * inv, Y);
#pragma unroll
  for (int q = 0; q < S; ++q) yout[e * S + q] = (TO)Y[q];
  // radial embedding: (TO)bessel * (TO)cutoff * (TO)prefactor, as the reference rounds it
  const double x = kTyped ? r * edge_recip(et, E, e) : r / prm.r_max;
  const TO fc = (TO)poly_cutoff(x, prm.poly_p);
  const TO pre = (TO)prm.prefactor;
  for (int n = 1; n <= prm.num_bessel; ++n) {
    const double t = (double)n * x;
    const double sinc = (t == 0.0) ? 1.0 : sinpi(t) / (M_PI * t);
    const TO b = (TO)(sinc * (double)n);
    emb[e * prm.num_bessel + (n - 1)] = pre * (b * fc);
  }
}

template <int LMAX, typename TO, bool kTyped = false>
__global__ void k_edge_embed_bwd(EmbedParams prm, const double* __restrict__ vec, const int64_t* __restrict__ eidx,
                                 int64_t E, const TO* __restrict__ gy, const TO* __restrict__ gemb,
                                 double* __restrict__ gpos, double* __restrict__ gvec, EdgeTypes et) {
  constexpr int S = (LMAX + 1) * (LMAX + 1);
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const double vx = vec[3 * e], vy = vec[3 * e + 1], vz = vec[3 * e + 2];
  const double r = sqrt(vx * vx + vy * vy + vz * vz);
  const double inv = 1.0 / fmax(r, 1e-12);
  const double ux = vx * inv, uy = vy * inv, uz = vz * inv;
  double gxv = 0.0, gyv = 0.0, gzv = 0.0;
  if (gy != nullptr) {
    double g[NQB_MAX_S];
#pragma unroll
    for (int q = 0; q < S; ++q) g[q] = (double)gy[e * S + q];
    double Gx, Gy, Gz, D;
    sh_vjp<LMAX>(ux, uy, uz, g, Gx, Gy, Gz, D);
    gxv = (Gx - D * ux) * inv; gyv = (Gy - D * uy) * inv; gzv = (Gz - D * uz) * inv;
  }
  if (gemb != nullptr) {
    const double recip = kTyped ? edge_recip(et, E, e) : 0.0;
    const double x = kTyped ? r * recip : r / prm.r_max;
    const double fc = poly_cutoff(x, prm.poly_p), dfc = poly_cutoff_deriv(x, prm.poly_p);
    double dr = 0.0;
    for (int n = 1; n <= prm.num_bessel; ++n) {
      const double t = (double)n * x;
      double b, db;  // b = sin(pi n x)/(pi x), db = d b / d x
      if (t == 0.0) { b = (double)n; db = 0.0; }
      else {
        const double s = sinpi(t), c = cospi(t);
        b = s / (M_PI * x);
        db = ((double)n * c) / x - s / (M_PI * x * x);
      }
      dr += (double)gemb[e * prm.num_bessel + (n - 1)] * (db * fc + b * dfc);
    }
    dr *= kTyped ? prm.prefactor * recip : prm.prefactor / prm.r_max;  // dx/dr = recip (typed) or 1 / r_max
    gxv += dr * ux; gyv += dr * uy; gzv += dr * uz;
  }
  if (gvec != nullptr) { gvec[3 * e] = gxv; gvec[3 * e + 1] = gyv; gvec[3 * e + 2] = gzv; }
  if (gpos != nullptr) {
    const int64_t i0 = eidx[e], i1 = eidx[E + e];
    atomicAdd(gpos + 3 * i1, gxv); atomicAdd(gpos + 3 * i1 + 1, gyv); atomicAdd(gpos + 3 * i1 + 2, gzv);
    atomicAdd(gpos + 3 * i0, -gxv); atomicAdd(gpos + 3 * i0 + 1, -gyv); atomicAdd(gpos + 3 * i0 + 2, -gzv);
  }
}

extern "C" int nqb_edge_embed_fwd(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                                  const double* pos, const int64_t* edge_index, const double* shift,
                                  const double* cell, int64_t N, int64_t E, int out_dtype, double* vec, void* y,
                                  void* emb, nqb_stream_t st) {
  (void)N;
  if (lmax < 0 || lmax > 4) return fail("nqb_edge_embed_fwd: lmax=%d unsupported (0..4)", lmax);
  if (num_bessel < 1 || num_bessel > NQB_MAX_BESSEL) return fail("nqb_edge_embed_fwd: bad num_bessel %d", num_bessel);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_edge_embed_fwd: bad dtype");
  if (!(r_max > 0.0) || !(poly_p >= 2.0)) return fail("nqb_edge_embed_fwd: need r_max > 0 and p >= 2");
  if (E < 0) return fail("nqb_edge_embed_fwd: negative size");
  if (E == 0) return 0;
  if (!pos || !edge_index || !vec || !y || !emb) return fail("nqb_edge_embed_fwd: null pointer");
  if ((shift == nullptr) != (cell == nullptr)) return fail("nqb_edge_embed_fwd: shift and cell must come together");
  EmbedParams prm{num_bessel, r_max, poly_p, prefactor};
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
#define EE_FWD(L, TT) k_edge_embed_fwd<L, TT><<<blocks, 128, 0, s>>>(prm, pos, edge_index, shift, cell, E, vec, (TT*)y, (TT*)emb, EdgeTypes{}, nullptr)
  if (out_dtype == NQB_F32) {
    switch (lmax) { case 0: EE_FWD(0, float); break; case 1: EE_FWD(1, float); break; case 2: EE_FWD(2, float); break; case 3: EE_FWD(3, float); break; default: EE_FWD(4, float); break; }
  } else {
    switch (lmax) { case 0: EE_FWD(0, double); break; case 1: EE_FWD(1, double); break; case 2: EE_FWD(2, double); break; case 3: EE_FWD(3, double); break; default: EE_FWD(4, double); break; }
  }
#undef EE_FWD
  NQB_LAUNCH_CHECK("nqb_edge_embed_fwd");
  return 0;
}

extern "C" int nqb_edge_embed_bwd(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                                  const double* vec, const int64_t* edge_index, int64_t N, int64_t E,
                                  int out_dtype, const void* grad_y, const void* grad_emb, double* grad_pos,
                                  double* grad_vec, nqb_stream_t st) {
  (void)N;
  if (lmax < 0 || lmax > 4) return fail("nqb_edge_embed_bwd: lmax=%d unsupported (0..4)", lmax);
  if (num_bessel < 1 || num_bessel > NQB_MAX_BESSEL) return fail("nqb_edge_embed_bwd: bad num_bessel %d", num_bessel);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_edge_embed_bwd: bad dtype");
  if (E < 0) return fail("nqb_edge_embed_bwd: negative size");
  if (E == 0) return 0;
  if (!vec) return fail("nqb_edge_embed_bwd: null vec");
  if (grad_pos && !edge_index) return fail("nqb_edge_embed_bwd: grad_pos needs edge_index");
  EmbedParams prm{num_bessel, r_max, poly_p, prefactor};
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
#define EE_BWD(L, TT) k_edge_embed_bwd<L, TT><<<blocks, 128, 0, s>>>(prm, vec, edge_index, E, (const TT*)grad_y, (const TT*)grad_emb, grad_pos, grad_vec, EdgeTypes{})
  if (out_dtype == NQB_F32) {
    switch (lmax) { case 0: EE_BWD(0, float); break; case 1: EE_BWD(1, float); break; case 2: EE_BWD(2, float); break; case 3: EE_BWD(3, float); break; default: EE_BWD(4, float); break; }
  } else {
    switch (lmax) { case 0: EE_BWD(0, double); break; case 1: EE_BWD(1, double); break; case 2: EE_BWD(2, double); break; case 3: EE_BWD(3, double); break; default: EE_BWD(4, double); break; }
  }
#undef EE_BWD
  NQB_LAUNCH_CHECK("nqb_edge_embed_bwd");
  return 0;
}

static int check_edge_types(const char* what, const int64_t* types, const int64_t* type_index, const double* recip,
                            int T) {
  if (T < 1) return fail("%s: need at least one type", what);
  if (!types || !type_index || !recip) return fail("%s: null types / type_index / recip", what);
  return 0;
}

extern "C" int nqb_edge_embed_fwd_typed(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                                        const double* pos, const int64_t* edge_index, const double* shift,
                                        const double* cell, int64_t N, int64_t E, const int64_t* types,
                                        const int64_t* type_index, const double* recip, int T, int out_dtype,
                                        double* vec, void* y, void* emb, nqb_stream_t st) {
  (void)N;
  if (lmax < 0 || lmax > 4) return fail("nqb_edge_embed_fwd_typed: lmax=%d unsupported (0..4)", lmax);
  if (num_bessel < 1 || num_bessel > NQB_MAX_BESSEL) return fail("nqb_edge_embed_fwd_typed: bad num_bessel %d", num_bessel);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_edge_embed_fwd_typed: bad dtype");
  if (!(r_max > 0.0) || !(poly_p >= 2.0)) return fail("nqb_edge_embed_fwd_typed: need r_max > 0 and p >= 2");
  if (E < 0) return fail("nqb_edge_embed_fwd_typed: negative size");
  if (E == 0) return 0;
  if (!pos || !edge_index || !vec || !y || !emb) return fail("nqb_edge_embed_fwd_typed: null pointer");
  if ((shift == nullptr) != (cell == nullptr)) return fail("nqb_edge_embed_fwd_typed: shift and cell must come together");
  if (int rc = check_edge_types("nqb_edge_embed_fwd_typed", types, type_index, recip, T)) return rc;
  EmbedParams prm{num_bessel, r_max, poly_p, prefactor};
  const EdgeTypes et{types, type_index, recip, T};
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
#define EE_FWD(L, TT) k_edge_embed_fwd<L, TT, true><<<blocks, 128, 0, s>>>(prm, pos, edge_index, shift, cell, E, vec, (TT*)y, (TT*)emb, et, nullptr)
  if (out_dtype == NQB_F32) {
    switch (lmax) { case 0: EE_FWD(0, float); break; case 1: EE_FWD(1, float); break; case 2: EE_FWD(2, float); break; case 3: EE_FWD(3, float); break; default: EE_FWD(4, float); break; }
  } else {
    switch (lmax) { case 0: EE_FWD(0, double); break; case 1: EE_FWD(1, double); break; case 2: EE_FWD(2, double); break; case 3: EE_FWD(3, double); break; default: EE_FWD(4, double); break; }
  }
#undef EE_FWD
  NQB_LAUNCH_CHECK("nqb_edge_embed_fwd_typed");
  return 0;
}

extern "C" int nqb_edge_embed_bwd_typed(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                                        const double* vec, const int64_t* edge_index, int64_t N, int64_t E,
                                        const int64_t* types, const int64_t* type_index, const double* recip, int T,
                                        int out_dtype, const void* grad_y, const void* grad_emb, double* grad_pos,
                                        double* grad_vec, nqb_stream_t st) {
  (void)N;
  if (lmax < 0 || lmax > 4) return fail("nqb_edge_embed_bwd_typed: lmax=%d unsupported (0..4)", lmax);
  if (num_bessel < 1 || num_bessel > NQB_MAX_BESSEL) return fail("nqb_edge_embed_bwd_typed: bad num_bessel %d", num_bessel);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_edge_embed_bwd_typed: bad dtype");
  if (E < 0) return fail("nqb_edge_embed_bwd_typed: negative size");
  if (E == 0) return 0;
  if (!vec) return fail("nqb_edge_embed_bwd_typed: null vec");
  if (grad_pos && !edge_index) return fail("nqb_edge_embed_bwd_typed: grad_pos needs edge_index");
  if (int rc = check_edge_types("nqb_edge_embed_bwd_typed", types, type_index, recip, T)) return rc;
  EmbedParams prm{num_bessel, r_max, poly_p, prefactor};
  const EdgeTypes et{types, type_index, recip, T};
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
#define EE_BWD(L, TT) k_edge_embed_bwd<L, TT, true><<<blocks, 128, 0, s>>>(prm, vec, edge_index, E, (const TT*)grad_y, (const TT*)grad_emb, grad_pos, grad_vec, et)
  if (out_dtype == NQB_F32) {
    switch (lmax) { case 0: EE_BWD(0, float); break; case 1: EE_BWD(1, float); break; case 2: EE_BWD(2, float); break; case 3: EE_BWD(3, float); break; default: EE_BWD(4, float); break; }
  } else {
    switch (lmax) { case 0: EE_BWD(0, double); break; case 1: EE_BWD(1, double); break; case 2: EE_BWD(2, double); break; case 3: EE_BWD(3, double); break; default: EE_BWD(4, double); break; }
  }
#undef EE_BWD
  NQB_LAUNCH_CHECK("nqb_edge_embed_bwd_typed");
  return 0;
}

// A batch of frames: as nqb_edge_embed_fwd with cells [F, 3, 3] (device) and frame [N] i64 (the frame of each atom);
// edge e takes the cell of frame[edge_index[0][e]].  Per-edge-type cutoffs as nqb_edge_embed_fwd_typed when types,
// type_index and recip are given, none when all three are NULL.  The backward is nqb_edge_embed_bwd(_typed).
extern "C" int nqb_edge_embed_fwd_frames(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                                         const double* pos, const int64_t* edge_index, const double* shift,
                                         const double* cells, const int64_t* frame, int64_t N, int64_t E,
                                         const int64_t* types, const int64_t* type_index, const double* recip, int T,
                                         int out_dtype, double* vec, void* y, void* emb, nqb_stream_t st) {
  (void)N;
  if (lmax < 0 || lmax > 4) return fail("nqb_edge_embed_fwd_frames: lmax=%d unsupported (0..4)", lmax);
  if (num_bessel < 1 || num_bessel > NQB_MAX_BESSEL) return fail("nqb_edge_embed_fwd_frames: bad num_bessel %d", num_bessel);
  if (out_dtype != NQB_F32 && out_dtype != NQB_F64) return fail("nqb_edge_embed_fwd_frames: bad dtype");
  if (!(r_max > 0.0) || !(poly_p >= 2.0)) return fail("nqb_edge_embed_fwd_frames: need r_max > 0 and p >= 2");
  if (E < 0) return fail("nqb_edge_embed_fwd_frames: negative size");
  if (E == 0) return 0;
  if (!pos || !edge_index || !shift || !cells || !frame || !vec || !y || !emb)
    return fail("nqb_edge_embed_fwd_frames: null pointer");
  const bool typed = types || type_index || recip;
  if (typed)
    if (int rc = check_edge_types("nqb_edge_embed_fwd_frames", types, type_index, recip, T)) return rc;
  EmbedParams prm{num_bessel, r_max, poly_p, prefactor};
  const EdgeTypes et{types, type_index, recip, T};
  unsigned blocks = (unsigned)((E + 127) / 128);
  cudaStream_t s = (cudaStream_t)st;
#define EE_FWD(L, TT)                                                                                                  \
  (typed ? k_edge_embed_fwd<L, TT, true, true><<<blocks, 128, 0, s>>>(prm, pos, edge_index, shift, cells, E, vec,      \
                                                                      (TT*)y, (TT*)emb, et, frame)                     \
         : k_edge_embed_fwd<L, TT, false, true><<<blocks, 128, 0, s>>>(prm, pos, edge_index, shift, cells, E, vec,     \
                                                                       (TT*)y, (TT*)emb, et, frame))
  if (out_dtype == NQB_F32) {
    switch (lmax) { case 0: EE_FWD(0, float); break; case 1: EE_FWD(1, float); break; case 2: EE_FWD(2, float); break; case 3: EE_FWD(3, float); break; default: EE_FWD(4, float); break; }
  } else {
    switch (lmax) { case 0: EE_FWD(0, double); break; case 1: EE_FWD(1, double); break; case 2: EE_FWD(2, double); break; case 3: EE_FWD(3, double); break; default: EE_FWD(4, double); break; }
  }
#undef EE_FWD
  NQB_LAUNCH_CHECK("nqb_edge_embed_fwd_frames");
  return 0;
}

// ------------------------------------------------------------------------------------------
// Gate nonlinearity (e3nn nn.Gate with normalize2mom'd SiLU / tanh; nequip/nn/convnetlayer.py:42-56,
// 104-112), forward and backward as one kernel each instead of ~30 strided torch ops per layer.
//   out[n, j] = gate[j] < 0 ? act_kind[j](x[n, src[j]]) : x[n, src[j]] * act_kind[j](x[n, gate[j]])
// The tables are built by the host from the irreps (any layout): src/gate = input columns, kind = 0 for
// c_silu * silu, 1 for c_tanh * tanh.  Backward table per INPUT column i (6 ints):
//   {role, a, b, c, d, kind}: role 0 scalar: a = output column
//                             role 1 gated value: a = output column, b = its gate's input column
//                             role 2 gate: a = first output column, b = first gated input column,
//                                          c = stride between the (2l+1) components, d = 2l+1
// ------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T gate_act(T v, int kind) {
  const T c_silu = (T)1.6791767923989418, c_tanh = (T)1.5937334472592692;
  if (kind == 0) return c_silu * v / ((T)1 + exp(-v));
  return c_tanh * tanh(v);
}
template <typename T>
__device__ __forceinline__ T gate_act_grad(T v, int kind) {
  const T c_silu = (T)1.6791767923989418, c_tanh = (T)1.5937334472592692;
  if (kind == 0) {
    const T s = (T)1 / ((T)1 + exp(-v));
    return c_silu * s * ((T)1 + v * ((T)1 - s));
  }
  const T t = tanh(v);
  return c_tanh * ((T)1 - t * t);
}

template <typename T>
__global__ void k_gate_fwd(const T* __restrict__ x, int64_t N, int d_in, int d_out, const int32_t* __restrict__ src,
                           const int32_t* __restrict__ gate, const int32_t* __restrict__ kind, T* __restrict__ out) {
  const int64_t total = N * (int64_t)d_out;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = idx / d_out;
    const int j = (int)(idx - n * d_out);
    const T* xr = x + n * d_in;
    const int g = gate[j];
    const T v = xr[src[j]];
    out[idx] = g < 0 ? gate_act(v, kind[j]) : v * gate_act(xr[g], kind[j]);
  }
}

template <typename T>
__global__ void k_gate_bwd(const T* __restrict__ x, const T* __restrict__ gout, int64_t N, int d_in, int d_out,
                           const int32_t* __restrict__ tab, T* __restrict__ gx) {
  const int64_t total = N * (int64_t)d_in;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = idx / d_in;
    const int i = (int)(idx - n * d_in);
    const int32_t* t = tab + 6 * i;
    const T* xr = x + n * d_in;
    const T* gr = gout + n * d_out;
    T r;
    if (t[0] == 0) {
      r = gr[t[1]] * gate_act_grad(xr[i], t[5]);
    } else if (t[0] == 1) {
      r = gr[t[1]] * gate_act(xr[t[2]], t[5]);
    } else {
      T s = (T)0;
      for (int c = 0; c < t[4]; ++c) s += gr[t[1] + c * t[3]] * xr[t[2] + c * t[3]];
      r = s * gate_act_grad(xr[i], t[5]);
    }
    gx[idx] = r;
  }
}

static unsigned gate_grid(int64_t total) {
  const int64_t need = (total + 255) / 256;
  return (unsigned)(need < 132 * 16 ? need : 132 * 16);
}

extern "C" int nqb_gate_fwd(int dtype, const void* x, int64_t N, int d_in, int d_out, const int32_t* src,
                            const int32_t* gate, const int32_t* kind, void* out, nqb_stream_t st) {
  if (dtype != NQB_F32 && dtype != NQB_F64) return fail("nqb_gate_fwd: bad dtype");
  if (N < 0 || d_in <= 0 || d_out <= 0) return fail("nqb_gate_fwd: bad shape");
  if (N == 0) return 0;
  if (!x || !src || !gate || !kind || !out) return fail("nqb_gate_fwd: null pointer");
  const int64_t total = N * (int64_t)d_out;
  if (dtype == NQB_F32)
    k_gate_fwd<float><<<gate_grid(total), 256, 0, (cudaStream_t)st>>>((const float*)x, N, d_in, d_out, src, gate, kind, (float*)out);
  else
    k_gate_fwd<double><<<gate_grid(total), 256, 0, (cudaStream_t)st>>>((const double*)x, N, d_in, d_out, src, gate, kind, (double*)out);
  NQB_LAUNCH_CHECK("nqb_gate_fwd");
  return 0;
}

extern "C" int nqb_gate_bwd(int dtype, const void* x, const void* grad_out, int64_t N, int d_in, int d_out,
                            const int32_t* tab, void* grad_x, nqb_stream_t st) {
  if (dtype != NQB_F32 && dtype != NQB_F64) return fail("nqb_gate_bwd: bad dtype");
  if (N < 0 || d_in <= 0 || d_out <= 0) return fail("nqb_gate_bwd: bad shape");
  if (N == 0) return 0;
  if (!x || !grad_out || !tab || !grad_x) return fail("nqb_gate_bwd: null pointer");
  const int64_t total = N * (int64_t)d_in;
  if (dtype == NQB_F32)
    k_gate_bwd<float><<<gate_grid(total), 256, 0, (cudaStream_t)st>>>((const float*)x, (const float*)grad_out, N, d_in, d_out, tab, (float*)grad_x);
  else
    k_gate_bwd<double><<<gate_grid(total), 256, 0, (cudaStream_t)st>>>((const double*)x, (const double*)grad_out, N, d_in, d_out, tab, (double*)grad_x);
  NQB_LAUNCH_CHECK("nqb_gate_bwd");
  return 0;
}
