/*
 * nqb.h -- C ABI of the H100-native NequIP hot path (libnqb.so).
 *
 * Plain C: raw device pointers, sizes, a CUDA stream.  No torch / C++ types cross
 * this boundary.  Every tensor is caller-allocated (torch caching allocator on the
 * Python side) and only borrowed for the stream-ordered duration of the call; the
 * library never allocates device memory per call and never synchronises the
 * device.  All functions return 0 on success; otherwise nqb_last_error() holds a
 * thread-local message (the Python wrapper raises RuntimeError, in the style of
 * the reference's modifiers, nequip/nn/_tp_scatter_base.py:57-58).
 *
 * Reference interfaces these entry points replace (paths under /root/reference):
 *   nqb_tp_scatter_fwd/bwd  TensorProductScatter.forward + its autograd
 *                           nequip/nn/_tp_scatter_base.py:35-38
 *                           (e3nn o3.TensorProduct 'uvu' + nequip/nn/utils.py:24-53 scatter;
 *                            same seat as OpenEquivariance's TensorProductConv,
 *                            nequip/nn/_tp_scatter_oeq.py:29-57, and cuEquivariance's
 *                            fused_tp, nequip/nn/_tp_scatter_cueq.py:90-122)
 *   nqb_plan_create         TensorProductScatter.__init__  nequip/nn/_tp_scatter_base.py:10-33
 *                           (path table built at nequip/nn/interaction_block.py:89-116)
 *   nqb_csr_*               the (dst,src)-sorted edge contract of
 *                           nequip/data/transforms/neighborlist.py:120-157
 *   nqb_edge_embed_fwd/bwd  with_edge_vectors_  nequip/nn/utils.py:68-118,
 *                           SphericalHarmonicEdgeAttrs.forward  nequip/nn/embedding/_edge.py:193-198,
 *                           EdgeLengthNormalizer :65-80, BesselEdgeLengthEncoding :136-150,
 *                           PolynomialCutoff  nequip/nn/embedding/cutoffs.py:17-27,
 *                           ApplyFactor  nequip/nn/misc.py:46-48
 *   nqb_sh_fwd/bwd          e3nn o3.SphericalHarmonics(normalize=True, "component") as
 *                           constructed at nequip/nn/embedding/_edge.py:187-189
 */
#ifndef NQB_H
#define NQB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* nqb_stream_t; /* == cudaStream_t */
typedef struct nqb_plan nqb_plan;

typedef struct nqb_irrep {
  int32_t mul;
  int32_t l;
  int32_t p; /* +1 even, -1 odd */
} nqb_irrep;

typedef struct nqb_instruction {
  int32_t i_in1;
  int32_t i_in2;
  int32_t i_out; /* 'uvu', has_weight=True */
} nqb_instruction;

enum { NQB_F32 = 0, NQB_F64 = 1 };

/* library / error handling */
int nqb_abi_version(void);
const char* nqb_last_error(void);

/* Plan: immutable description of one TensorProductScatter signature bound to the
 * specialised kernel library generated for it (spec_lib_path, built by
 * nequip_b200.build; its embedded signature string is validated against the
 * descriptors).  Thread-safe to share between the forward and autograd threads. */
int nqb_plan_create(const nqb_irrep* in1, int n_in1, const nqb_irrep* in2, int n_in2,
                    const nqb_irrep* out, int n_out, const nqb_instruction* ins, int n_ins,
                    const char* spec_lib_path, nqb_plan** plan);
void nqb_plan_destroy(nqb_plan* plan);
int nqb_plan_dims(const nqb_plan* plan, int* d_in, int* s_dim, int* weight_numel, int* d_out);
/* writes the canonical signature (NUL terminated) into buf; returns needed length */
int nqb_plan_signature(const nqb_plan* plan, char* buf, int buflen);

/* Destination-CSR helpers.  edge_dst must be non-decreasing for
 * nqb_csr_from_sorted (the reference's neighbour lists are grouped by centre atom);
 * nqb_csr_check_sorted writes 1/0 into *flag_dev (fully written).  For unsorted edges the caller
 * supplies perm (stable argsort of edge_dst) and the sorted keys.
 * row_ptr [N+1] is fully written (row_ptr[n] = first slot whose key >= n; E = 0 gives all zeros). */
int nqb_csr_check_sorted(const int64_t* keys, int64_t E, int32_t* flag_dev, nqb_stream_t st);
int nqb_csr_from_sorted(const int64_t* sorted_keys, int64_t E, int64_t N, int64_t* row_ptr /* [N+1] */,
                        nqb_stream_t st);

/* out[N, D_mid] = scatter_dst( TP_uvu( x[src], y, w ) ).  Every element of out is
 * written exactly once (no pre-zeroing needed, deterministic).
 *   x [N, D_in], y [E, S], w [E, W], out [N, D_mid]: dtype NQB_F32/NQB_F64, row-major, in the layout the plan's
 *   kernel library was generated for (mul_ir or ir_mul, nequip_b200/codegen.py GenOptions.layout).
 *   out is fully written, also for nodes without edges (E = 0 included) and in irreps_out chunks no instruction
 *   writes (zeros).
 *   row_ptr [N+1]: CSR over edges ordered by destination; perm [E] or NULL (identity):
 *   slot s of the CSR refers to edge perm[s]; src [E]: source node of each edge (original order). */
int nqb_tp_scatter_fwd(const nqb_plan* plan, int dtype, const void* x, const void* y, const void* w,
                       const int64_t* row_ptr, const int64_t* perm, const int64_t* src, int64_t N,
                       int64_t E, void* out, nqb_stream_t st);

/* Gradients of the above.  grad_w [E, W] is fully written.  grad_y [E, S] and
 * grad_x [N, D_in] are ACCUMULATED INTO (caller zero-fills); grad_x may be NULL
 * (skips the source-row reduction, e.g. first layer at inference; grad_y and grad_w are the same as with it).
 * E = 0 writes nothing (grad_w has no rows). */
int nqb_tp_scatter_bwd(const nqb_plan* plan, int dtype, const void* x, const void* y, const void* w,
                       const int64_t* row_ptr, const int64_t* perm, const int64_t* src,
                       const void* grad_out, int64_t N, int64_t E, void* grad_x, void* grad_y,
                       void* grad_w, int deterministic,
                       nqb_stream_t st);
/* deterministic != 0 (bitwise-repeatable backward; the default accumulates grad_x / grad_Y with red.global.add in
 * whatever order the edges retire, as the reference's OpenEquivariance back-end does, nequip/nn/_tp_scatter_oeq.py:46):
 *   grad_x is then an [E, D_in] buffer, FULLY WRITTEN -- every edge stores its contribution to its SOURCE atom in its
 *   own row, zeros in the columns of irreps_in1 chunks no instruction reads -- to be
 *   reduced over the source-sorted edges with nqb_segment_sum (perm = stable argsort of edge_src, the
 *   edge_transpose_perm of nequip/data/transforms/neighborlist.py:150-155; seg_ptr = CSR over the sorted sources);
 *   grad_y is [nqb_tp_scatter_gy_slices(plan, dtype), E, S], ACCUMULATED INTO (zero-initialised by the caller): each
 *   writer owns a slice, the caller sums the slices in index order.
 * nqb_segment_sum: out [N, D] is fully written (a segment without rows gives 0). */
int nqb_tp_scatter_gy_slices(const nqb_plan* plan, int dtype);
int nqb_segment_sum(int dtype, const void* rows /* [R, D] */, int D, const int64_t* perm, const int64_t* seg_ptr /* [N+1] */,
                    int64_t N, void* out /* [N, D] */, nqb_stream_t st);

/* Real spherical harmonics, "component" normalisation, input normalised (lmax <= 4).
 *   vec [E,3] f64 -> y [E,(lmax+1)^2] of out_dtype (computed in f64, then cast); y is fully written. */
int nqb_sh_fwd(int lmax, const double* vec, int64_t E, int out_dtype, void* y, nqb_stream_t st);
/*   grad_vec [E,3] f64 = J^T grad_y (includes the normalisation Jacobian); fully written */
int nqb_sh_bwd(int lmax, const double* vec, int64_t E, int out_dtype, const void* grad_y,
               double* grad_vec, nqb_stream_t st);

/* Fused "last radial-MLP layer -> tensor product -> scatter" forward (SURVEY.md section 8f-1):
 *   out[n] = sum_{e: dst[e] = n} TP_uvu(x[src[e]], y[e], w[e]),   w[e] = h[e, :K] @ (W2 * alpha2)
 * i.e. nequip/nn/mlp.py:262-268 (the last ScalarLinearLayer built at nequip/nn/interaction_block.py:119-127)
 * composed with TensorProductScatter.forward (nequip/nn/_tp_scatter_base.py:35-38) so that the [E, W] weight
 * tensor is never written (w_out == NULL) -- or is written once on the side for an unfused backward.
 * out [N, D_mid] is fully written (nodes without edges and E = 0 included); w_out [E, W], when given, is fully
 * written.  h [E, ldh] is read in its first K columns only; h must be 16-byte aligned.
 * float32, ir_mul node layout, edges grouped by destination (row_ptr; no permutation), K <= 128, K % 8 == 0.
 * nqb_tp_fused_slices(plan): number of 128-row weight slices of the signature, 0 = no fused kernel built.
 * w2_prepared: per slice, the tf32 hi and lo parts of the [128 x 128] block W2^T (rows = the slice's columns of the
 *   weight matrix in nequip_b200/codegen.py TPGenerator.fused_layout()["cols"] order, -1 = zero row; K zero padded
 *   to 128), scaled by alpha2, each block in the canonical K-major core-matrix order (ops.FusedTPWeights).
 * slice_cta0 [slices + 1] (device, int32): CTAs [cta0[s], cta0[s+1]) process slice s; nctas = cta0[slices]
 *   (one CTA per SM; the host splits the grid in proportion to the slices' costs). */
int nqb_tp_fused_slices(const nqb_plan* plan);
int nqb_tp_fused_fwd(const nqb_plan* plan, const float* x, const float* y, const float* h, int64_t ldh, int K,
                     const float* w2_prepared, const int64_t* row_ptr, const int64_t* src, int64_t N, int64_t E,
                     float* out, float* w_out, const int32_t* slice_cta0, int nctas, nqb_stream_t st);

/* Fused edge geometry + embeddings:
 *   r_ij = pos[idx1] - pos[idx0] + shift @ cell ; Y = SH(r_ij) ;
 *   emb[:, n] = sinc(n x) n * f_cut(x) * prefactor , x = |r|/r_max, n = 1..num_bessel
 * edge_index [2,E] i64; shift [E,3] f64 or NULL; cell [3,3] f64 (rows = lattice vectors) or NULL.
 * Outputs, each fully written: vec [E,3] f64 (kept for backward), y [E,S], emb [E,num_bessel] (out_dtype). */
int nqb_edge_embed_fwd(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                       const double* pos, const int64_t* edge_index, const double* shift,
                       const double* cell, int64_t N, int64_t E, int out_dtype, double* vec, void* y,
                       void* emb, nqb_stream_t st);
/* grad_pos [N,3] f64 is ACCUMULATED INTO (caller zero-fills):
 *   g = J_Y^T grad_y + J_emb^T grad_emb ;  grad_pos[idx1] += g ; grad_pos[idx0] -= g.
 * grad_vec [E,3] f64 (may be NULL) receives g itself (per-edge forces / virial assembly); fully written. */
int nqb_edge_embed_bwd(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                       const double* vec, const int64_t* edge_index, int64_t N, int64_t E,
                       int out_dtype, const void* grad_y, const void* grad_emb, double* grad_pos,
                       double* grad_vec, nqb_stream_t st);
/* Per-edge-type cutoffs (nequip/nn/embedding/_edge.py:65-80 with per_edge_type_cutoff): as nqb_edge_embed_fwd/bwd,
 * with the normalised length x = |r| * recip[T * types[type_index[0][e]] + types[type_index[1][e]]] (and dx/d|r| =
 * that recip) in place of |r| / r_max; prefactor stays the caller's (2 pi / r_max^2 of the global r_max).
 * types [N'] i64 in [0, T), type_index [2,E] i64, recip [T*T] f64 (1 / rc[source, target]): device arrays.
 * type_index is edge_index for positions; given edge vectors come with made-up positions, and type_index is then the
 * real list.  Same write contracts. */
int nqb_edge_embed_fwd_typed(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                             const double* pos, const int64_t* edge_index, const double* shift,
                             const double* cell, int64_t N, int64_t E, const int64_t* types,
                             const int64_t* type_index, const double* recip, int T, int out_dtype, double* vec,
                             void* y, void* emb, nqb_stream_t st);
int nqb_edge_embed_bwd_typed(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                             const double* vec, const int64_t* edge_index, int64_t N, int64_t E,
                             const int64_t* types, const int64_t* type_index, const double* recip, int T,
                             int out_dtype, const void* grad_y, const void* grad_emb, double* grad_pos,
                             double* grad_vec, nqb_stream_t st);
/* A batch of frames (nequip/nn/utils.py:96-106, the cell of an edge is cell[batch[edge_index[0]]]): as
 * nqb_edge_embed_fwd with shift [E,3], cells [F,3,3] and frame [N] i64 in [0, F) (the frame of each atom), all
 * device arrays and all required; edge e takes cells + 9 * frame[edge_index[0][e]] in the same shift expression, so
 * each frame's outputs are bitwise those of nqb_edge_embed_fwd with that frame's cell.  types / type_index / recip /
 * T as nqb_edge_embed_fwd_typed, or all three NULL for the untyped embedding.  Same write contracts.  The backward
 * reads the stored edge vectors only: nqb_edge_embed_bwd(_typed) serves framed edges unchanged. */
int nqb_edge_embed_fwd_frames(int lmax, int num_bessel, double r_max, double poly_p, double prefactor,
                              const double* pos, const int64_t* edge_index, const double* shift, const double* cells,
                              const int64_t* frame, int64_t N, int64_t E, const int64_t* types,
                              const int64_t* type_index, const double* recip, int T, int out_dtype, double* vec,
                              void* y, void* emb, nqb_stream_t st);

/* ZBL pair energy (nequip/nn/pair_potential.py:230-386), everything in fp64.  Per edge e = (i -> j), i =
 * edge_index[0][e]:  eps_e = A[ti,tj] / r * psi((S[ti,tj] * r) / a0) * f_c(r / r_max),  psi = the four-exponential
 * LAMMPS screening function, f_c = PolynomialCutoff(poly_p) (rounded to float32 when cutoff_f32 != 0).
 *   Geometry: either pos [N,3] with optional shift [E,3] + cell [3,3] (r = pos[j] - pos[i] + shift @ cell, the
 *   arithmetic of nqb_edge_embed_fwd), or given edge vectors vec [E,3] (pos, shift, cell NULL).
 *   types [N] i64 in [0, T); table [T,T,2] f64: {A = 0.5 * qqr2e * Z_i Z_j, S = Z_i^0.23 + Z_j^0.23} per ordered pair.
 * nqb_zbl_fwd: row_ptr [N+1] / perm [E] or NULL: the destination CSR of edge_index[0] (nqb_csr_from_sorted).
 *   e_atom [N] is fully written, each element once, no atomics: e_atom[i] = sum of the row's eps_e in CSR order
 *   (bitwise repeatable; a row without edges gives 0; an edge with r >= r_max adds exactly +0).
 * nqb_zbl_bwd: g_e = grad_e_atom[i] * d eps_e / dr * r / |r|.  grad_pos [N,3] (positions only) is ACCUMULATED INTO:
 *   grad_pos[j] += g_e, grad_pos[i] -= g_e (fp64 atomics); grad_vec [E,3] is fully written with g_e.  At least one
 *   of the two must be given; E = 0 writes nothing. */
int nqb_zbl_fwd(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                const double* vec, const int64_t* types, const double* table, int T, const int64_t* row_ptr,
                const int64_t* perm, int64_t N, int64_t E, double r_max, double poly_p, int cutoff_f32,
                double* e_atom, nqb_stream_t st);
int nqb_zbl_bwd(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                const double* vec, const int64_t* types, const double* table, int T, int64_t N, int64_t E,
                double r_max, double poly_p, int cutoff_f32, const double* grad_e_atom, double* grad_pos,
                double* grad_vec, nqb_stream_t st);
/* Per-edge-type cutoffs: the envelope takes x = r * recip[T * t_i + t_j] (recip [T*T] f64, device) instead of
 * r * (1 / r_max); the ZBL term itself keeps r.  An edge with x >= 1 adds exactly +0.  Same write contracts. */
int nqb_zbl_fwd_typed(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                      const double* vec, const int64_t* types, const double* table, int T, const int64_t* row_ptr,
                      const int64_t* perm, int64_t N, int64_t E, double r_max, double poly_p, int cutoff_f32,
                      const double* recip, double* e_atom, nqb_stream_t st);
int nqb_zbl_bwd_typed(const double* pos, const int64_t* edge_index, const double* shift, const double* cell,
                      const double* vec, const int64_t* types, const double* table, int T, int64_t N, int64_t E,
                      double r_max, double poly_p, int cutoff_f32, const double* recip, const double* grad_e_atom,
                      double* grad_pos, double* grad_vec, nqb_stream_t st);
/* A batch of frames: as nqb_zbl_fwd / nqb_zbl_bwd on positions, with shift [E,3], cells [F,3,3] and frame [N] i64
 * in [0, F) (device arrays, required when E > 0); edge e takes cells + 9 * frame[edge_index[0][e]].  recip as the
 * _typed calls, or NULL for the untyped envelope.  Same write contracts. */
int nqb_zbl_fwd_frames(const double* pos, const int64_t* edge_index, const double* shift, const double* cells,
                       const int64_t* frame, const int64_t* types, const double* table, int T, const int64_t* row_ptr,
                       const int64_t* perm, int64_t N, int64_t E, double r_max, double poly_p, int cutoff_f32,
                       const double* recip, double* e_atom, nqb_stream_t st);
int nqb_zbl_bwd_frames(const double* pos, const int64_t* edge_index, const double* shift, const double* cells,
                       const int64_t* frame, const int64_t* types, const double* table, int T, int64_t N, int64_t E,
                       double r_max, double poly_p, int cutoff_f32, const double* recip, const double* grad_e_atom,
                       double* grad_pos, double* grad_vec, nqb_stream_t st);

/* Neighbour list on the device (cell list; full list, both directions, periodic images, no self edge in the home
 * image) -- replaces the host construction of nequip/data/_nl.py:60-152,292-361 and emits what
 * SortedNeighborListTransform (nequip/data/transforms/neighborlist.py:120-157) produces: edges sorted by
 * (centre, neighbour) = the destination CSR of the convolution.  Three calls around two host-side scans
 * (nequip_b200/ops.py neighbor_list): bins -> [sort atoms by bin] -> counts -> [exclusive scan] -> fill.
 * cell/inv: 3x3 row-major HOST arrays (rows = lattice vectors, inv = cell^-1); pbc/nbins/search: 3 ints;
 * lo/width: bounding box of the fractional coordinates in non-periodic directions (NULL if all periodic).
 * edge vector = pos[j] - pos[i] + shifts @ cell, i = edge_index[0][e] (centre), j = edge_index[1][e]. */
int nqb_nl_bin(const double* pos, int64_t N, const double* cell_host, const double* inv_host, const int* pbc,
               const int* nbins, const int* search, const double* lo, const double* width, double r_max,
               double* wpos /* [N,3] */, int32_t* base /* [N,3] */, int64_t* bin /* [N] */, int32_t* cidx /* [N,3] */,
               nqb_stream_t st);
int nqb_nl_count(int64_t N, const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                 const int* search, double r_max, const double* wpos, const int32_t* cidx, const int64_t* order,
                 const int64_t* bin_start, int64_t* counts /* [N] */, nqb_stream_t st);
int nqb_nl_fill(int64_t N, int64_t E, const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                const int* search, double r_max, const double* wpos, const int32_t* cidx, const int32_t* base,
                const int64_t* order, const int64_t* bin_start, const int64_t* row_ptr /* [N+1] */,
                int64_t* edge_index /* [2,E] */, double* shifts /* [E,3] */, nqb_stream_t st);
/* Capacity mode: a list of fixed length `capacity` whatever the frame's edge count E, so positions -> list -> model
 * is capturable in one CUDA graph (no host read of E).  Unused slots hold null edges (i, i, pad_shift): a self-edge
 * to a periodic image at least r_max + one lattice vector away, which contributes exactly zero energy and force.
 * nqb_nl_pad runs after the exclusive scan (row_ptr [N+1] of the exact list, N > 0):
 *   row_ptr_pad [N+1] fully written: row_ptr[i] + floor((capacity - E) * i / N), row_ptr_pad[N] = capacity, so
 *   every row gets floor or ceil of (capacity - E) / N null edges; when E > capacity, floor(capacity * i / N);
 *   num_edges [1] fully written: the true E (also on overflow); overflow [1] fully written: 1 if E > capacity, else 0. */
int nqb_nl_pad(int64_t N, int64_t capacity, const int64_t* row_ptr, int64_t* row_ptr_pad, int64_t* num_edges,
               int32_t* overflow, nqb_stream_t st);
/* edge_index [2,capacity] and shifts [capacity,3] fully written, nothing past capacity: row i holds
 * [row_ptr_pad[i], row_ptr_pad[i+1]), its real edges first (order and shifts as nqb_nl_fill; none on overflow), then
 * null edges (i, i, pad_shift).  pad_shift: 3 integer-valued doubles on the HOST; overflow: device flag of nqb_nl_pad. */
int nqb_nl_fill_capacity(int64_t N, int64_t capacity, const double* cell_host, const double* inv_host, const int* pbc,
                         const int* nbins, const int* search, double r_max, const double* wpos, const int32_t* cidx,
                         const int32_t* base, const int64_t* order, const int64_t* bin_start,
                         const int64_t* row_ptr_pad /* [N+1] */, const int32_t* overflow /* [1] */,
                         const double* pad_shift_host, int64_t* edge_index /* [2,capacity] */,
                         double* shifts /* [capacity,3] */, nqb_stream_t st);
/* Variable cell: the cell-dependent arguments (cell, inverse, periodicity, bin grid, search range, r_max and the
 * null-edge shift) live in a parameter block in DEVICE memory, so one captured graph follows a cell that changes between
 * replays.  The block's layout is private to the library: nqb_nl_params_bytes() is its size, and
 * nqb_nl_params_pack fills out_host [nqb_nl_params_bytes()] on the HOST with exactly the values the by-value calls
 * derive from the same arguments (host only, no CUDA call; every direction must be periodic).  The caller copies the
 * block to the device, stream-ordered before the calls that read it.
 * nqb_nl_bin_dp, nqb_nl_count_dp and nqb_nl_fill_capacity_dp have the write contracts of nqb_nl_bin (wpos, base, bin,
 * cidx fully written), nqb_nl_count (counts fully written) and nqb_nl_fill_capacity (edge_index, shifts fully written,
 * nothing past capacity; null edges carry the block's pad_shift). */
int64_t nqb_nl_params_bytes(void);
int nqb_nl_params_pack(const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                       const int* search, double r_max, const double* pad_shift_host, void* out_host);
int nqb_nl_bin_dp(const double* pos, int64_t N, const void* params_dev, double* wpos /* [N,3] */,
                  int32_t* base /* [N,3] */, int64_t* bin /* [N] */, int32_t* cidx /* [N,3] */, nqb_stream_t st);
int nqb_nl_count_dp(int64_t N, const void* params_dev, const double* wpos, const int32_t* cidx, const int64_t* order,
                    const int64_t* bin_start, int64_t* counts /* [N] */, nqb_stream_t st);
int nqb_nl_fill_capacity_dp(int64_t N, int64_t capacity, const void* params_dev, const double* wpos,
                            const int32_t* cidx, const int32_t* base, const int64_t* order, const int64_t* bin_start,
                            const int64_t* row_ptr_pad /* [N+1] */, const int32_t* overflow /* [1] */,
                            int64_t* edge_index /* [2,capacity] */, double* shifts /* [capacity,3] */,
                            nqb_stream_t st);
/* Open directions (pbc[d] == 0) in a parameter block, so that a captured list follows a molecule or slab whose
 * bounding box moves.  nqb_nl_params_pack_open fills out_host [nqb_nl_params_bytes()] fully, on the HOST, like
 * nqb_nl_params_pack but accepting open directions: periodic directions get the values nqb_nl_params_pack gives them;
 * an open direction's bounding box and grid are left for nqb_nl_bbox (a one-bin grid until it runs).  cap >= 1: most
 * bins along an open direction (the caller's scratch grid); perp_host: 3 finite positive doubles, the distance between
 * opposite faces of the cell along each lattice direction (1 / |column d of inv|); r_max finite and > 0.
 * nqb_nl_bbox (N >= 0; nothing for N = 0) writes, in the DEVICE block params_dev and nowhere else in it, for each
 * open direction d: lo = min over atoms of the fractional coordinate (computed as nqb_nl_bin_dp computes it),
 * width = max(fmax - fmin, 1e-9) * (1 + 1e-9), nb = min(cap, max(1, floor(perp[d] * width / r_max))), search = 1.
 * NaN coordinates are skipped; nb lies in [1, cap] for any input.  work [8] u64: zero before the first call, and
 * every call leaves it zero again (one work buffer per stream; no host synchronisation, capturable).  Run it
 * stream-ordered before nqb_nl_bin_dp; count, fill and the bin scratch then follow the device grid. */
int nqb_nl_params_pack_open(const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                            const int* search, double r_max, const double* pad_shift_host, int cap,
                            const double* perp_host, void* out_host);
int nqb_nl_bbox(const double* pos /* [N,3] */, int64_t N, void* params_dev, uint64_t* work /* [8] */,
                nqb_stream_t st);
/* Per-edge-type cutoffs: count, fill and fill with capacity (by value and _dp) with the membership test
 * d2 < rc2[T * types[i] + types[j]] in place of d2 < r_max^2.  types [N] i64 in [0, T) and rc2 [T*T] f64 (rc * rc in
 * float64, every rc <= r_max) are device arrays; bins, search ranges and parameter blocks stay those of r_max, so
 * nqb_nl_bin, nqb_nl_pad and nqb_nl_params_pack are shared.  Same write contracts as the untyped calls. */
int nqb_nl_count_typed(int64_t N, const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                       const int* search, double r_max, const double* wpos, const int32_t* cidx, const int64_t* order,
                       const int64_t* bin_start, const int64_t* types, const double* rc2, int T,
                       int64_t* counts /* [N] */, nqb_stream_t st);
int nqb_nl_fill_typed(int64_t N, int64_t E, const double* cell_host, const double* inv_host, const int* pbc,
                      const int* nbins, const int* search, double r_max, const double* wpos, const int32_t* cidx,
                      const int32_t* base, const int64_t* order, const int64_t* bin_start,
                      const int64_t* row_ptr /* [N+1] */, const int64_t* types, const double* rc2, int T,
                      int64_t* edge_index /* [2,E] */, double* shifts /* [E,3] */, nqb_stream_t st);
int nqb_nl_fill_capacity_typed(int64_t N, int64_t capacity, const double* cell_host, const double* inv_host,
                               const int* pbc, const int* nbins, const int* search, double r_max, const double* wpos,
                               const int32_t* cidx, const int32_t* base, const int64_t* order,
                               const int64_t* bin_start, const int64_t* row_ptr_pad /* [N+1] */,
                               const int32_t* overflow /* [1] */, const double* pad_shift_host, const int64_t* types,
                               const double* rc2, int T, int64_t* edge_index /* [2,capacity] */,
                               double* shifts /* [capacity,3] */, nqb_stream_t st);
int nqb_nl_count_dp_typed(int64_t N, const void* params_dev, const double* wpos, const int32_t* cidx,
                          const int64_t* order, const int64_t* bin_start, const int64_t* types, const double* rc2,
                          int T, int64_t* counts /* [N] */, nqb_stream_t st);
int nqb_nl_fill_capacity_dp_typed(int64_t N, int64_t capacity, const void* params_dev, const double* wpos,
                                  const int32_t* cidx, const int32_t* base, const int64_t* order,
                                  const int64_t* bin_start, const int64_t* row_ptr_pad /* [N+1] */,
                                  const int32_t* overflow /* [1] */, const int64_t* types, const double* rc2, int T,
                                  int64_t* edge_index /* [2,capacity] */, double* shifts /* [capacity,3] */,
                                  nqb_stream_t st);
/* A batch of independent frames in one exact list (the nvalchemiops batch_cell_list contract of
 * nequip/data/_nl.py:212-289): atoms of frame f are a contiguous range, batch [N] i64 is non-decreasing in [0, F).
 * nqb_nl_frames_pack fills out_host [F * nqb_nl_params_bytes()] on the HOST with one block per frame, from per-frame
 * arrays laid out as the by-value calls take them (cell / inv [F,9], pbc / nbins / search [F,3], lo / width [F,3]):
 * block f holds exactly what nqb_nl_bin, nqb_nl_count and nqb_nl_fill derive from frame f's arguments.  The caller
 * copies the blocks to the device.  bin_base [F+1] i64 (device) is the exclusive scan of the frames' bin counts: frame
 * f's bins are [bin_base[f], bin_base[f+1]) of one global range, so bin [N] holds global bin ids and order / bin_start
 * ([bin_base[F] + 1]) come from one sort and one searchsorted over all frames.  An atom only meets atoms of its own
 * frame.  types / rc2 / T as the _typed calls, or types and rc2 NULL for the r_max test.  Write contracts of
 * nqb_nl_bin, nqb_nl_count and nqb_nl_fill; each frame's rows are those of a single-frame list of that frame, with
 * atom indices global. */
int nqb_nl_frames_pack(int F, const double* cell_host, const double* inv_host, const int* pbc, const int* nbins,
                       const int* search, const double* lo, const double* width, double r_max, void* out_host);
int nqb_nl_bin_frames(const double* pos, int64_t N, const void* blocks_dev, const int64_t* batch,
                      const int64_t* bin_base, double* wpos /* [N,3] */, int32_t* base /* [N,3] */,
                      int64_t* bin /* [N] */, int32_t* cidx /* [N,3] */, nqb_stream_t st);
int nqb_nl_count_frames(int64_t N, const void* blocks_dev, const int64_t* batch, const int64_t* bin_base,
                        const double* wpos, const int32_t* cidx, const int64_t* order, const int64_t* bin_start,
                        const int64_t* types, const double* rc2, int T, int64_t* counts /* [N] */, nqb_stream_t st);
int nqb_nl_fill_frames(int64_t N, int64_t E, const void* blocks_dev, const int64_t* batch, const int64_t* bin_base,
                       const double* wpos, const int32_t* cidx, const int32_t* base, const int64_t* order,
                       const int64_t* bin_start, const int64_t* row_ptr /* [N+1] */, const int64_t* types,
                       const double* rc2, int T, int64_t* edge_index /* [2,E] */, double* shifts /* [E,3] */,
                       nqb_stream_t st);
/* A batch of frames in a list of fixed length (NeighborListPlan with batch=).  nqb_nl_frames_pack_capacity fills
 * out_host [F * nqb_nl_params_bytes()] on the HOST: block f is that of nqb_nl_frames_pack plus frame f's null-edge
 * shift pad_shift [F,3] and the open-direction fields of nqb_nl_params_pack_open (open[d] = !pbc[3f+d], cap [F] >= 1,
 * perp [F,3] finite and positive, r_max finite and > 0).
 * nqb_nl_bbox_frames (capturable, no work buffer) runs one CTA per frame over its atoms [atom_ptr[f], atom_ptr[f+1])
 * (atom_ptr [F+1] i64, device) and writes, in the DEVICE block f and nowhere else, lo / width / nb / search of each open
 * direction as nqb_nl_bbox does for one block; a frame without an open direction or without atoms is left as packed.
 * nqb_nl_fill_capacity_frames: nqb_nl_fill_capacity over frames (row_ptr_pad and overflow from nqb_nl_pad over all N
 * atoms, one capacity for the batch); the null edges of atom i carry the pad_shift of blocks[batch[i]].  Write contract
 * of nqb_nl_fill_capacity. */
int nqb_nl_frames_pack_capacity(int F, const double* cell_host, const double* inv_host, const int* pbc,
                                const int* nbins, const int* search, const double* lo, const double* width,
                                double r_max, const double* pad_shift_host, const int* cap, const double* perp_host,
                                void* out_host);
int nqb_nl_bbox_frames(const double* pos /* [N,3] */, int F, const int64_t* atom_ptr /* [F+1] */, void* blocks_dev,
                       nqb_stream_t st);
int nqb_nl_fill_capacity_frames(int64_t N, int64_t capacity, const void* blocks_dev, const int64_t* batch,
                                const int64_t* bin_base, const double* wpos, const int32_t* cidx, const int32_t* base,
                                const int64_t* order, const int64_t* bin_start, const int64_t* row_ptr_pad /* [N+1] */,
                                const int32_t* overflow /* [1] */, const int64_t* types, const double* rc2, int T,
                                int64_t* edge_index /* [2,capacity] */, double* shifts /* [capacity,3] */,
                                nqb_stream_t st);

/* Cells of a batched variable-cell plan packed on the device (NeighborListPlan.set_cell_device): thread f reads
 * cells[f] ([F,3,3] float64, device, rows = lattice vectors) and rewrites in blocks[f] (device, F * nqb_nl_params_bytes())
 * every field the host pack derives from the cell: cell, inverse (adjugate / determinant), diag and the orthorhombic
 * test, perp, the search range sr = max(1, ceil(r_max / (perp_d / nb_d) - 1e-12)) on the block's grid, and the
 * null-edge shift k e_d (d the first longest lattice vector, k = floor(r_max / |a_d|) + 2).  A non-finite cell or one
 * with |det| <= 1e-12 |a_0| |a_1| |a_2| keeps its block and sets bad[f] = 1 (bad [F] int32, never cleared here).
 * Writes those fields and bad, nothing else; no host synchronisation (capturable). */
int nqb_nl_frames_set_cells(int F, const double* cells, void* blocks_dev, int32_t* bad, nqb_stream_t st);

/* Molecular dynamics on the device (nqb_md.cu, nequip_b200/md.py GraphedMD): velocity Verlet with the reference's
 * Nose-Hoover thermostat (nequip/ase/nosehoover.py, NoseHoover.step) per frame f, all float64, in the reference's units
 * (Angstrom, eV, amu; time in Angstrom sqrt(amu / eV)).  The atoms of frame f are [atom_ptr[f], atom_ptr[f+1])
 * (atom_ptr [F+1] i64, device, non-decreasing).  The atom kernels run (nblk, F) CTAs of 256 threads; nblk in
 * [1, 65535] is the caller's choice and sizes the workspaces part [F, nblk, 2] and ke_part [F, nblk].  No floating-point
 * atomics: the sums over atoms are a fixed-order function of the inputs for a given nblk.  F <= 65535.
 * nqb_md_kick_drift: a = forces/mass - zeta[f] v;  pos += dt v + dt^2/2 a;  vel = v + dt/2 a;
 *   part[f, b] = {sum m v^2, sum m vel^2} over the atoms of CTA (b, f).  Writes pos and vel of every atom of the
 *   frames and all of part, nothing else.
 * nqb_md_bath (Nose-Hoover only): s0, s1 = sums of part[f, :, 0], part[f, :, 1] in index order;
 *   zeta_h = zeta + dt/2 * (s0 - gkT) / 2 / Q;  zeta' = zeta_h + dt/2 * (s1 - gkT) / 2 / Q;
 *   eta += dt/2 (zeta + zeta');  zeta = zeta'  (gkT = g_f k_B T_f with g_f = 3 N_f + 1, Q = nvt_q, both [F]).
 *   Writes zeta [F] and eta [F], nothing else.
 * nqb_md_kick: vel = (vel + dt/2 f_new/mass) / (1 + dt/2 zeta[f]);  forces = f_new;  ke_part[f, b] = sum m vel^2 of
 *   CTA (b, f).  Writes vel and forces of every atom of the frames and all of ke_part, nothing else.
 * nqb_md_log (one CTA): s = *step; row s % rows of log [rows, F, NQB_MD_LOG_FIELDS] gets, per frame,
 *   {E_pot = e_pot[f], E_kin = sum_b ke_part[f, b] / 2, T = 2 E_kin / dof_kB[f], zeta, eta,
 *    H = E_pot + E_kin + Q zeta^2 + gkT eta};  flags [4] i64 (sticky over the steps since the caller reset them to
 *   {0, 0, -1, 0}): flags[0] |= overflow != 0, flags[1] |= sorted != 1, flags[2] = s at the first overflow,
 *   flags[3] = max(flags[3], num_edges); then *step = s + 1.  Writes that log row, flags and step, nothing else. */
#define NQB_MD_LOG_FIELDS 6
int nqb_md_kick_drift(int F, int nblk, const int64_t* atom_ptr, const double* mass /* [N] */,
                      const double* forces /* [N,3] */, const double* zeta /* [F] */, double dt, double* pos /* [N,3] */,
                      double* vel /* [N,3] */, double* part /* [F,nblk,2] */, nqb_stream_t st);
int nqb_md_bath(int F, int nblk, const double* part, const double* gkT, const double* Q, double dt, double* zeta,
                double* eta, nqb_stream_t st);
int nqb_md_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new /* [N,3] */,
                const double* zeta, double dt, double* vel, double* forces, double* ke_part /* [F,nblk] */,
                nqb_stream_t st);
int nqb_md_log(int F, int nblk, const double* e_pot /* [F] */, const double* ke_part, const double* zeta,
               const double* eta, const double* Q, const double* gkT, const double* dof_kB, const int64_t* num_edges,
               const int32_t* overflow, const int32_t* sorted, int64_t rows, int64_t* step, double* log,
               int64_t* flags /* [4] */, nqb_stream_t st);

/* Structure relaxation on the device (nqb_relax.cu, nequip_b200/relax.py GraphedRelax): ASE's FIRE.step per frame f,
 * optionally on the degrees of freedom of ASE's FrechetCellFilter (has_cell), all float64.  Atoms and CTAs as in the
 * nqb_md kernels ((nblk, F) CTAs of 256 threads, nblk in [1, 65535], F <= 65535, no floating-point atomics).
 * Per-frame state: fs [F,2] {dt, a}; is [F, NQB_RELAX_ISTATE] i64 {Nsteps, first, converged, failed, steps};
 * a frame with converged or failed set is frozen.  Cell DOF (has_cell, all [F,9] row-major): Q = c log Fd, its
 * velocity vcell and force gcell, Fd = exp(Q / c), the initial cell C0 and cell = C0 Fd^T; cfac [F] = c.
 * nqb_relax_fire (one thread per frame): fire_host [7] = {maxstep, dtmax, finc, fdec, astart, fa, Nmin} on the HOST.
 *   For an active frame, with vg, vv, gg = v.g, v.v, g.g over the frame's whole vector (part [F,nblk,4] in index
 *   order, then the cell rows): first step v = 0; else v.g > 0 mixes v = (1-a) v + a |v| g / |g| (and dt, a grow
 *   after Nmin steps, Nsteps += 1), v.g <= 0 resets v = 0, a = astart, dt *= fdec, Nsteps = 0; then v += dt g,
 *   dr = dt v clipped to |dr| <= maxstep.  coef [F,4] = {cv, cg, sc, 1} so that v' = cv v + cg g, dr = sc v';
 *   steps += 1; with has_cell it also moves vcell, Q, Fd and cell.  A frozen frame gets coef {1, 0, 0, 0} only.
 *   Writes coef, fs, is and (has_cell) vcell, Q, Fd, cell of active frames, nothing else.
 * nqb_relax_move: the atoms of active frames: vel = cv vel + cg g; s += sc vel; pos = s Fd^T (has_cell; without a
 *   cell, s is not read and pos += sc vel).  Writes vel, s and pos of those atoms, nothing else.
 * nqb_relax_gforce: g = forces Fd (has_cell) or forces; part[f, b] = {sum v.g, sum v.v, sum g.g, max |g_i|^2} of CTA
 *   (b, f), a non-finite row counting +inf.  Writes g of every atom and all of part, nothing else.
 * nqb_relax_finish (one CTA): per frame, with V = |det cell|: (has_cell) gcell = (1/c) D exp(L^T)[(virial - p V I)
 *   Fd^-T], L = Q / c; m = the largest |g_i|^2 over part and the cell rows; a frame not frozen becomes failed if not
 *   m <= fail_force^2, else converged if m < fmax^2; log row step % rows [rows, F, NQB_RELAX_LOG_FIELDS] =
 *   {e_pot, e_pot + p V, sqrt(m), V}; flags [4] as in nqb_md_log; step += 1.  Writes gcell (has_cell), the
 *   converged / failed words of is, that log row, flags and step, nothing else. */
#define NQB_RELAX_ISTATE 5
#define NQB_RELAX_LOG_FIELDS 4
int nqb_relax_fire(int F, int nblk, const double* part, const double* fire_host, int has_cell, const double* cfac,
                   const double* C0, const double* gcell, double* Q, double* vcell, double* Fd, double* cell,
                   double* fs, int64_t* is, double* coef, nqb_stream_t st);
int nqb_relax_move(int F, int nblk, const int64_t* atom_ptr, const double* coef, int has_cell, const double* Fd,
                   const double* g, double* vel, double* s, double* pos, nqb_stream_t st);
int nqb_relax_gforce(int F, int nblk, const int64_t* atom_ptr, int has_cell, const double* Fd, const double* forces,
                     const double* vel, double* g, double* part, nqb_stream_t st);
int nqb_relax_finish(int F, int nblk, const double* part, int has_cell, double pressure, const double* cfac,
                     const double* Q, const double* Fd, const double* cell, const double* virial, const double* e_pot,
                     double fmax, double fail_force, double* gcell, int64_t* is, const int64_t* num_edges,
                     const int32_t* overflow, const int32_t* sorted, int64_t rows, int64_t* step, double* log,
                     int64_t* flags, nqb_stream_t st);

/* Constant-pressure MD on the device (nqb_npt.cu, nequip_b200/npt.py GraphedNPT): isotropic MTK with Nose-Hoover
 * chains on the particles (M = tchain members, tloop sub-steps) and on the barostat (Mp = pchain, ploop), in the
 * splitting of Tuckerman et al. (2006), per frame f, all float64, in the units of the nqb_md kernels.  Atoms and CTAs
 * as in the nqb_md kernels ((nblk, F) CTAs of 256 threads, nblk in [1, 65535], F <= 65535, no floating-point atomics).
 * M, Mp in [0, NQB_NPT_MAX_CHAIN] (0: no chain), tloop, ploop >= 1.
 * prm [F, NQB_NPT_PARAMS] = {kT, P, W, N_f, V0, N_f k_B, Q[NQB_NPT_MAX_CHAIN], Q'[NQB_NPT_MAX_CHAIN]} (alpha =
 *   1 + 3 / N_f).  state [F, NQB_NPT_STATE] = {eps, v_eps, K2 = sum m v^2, xi[8], v_xi[8], eta[8], v_eta[8]};
 *   vir [F,9] the model's virial at the state's positions; cell [F,9] = C0 e^eps; err [F] int32 sticky error flags;
 *   coef [F, NQB_NPT_COEF] = {s, e^{-alpha v_eps dt/2}, kick factor, e^{v_eps dt}, drift factor, active, final scale};
 *   work [F, NQB_NPT_STATE] a workspace.  NHC(h) is the chain half-step of DESIGN.md section 4.16.
 * nqb_npt_pre (one thread per frame): a frame with err set gets coef {1, 1, 0, 1, 0, 0, 1} only.  Otherwise
 *   NHC_baro(dt/2) on (v_eps, W); NHC_part(dt/2) on K2 (scale s); v_eps += dt/2 (alpha K2 + tr vir - 3 P V0 e^{3 eps}) / W;
 *   the coefficients; eps += dt v_eps; cell = C0 e^eps.  If any result is non-finite: err[f] = 1, coef as for err,
 *   state and cell unchanged.  Writes coef, work and, for a frame that passes, its state row and cell, nothing else.
 * nqb_npt_move: the atoms of active frames: v = s v; v = v e + kf forces/m; pos = pos e^{v_eps dt} + df v.  Writes pos
 *   and vel of those atoms, nothing else.
 * nqb_npt_kick: the atoms of active frames: vel = vel e + kf f_new/m; forces = f_new; part [F, nblk] = sum m vel^2 of
 *   CTA (b, f) (0 for an inactive frame).  Writes vel and forces of those atoms and all of part, nothing else.
 * nqb_npt_post (one thread per frame, frames with err set get coef[6] = 1 only): K2 = sum of part[f, :] in index
 *   order; v_eps += dt/2 G_eps / W with vir_new; NHC_part(dt/2) (scale coef[6]); NHC_baro(dt/2).  If any result is
 *   non-finite: err[f] = 1, coef[6] = 1, state and vir unchanged; else state row and vir = vir_new.  Writes coef[:, 6],
 *   work, err and those rows, nothing else.
 * nqb_npt_scale: the atoms of active frames: vel = coef[6] vel.  Writes those velocities, nothing else.
 * nqb_npt_log (one CTA): log row step % rows [rows, F, NQB_NPT_LOG_FIELDS] = {E_pot, K2/2, K2 / (N_f k_B), V,
 *   (K2 + tr vir) / (3 V), H} with H = E_pot + K2/2 + W v_eps^2/2 + P V + sum Q_k v_xi_k^2/2 + N_f kT xi_0
 *   + kT sum_{k>=1} xi_k + sum Q'_k v_eta_k^2/2 + kT sum eta_k; flags [4] as in nqb_md_log; step += 1.  Writes that
 *   log row, flags and step, nothing else. */
#define NQB_NPT_MAX_CHAIN 8
#define NQB_NPT_PARAMS 22
#define NQB_NPT_STATE 35
#define NQB_NPT_COEF 7
#define NQB_NPT_LOG_FIELDS 6
#define NQB_NPT_SINHC_TAYLOR 0.1
int nqb_npt_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* prm, const double* C0 /* [F,9] */,
                const double* vir, double* state, double* cell, double* coef, int32_t* err, double* work,
                nqb_stream_t st);
int nqb_npt_move(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* forces,
                 const double* coef, double* pos, double* vel, nqb_stream_t st);
int nqb_npt_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new,
                 const double* coef, double* vel, double* forces, double* part, nqb_stream_t st);
int nqb_npt_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt, const double* prm,
                 const double* part, const double* vir_new /* [F,9] */, double* state, double* vir, double* coef,
                 int32_t* err, double* work, nqb_stream_t st);
int nqb_npt_scale(int F, int nblk, const int64_t* atom_ptr, const double* coef, double* vel, nqb_stream_t st);
int nqb_npt_log(int F, int M, int Mp, const double* e_pot, const double* prm, const double* state, const double* vir,
                const int64_t* num_edges, const int32_t* overflow, const int32_t* sorted, int64_t rows, int64_t* step,
                double* log, int64_t* flags, nqb_stream_t st);

/* The fully flexible cell (nqb_npt.cu, GraphedNPT(barostat="flexible"), DESIGN.md section 4.17): fully flexible MTK
 * with a symmetric cell velocity v_g, chains, CTAs, err and the launch limits as above.  prm has the isotropic layout
 * with W = W_g = (N_f + 3) kT tau_P^2 / 3 and Q'_1 = 6 kT tau_P^2 (V0 unused).  state [F, NQB_NPTF_STATE] = {v_g[9],
 *   Kt[9] = sum m v (x) v, xi[8], v_xi[8], eta[8], v_eta[8]} (3x3 row-major, symmetric); cell [F,9] the cell (rows are
 *   lattice vectors); coef [F, NQB_NPTF_COEF] = {s, active, final scale, E_v[9], K[9], E_r[9], D[9]}; work [F,
 *   NQB_NPTF_STATE].  G_g = sym(Kt + vir) - P |det cell| I + (tr Kt / N_f) I; the barostat chain couples to W_g tr(v_g^2)
 *   with 6 degrees of freedom; v_g = O diag(lambda) O^T by NQB_NPTF_JACOBI_SWEEPS cyclic Jacobi sweeps, mu = lambda +
 *   tr(v_g) / N_f, E_v = O e^{-mu dt/2} O^T, K = O (dt/2) e^{-mu dt/4} sinhc(mu dt/4) O^T, E_r = O e^{lambda dt} O^T,
 *   D = O dt e^{lambda dt/2} sinhc(lambda dt/2) O^T.
 * nqb_nptf_pre (one thread per frame): a frame with err set gets coef {1, 0, 1, I, 0, I, 0} only.  Otherwise
 *   NHC_baro(dt/2) (v_g scaled); NHC_part(dt/2) (Kt *= s^2); v_g += dt/2 G_g / W_g with vir and the cell; E_v, K, E_r, D;
 *   cell = cell E_r.  If any result is non-finite: err[f] = 1, coef as for err, state and cell unchanged.  Writes coef,
 *   work and, for a frame that passes, its state row and cell, nothing else.
 * nqb_nptf_move: the atoms of active frames: v = s v; v = E_v v + K forces/m; pos = E_r pos + D v.  Writes pos and vel
 *   of those atoms, nothing else.
 * nqb_nptf_kick: the atoms of active frames: vel = E_v vel + K f_new/m; forces = f_new; part [F, nblk, 6] = sum m vel
 *   (x) vel of CTA (b, f) as {xx, yy, zz, yz, xz, xy} (0 for an inactive frame).  Writes vel and forces of those atoms
 *   and all of part, nothing else.
 * nqb_nptf_post (one thread per frame, frames with err set get coef[2] = 1 only): Kt = sum of part[f, :, :] in index
 *   order; v_g += dt/2 G_g / W_g with vir_new and the cell; NHC_part(dt/2) (scale coef[2], Kt *= s^2); NHC_baro(dt/2).
 *   If any result is non-finite: err[f] = 1, coef[2] = 1, state and vir unchanged; else state row and vir = vir_new.
 *   Writes coef[:, 2], work, err and those rows, nothing else.
 * nqb_nptf_scale: the atoms of active frames: vel = coef[2] vel.  Writes those velocities, nothing else.
 * nqb_nptf_log (one CTA): log row step % rows [rows, F, NQB_NPTF_LOG_FIELDS] = {E_pot, tr Kt/2, tr Kt / (N_f k_B), V,
 *   tr(P_int) / 3, H, cell[9], P_int[9]} with V = |det cell|, P_int = (Kt + vir) / V and H = E_pot + tr Kt/2
 *   + W_g tr(v_g^2)/2 + P V + sum Q_k v_xi_k^2/2 + N_f kT xi_0 + kT sum_{k>=1} xi_k + sum Q'_k v_eta_k^2/2 + 6 kT eta_0
 *   + kT sum_{k>=1} eta_k; flags [4] as in nqb_md_log; step += 1.  Writes that log row, flags and step, nothing else. */
#define NQB_NPTF_STATE 50
#define NQB_NPTF_COEF 39
#define NQB_NPTF_LOG_FIELDS 24
#define NQB_NPTF_JACOBI_SWEEPS 6
int nqb_nptf_pre(int F, int M, int Mp, int tloop, int ploop, double dt, const double* prm, const double* vir,
                 double* state, double* cell, double* coef, int32_t* err, double* work, nqb_stream_t st);
int nqb_nptf_move(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* forces,
                  const double* coef, double* pos, double* vel, nqb_stream_t st);
int nqb_nptf_kick(int F, int nblk, const int64_t* atom_ptr, const double* mass, const double* f_new,
                  const double* coef, double* vel, double* forces, double* part, nqb_stream_t st);
int nqb_nptf_post(int F, int nblk, int M, int Mp, int tloop, int ploop, double dt, const double* prm,
                  const double* part, const double* vir_new, const double* cell, double* state, double* vir,
                  double* coef, int32_t* err, double* work, nqb_stream_t st);
int nqb_nptf_scale(int F, int nblk, const int64_t* atom_ptr, const double* coef, double* vel, nqb_stream_t st);
int nqb_nptf_log(int F, int M, int Mp, const double* e_pot, const double* prm, const double* state, const double* vir,
                 const double* cell, const int64_t* num_edges, const int32_t* overflow, const int32_t* sorted,
                 int64_t rows, int64_t* step, double* log, int64_t* flags, nqb_stream_t st);

/* First radial layer (K = 8, CUDA cores):  h[E,128] = silu(emb[E,8] @ W1s[8,128])  and
 * grad_emb[E,8] = (grad_h * silu'(emb @ W1s)) @ W1s^T  (pre-activation recomputed, nothing saved).
 * Together with nqb_gemm_grouped for the second layer this is ScalarMLPFunction (nequip/nn/mlp.py:80-195).
 * h [E, hidden] and grad_emb [E, num_bessel] are fully written. */
int nqb_mlp_hidden_fwd(const float* emb, const float* W1s, int64_t E, int num_bessel, int hidden, float* h,
                       nqb_stream_t st);
int nqb_mlp_hidden_bwd(const float* emb, const float* W1s, const float* grad_h, int64_t E, int num_bessel,
                       int hidden, float* grad_emb, nqb_stream_t st);

/* Reverse-edge pair map of the radial MLP: the MLP's input is the edge embedding alone, so two edges whose embedding
 * rows are bitwise equal get bitwise-equal MLP outputs, and the rows can be computed once.
 *   edge_index [2,E] i64 (i = edge_index[0][e], j = edge_index[1][e]); shift [E,3] f64 or NULL (all zero);
 *   emb [E,num_bessel] f32; row_ptr [N+1] / perm [E] or NULL: the destination CSR of edge_index[0]
 *   (nqb_csr_from_sorted).
 *   The candidate of e = (i -> j) is the first edge f != e in CSR order of row j with edge_index[1][f] = i,
 *   shift[f] = -shift[e] (compared as values: -0 equals 0) and emb[f] bitwise equal to emb[e].  e and f are
 *   partners when each is the other's candidate; an edge without a partner has a slot of its own.
 *   pair_rows [E,2] i64 (16-byte aligned): slot u < U holds {representative edge, partner or -1}, the representative
 *   being the smaller edge id of a pair, slots ordered by representative.  count [1] i64 = U (left on the device).
 *   Writes pair_rows rows < U and count, nothing else (E = 0: count = 0 only).  No host synchronisation: the launches
 *   depend on E only, so they can be captured in a CUDA graph.
 *   work: nqb_edge_pairs_work_size(E) i64 of scratch. */
int64_t nqb_edge_pairs_work_size(int64_t E);
int nqb_edge_pairs(const int64_t* edge_index, int64_t E, int64_t N, const double* shift, const float* emb,
                   int num_bessel, const int64_t* row_ptr, const int64_t* perm, int64_t* work, int64_t* pair_rows,
                   int64_t* count, nqb_stream_t st);
/* The first radial layer on the slots of nqb_edge_pairs:  h[u] = silu(emb[pair_rows[u][0]] @ W1s)  for
 * u < min(*count, capacity).  Writes rows < U of h [capacity, hidden] only; the grid depends on capacity alone. */
int nqb_mlp_hidden_fwd_rows(const float* emb, const float* W1s, const int64_t* pair_rows, const int64_t* count,
                            int64_t capacity, int num_bessel, int hidden, float* h, nqb_stream_t st);
/* Its backward on the same slots: for u < U = min(*count, capacity), with p = emb[pair_rows[u][0]] @ W1s,
 *   grad_emb[pair_rows[u][0]] = (grad_h[u] * silu'(p)) @ W1s^T  and  grad_emb[pair_rows[u][1]] = 0 (when >= 0).
 * grad_h [capacity, hidden] is read in rows < U (the slot's gradient, summed over both edges).  Writes exactly the
 * grad_emb rows named in pair_rows[0 .. U): every row when the map covers all E edges.  pair_rows must be 16-byte
 * aligned; the grid depends on capacity alone. */
int nqb_mlp_hidden_bwd_rows(const float* emb, const float* W1s, const float* grad_h, const int64_t* pair_rows,
                            const int64_t* count, int64_t capacity, int num_bessel, int hidden, float* grad_emb,
                            nqb_stream_t st);

/* Grouped fp32-accurate GEMM on the tensor cores (wgmma tf32, 3xTF32, segmented fp32
 * accumulation):  C_p[M, N_p] (+)= rowscale_p[m] * A_p[M, K_p] @ B_p[K_p, N_p]  for a list of problems
 * sharing M.  Replaces the dense algebra around the convolution: ScalarMLPFunction's torch.mm
 * (nequip/nn/mlp.py:262-268), e3nn o3.Linear linear_1/linear_2 and the self-connection
 * FullyConnectedTensorProduct (nequip/nn/interaction_block.py:82-87,129-146) in the ir_mul layout.
 * descs_dev: device array of ndesc records of 12 int64:
 *   {a_off, c_off, b_off, rs_off (row of the [R, rs_ld] row-scale matrix, -1 = none), lda, ldc, K, N, kchunks=ceil(K/32), ntiles=ceil(N/128),
 *    tile0 (prefix sum of ntiles), flags};  offsets in floats from the bases.
 *   flags: none: C is fully written (rows < M, columns < N_p); bit0 C is ACCUMULATED INTO (one writer per element
 *   within the launch); bit1 rows whose row scale is 0 are left untouched (disjoint row-masked writers); bit2 C is
 *   ACCUMULATED INTO with red.global.add (several problems add into the same C).  Nothing outside rows < M,
 *   columns [c_off + m * ldc, + N_p) is written; A is read in rows < M, columns < K_p only.  M = 0 writes nothing.
 * Requirements: K, N, lda, ldc, a_off, c_off multiples of 4; a_base, prepared_base, c_base 16-byte aligned
 * (checked: an error, no launch).
 * B_p is prepared once (split hi/lo, tiled) with nqb_gemm_prepare into nqb_gemm_prepared_floats(K,N) floats
 * (fully written).
 * tile_ctas_dev (nullable): int32 {first CTA, CTAs} per N-tile -- a cost-weighted split of sched_ctas CTAs over
 * the N-tiles computed by the host (problems of one launch differ in K, N and store mode); used when
 * sched_ctas <= #SMs, otherwise the even split is used. */
int64_t nqb_gemm_prepared_floats(int K, int N);
int nqb_gemm_prepare(const float* B, int64_t ldb, int K, int N, int transposed, float scale, float* prepared,
                     nqb_stream_t st);
int nqb_gemm_grouped(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                     int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                     const float* rowscale_base, int64_t rs_ld, int64_t M, nqb_stream_t st);
/* The same GEMM with an activation epilogue (the radial MLP's hidden layers, SiLU).  With v the finished value
 * (after the row scale), three more flag bits apply per problem:
 *   bit3  C = silu(v) instead of v;
 *   bit4  also aux = v (the pre-activation);
 *   bit5  C = v * silu'(aux)  with  silu'(p) = s(p) (1 + p (1 - s(p))),  s = sigmoid  (the gradient through the
 *         activation whose pre-activation was saved with bit4).
 * aux is addressed like C: element (m, n) of problem p is aux_base[c_off + m * ldc + n].  Bits 3-5 are never
 * combined with bit0 or bit2 (the host rejects it).  Problems without bits 3-5 behave as in nqb_gemm_grouped.
 * Write contract: with bit3 or bit4, C (and with bit4 aux) is fully written in rows < M, columns < N_p, and nothing
 * else of C or aux is written; with bit5, aux is read in rows < M, columns < N_p only, and C is fully written there.
 * aux_base must be non-null and 16-byte aligned (checked: an error, no launch; the entry point cannot see the
 * device descriptors, so it requires aux even when only bit3 is used, in which case aux is never touched and
 * c_base may be passed). */
int nqb_gemm_grouped_act(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                         int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                         const float* rowscale_base, int64_t rs_ld, int64_t M, float* aux_base, nqb_stream_t st);
/* The same GEMM on the slots of nqb_edge_pairs (plain problems only: no row scale, no flag bits; the host rejects
 * others).  M = min(*count_dev, capacity) is read on the device, A holds one row per slot (the compact h), and result
 * row m is stored to C rows pair_rows[m][0] and, when it is >= 0, pair_rows[m][1].  Write contract: every C row listed
 * in pair_rows[0 .. M) is written once in columns < N_p, nothing else of C is written; A is read in rows < M only.
 * pair_rows must be 16-byte aligned; the grid depends on capacity alone (capturable). */
int nqb_gemm_grouped_pairs(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                           int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                           const int64_t* pair_rows, const int64_t* count_dev, int64_t capacity, nqb_stream_t st);
/* The transpose direction on the same slots (plain problems only): M = min(*count_dev, capacity) is read on the
 * device and row m of the product is (A[pair_rows[m][0]] + A[pair_rows[m][1]]) @ B, the second row only when
 * pair_rows[m][1] >= 0 (the fp32 sum is formed in the kernel), stored to C row m.  Write contract: C rows < M, columns
 * < N_p are written, nothing else; A is read in the rows listed in pair_rows[0 .. M), columns < K_p only.
 * pair_rows must be 16-byte aligned and capacity < 2^31; the grid depends on capacity alone (capturable). */
int nqb_gemm_grouped_pair_sum(const void* descs_dev, int ndesc, int ntiles_total, const int32_t* tile_ctas_dev,
                              int sched_ctas, const float* a_base, const float* prepared_base, float* c_base,
                              const int64_t* pair_rows, const int64_t* count_dev, int64_t capacity, nqb_stream_t st);

/* Gate nonlinearity (e3nn nn.Gate with normalize2mom'd SiLU for even / tanh for odd scalars and gates,
 * nequip/nn/convnetlayer.py:42-56,104-112), one kernel per direction.  Column tables (device, int32) are
 * built by the host from the irreps, for either layout:
 *   forward, per OUTPUT column j: src[j], gate[j] (-1: scalar), kind[j] (0 silu, 1 tanh):
 *     out[n,j] = gate[j] < 0 ? act(x[n,src[j]]) : x[n,src[j]] * act(x[n,gate[j]])
 *   backward, per INPUT column i: tab[6*i..] = {role, a, b, c, d, kind}
 *     role 0 scalar (a = output column); role 1 gated value (a = output column, b = gate input column);
 *     role 2 gate (a = first output column, b = first gated input column, c = component stride, d = 2l+1).
 * out [N, d_out] and grad_x [N, d_in] are fully written. */
int nqb_gate_fwd(int dtype, const void* x, int64_t N, int d_in, int d_out, const int32_t* src,
                 const int32_t* gate, const int32_t* kind, void* out, nqb_stream_t st);
int nqb_gate_bwd(int dtype, const void* x, const void* grad_out, int64_t N, int d_in, int d_out,
                 const int32_t* tab, void* grad_x, nqb_stream_t st);

/* number of kernels the library has launched in this process (bench accounting) */
int64_t nqb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* NQB_H */
