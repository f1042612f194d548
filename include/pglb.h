/*
 * pglb.h -- C-ABI of libpglb.so: the H100 (sm_90a) send/recv message-passing path
 * behind PGL's Graph.send/recv API.
 *
 * The reference (PaddlePaddle/PGL @ 6dbb47c) has no native boundary of its own on this
 * path: it is Python over Paddle's operator API plus one Cython module.  Every entry point
 * below therefore names the reference call site(s) it replaces (paths relative to the
 * reference root).  See INTEGRATION.md for the reference-side binding.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes; no torch / CUDA C++ types.  `stream` is a
 *    cudaStream_t passed as void* (NULL = legacy default stream).
 *  - All device entry points are asynchronous on `stream`, re-entrant and thread-safe; the
 *    library never allocates or frees device memory and keeps no pointer past the call.
 *    Scratch space is caller-owned: query with the matching *_ws() and pass (ws, ws_bytes).
 *  - Index tensors are int64 (PGL mandates int64 edges: pgl/graph.py:130-135), features
 *    are float32 row-major with an explicit leading dimension where noted.
 *  - Return value: 0 = PGLB_OK; <0 = argument error (no device work was enqueued);
 *    >= PGLB_CUDA_ERR_BASE = PGLB_CUDA_ERR_BASE + cudaError_t.  pglb_last_error() returns a
 *    thread-local, human-readable description of the last non-zero return.
 *  - No C++ exception crosses this boundary.
 */
#ifndef PGLB_H_
#define PGLB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PGLB_VERSION 100 /* 0.1.0 */

#define PGLB_OK 0
#define PGLB_EINVAL (-1)    /* null pointer / negative size / unknown enum */
#define PGLB_ESHAPE (-2)    /* inconsistent sizes */
#define PGLB_EWORKSPACE (-3) /* workspace too small or misaligned */
#define PGLB_EUNSUPPORTED (-4)
#define PGLB_ENOLIB (-5)    /* optional host dependency (METIS) not loadable */
#define PGLB_CUDA_ERR_BASE 1000

/* reduce_op of send_u_recv / send_ue_recv / segment_* (pgl/graph.py:856-857, pgl/math.py:34-46) */
#define PGLB_REDUCE_SUM 0
#define PGLB_REDUCE_MEAN 1
#define PGLB_REDUCE_MAX 2
#define PGLB_REDUCE_MIN 3

/* message_op of send_ue_recv / send_uv (pgl/graph.py:923-927,958-962); COPY = no edge operand */
#define PGLB_MSG_COPY 0
#define PGLB_MSG_ADD 1
#define PGLB_MSG_SUB 2
#define PGLB_MSG_MUL 3
#define PGLB_MSG_DIV 4

/* how the second operand's row broadcasts against the D = H*Dh output columns */
#define PGLB_BCAST_FULL 0   /* y row has D values                      */
#define PGLB_BCAST_HEAD 1   /* y row has H values, y[c / Dh]  ([E,H,1] against [N,H,Dh]) */
#define PGLB_BCAST_SCALAR 2 /* y row has 1 value   ([E] or [E,1])       */

int pglb_version(void);
const char *pglb_last_error(void);
/* number of kernels this library has launched in the calling process (bench "gpu_launches") */
int64_t pglb_launch_count(void);

/* ------------------------------------------------------------------------------------
 * CSR build on the device.  Replaces EdgeIndex.from_edges (pgl/utils/edge_index.py:38-58;
 * tensor branch :43-54 = scatter-count + argsort + 2 gathers + cumsum) and is bit-identical
 * to the numpy branch's graph_kernel.build_index (pgl/graph_kernel.pyx:59-88): stable, i.e.
 * ascending edge id inside every bucket.
 *   u, v         : int64 device pointers, element i at u[i*u_stride] (so edges[:,1] of an
 *                  [E,2] array is (edges+1, stride 2) -- no strided copies as in
 *                  pgl/graph.py:859)
 *   degree[N], indptr[N+1], sorted_u[E], sorted_v[E], sorted_eid[E] : int64 outputs
 * ---------------------------------------------------------------------------------- */
int pglb_csr_build_ws(int64_t num_edges, int64_t num_nodes, size_t *ws_bytes);
int pglb_csr_build(const int64_t *u, int64_t u_stride, const int64_t *v, int64_t v_stride,
                   int64_t num_edges, int64_t num_nodes, int64_t *degree, int64_t *indptr,
                   int64_t *sorted_u, int64_t *sorted_v, int64_t *sorted_eid, void *ws,
                   size_t ws_bytes, void *stream);

/* Host twin of the above for numpy-mode graphs (EdgeIndex numpy branch,
 * pgl/utils/edge_index.py:56-57 -> pgl/graph_kernel.pyx:59-88).  Blocking, host pointers. */
int pglb_build_index_host(const int64_t *u, int64_t u_stride, const int64_t *v,
                          int64_t v_stride, int64_t num_edges, int64_t num_nodes,
                          int64_t *degree, int64_t *indptr, int64_t *sorted_u,
                          int64_t *sorted_v, int64_t *sorted_eid);

/* segment ids of a CSR: replaces Graph.get_segment_ids -> unique_segment
 * (pgl/graph.py:1397-1407, pgl/utils/helper.py:156-160; paddle.unique(return_inverse)).
 *   uniq_ind[K]   = rows with degree > 0 (ascending), segment_ids[E] = dense id per slot.
 *   num_uniq      : device int64 scalar that receives K.
 *   ws >= pglb_segment_ids_ws bytes. */
int pglb_segment_ids_ws(int64_t num_nodes, size_t *ws_bytes);
int pglb_segment_ids(const int64_t *indptr, int64_t num_nodes, int64_t num_edges,
                     int64_t *uniq_ind, int64_t *segment_ids, int64_t *num_uniq, void *ws,
                     size_t ws_bytes, void *stream);

/* sorted segment ids [E] -> indptr[K+1] (used by segment_* below; K = ids[E-1]+1, caller-known) */
int pglb_segment_indptr(const int64_t *segment_ids, int64_t num_edges, int64_t num_segments,
                        int64_t *indptr, void *stream);

/* ------------------------------------------------------------------------------------
 * Node-parallel CSR aggregation  out[d] = reduce_{slot j in row d} msg(j)   (K1/K2/K4)
 *   msg(j) = x[cols[j]]                       (msg_op = COPY)
 *          = x[cols[j]] (op) y[eid[j]]        (ADD/SUB/MUL/DIV, y broadcast per y_bcast)
 * Replaces paddle.geometric.send_u_recv / send_ue_recv as called at pgl/graph.py:860,886,
 * 930 (COO + atomics in the reference; here a cached dst-CSR, one writer per row,
 * summation in ascending edge id = the reference CPU loop's order), the legacy
 * helper.graph_send_recv (pgl/utils/helper.py:163-210) and, with cols == NULL (slot j
 * reads row j), paddle.geometric.segment_{sum,mean,max,min} (pgl/math.py:36-42).
 *   indptr[n_dst+1], cols[E] (nullable), eid[E] (nullable: y indexed by slot)
 *   x  [n_src, ldx] (first D columns used), y per y_bcast (nullable iff COPY), row stride ldy
 *   out[n_dst, ldo]; rows without a message are 0 for every reduce_op; MEAN divides by the
 *   row's slot count.
 *   scale_src[n_src] / scale_dst[n_dst] (nullable): msg *= scale_src[cols[j]] before the
 *   reduce, out[d] *= scale_dst[d] after it (GCNConv's two norm multiplies, conv.py:242,250)
 *   D = H * Dh output columns; head_dim = Dh (only used by PGLB_BCAST_HEAD).
 *   cols_packed[E] (nullable, uint32): a packed copy of cols made by pglb_pack_cols() (needs
 *   n_src < 2^31).  Halves the index traffic of the wide-row kernel; with PGLB_SPMM_L2_HINTS in
 *   flags, bit 31 marks sources worth keeping in L2 (evict_last, all other rows evict_first).
 *   Pure performance hints: results do not depend on them.
 *   max_degree_hint : max row length if the caller knows it (skips the hub pass when
 *   small), or -1.
 * ---------------------------------------------------------------------------------- */
int pglb_spmm_csr_ws(int64_t n_dst, int64_t num_edges, int64_t D, size_t *ws_bytes);
int pglb_spmm_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                      const float *x, int64_t ldx, const float *y, int64_t ldy, int y_bcast,
                      float *out, int64_t ldo, int64_t n_dst, int64_t n_src,
                      int64_t num_edges, int64_t D, int64_t head_dim, int msg_op,
                      int reduce_op, const float *scale_src, const float *scale_dst,
                      const uint32_t *cols_packed, int64_t max_degree_hint, int flags, void *ws,
                      size_t ws_bytes, void *stream);
/* pglb_spmm_csr_f32 plus scale_slot[E] (nullable, wins over scale_src): the source scale already laid out per CSR
 * slot (scale_slot[j] = scale_src[cols[j]]), streamed by the wide-row kernel instead of gathered, which would cost a
 * 32-byte sector per edge.  The kernels that do not stream it gather scale_src, so scale_slot needs scale_src
 * (PGLB_EINVAL otherwise).  pglb_spmm_csr_f32 is this call with scale_slot = NULL.  Same results either way. */
int pglb_spmm_csr_slot_scale_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid,
                                 const float *x, int64_t ldx, const float *y, int64_t ldy, int y_bcast,
                                 float *out, int64_t ldo, int64_t n_dst, int64_t n_src,
                                 int64_t num_edges, int64_t D, int64_t head_dim, int msg_op,
                                 int reduce_op, const float *scale_src, const float *scale_slot,
                                 const float *scale_dst, const uint32_t *cols_packed, int64_t max_degree_hint,
                                 int flags, void *ws, size_t ws_bytes, void *stream);
/* flags of pglb_spmm_csr_f32 */
#define PGLB_SPMM_ACCUMULATE 1 /* SUM only: out[d] = (out[d] + sum of messages) * scale_dst[d];
                                  lets a caller aggregate one edge subset while the feature rows of
                                  another subset (halo rows) are still in flight */
#define PGLB_SPMM_L2_HINTS 2   /* bit 31 of cols_packed carries an L2 residency hint */

/* 16-bit feature types of pglb_spmm_csr_x16 and the other *_x16 entries */
#define PGLB_DTYPE_BF16 1
#define PGLB_DTYPE_F16 2
/* Copy-message aggregation over 16-bit features: pglb_spmm_csr_slot_scale_f32 with msg_op = COPY (send_u_recv with
 * every reduce_op; cols == NULL = identity slots, i.e. segment_*), where x and out are bfloat16 or float16 (`dtype`)
 * and ldx / ldo count elements.  Numerics: every message is widened to fp32 exactly and reduced in fp32 in the same
 * slot order and with the same operations as the fp32 entry; mean, scale_src / scale_slot / scale_dst (float32) and
 * cut-row / hub partials (float32, in the workspace) stay fp32; each output element is rounded once, to nearest even.
 * So every output equals round16(the fp32 entry's output on the widened x) whenever both take the same kernel: the
 * wide-row kernel for copy sum / mean with 64 < D <= 128, D % 8 == 0, 16-byte aligned x and out and ldx, ldo % 8 == 0;
 * the node-parallel kernel otherwise.
 * ws: pglb_spmm_csr_ws(n_dst, E, D).  flags: PGLB_SPMM_L2_HINTS as above; PGLB_SPMM_ACCUMULATE is PGLB_EUNSUPPORTED
 * (it would round twice).  Unknown dtype: PGLB_EINVAL.  All argument checks precede any CUDA call. */
int pglb_spmm_csr_x16(const int64_t *indptr, const int64_t *cols, const void *x, int64_t ldx, void *out, int64_t ldo,
                      int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, int dtype, int reduce_op,
                      const float *scale_src, const float *scale_slot, const float *scale_dst,
                      const uint32_t *cols_packed, int64_t max_degree_hint, int flags, void *ws, size_t ws_bytes,
                      void *stream);

/* Send/recv with an edge operand over 16-bit features: pglb_spmm_csr_f32's arguments plus `dtype`, x and out bfloat16
 * or float16 (ldx / ldo in elements), y float32.  Instantiated for msg_op MUL / ADD, reduce_op SUM and y_bcast
 * PGLB_BCAST_HEAD / PGLB_BCAST_SCALAR over rows of D % 4 == 0 elements (8-byte aligned x and out, ldx, ldo % 4 == 0):
 * the gradient of the fused GAT aggregation wrt f, sum over the out-edges of alpha * grad_out[dst].  Any other msg_op,
 * reduce_op or broadcast, D % 4 != 0 and PGLB_SPMM_ACCUMULATE are PGLB_EUNSUPPORTED; misaligned rows PGLB_ESHAPE.
 * Numerics: each message x (op) y is formed and summed in fp32, in slot order, with the fp32 node-parallel kernel's
 * operations; hub partials are fp32; each output is rounded once, to nearest even.  Deterministic.  Rows of up to 1024
 * slots are summed sequentially.  cols_packed is not taken.  Unknown dtype: PGLB_EINVAL.  All argument checks precede
 * any CUDA call.  ws: pglb_spmm_csr_ws(n_dst, E, D). */
int pglb_spmm_csr_ue_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *x, int64_t ldx,
                         const float *y, int64_t ldy, int y_bcast, void *out, int64_t ldo, int64_t n_dst,
                         int64_t n_src, int64_t num_edges, int64_t D, int64_t head_dim, int dtype, int msg_op,
                         int reduce_op, const float *scale_src, const float *scale_dst, int64_t max_degree_hint,
                         int flags, void *ws, size_t ws_bytes, void *stream);

/* Packed column ids for pglb_spmm_csr_f32: count[n_src] (int32, zeroed by the call) receives how
 * often every source occurs in cols[E]; packed[j] = cols[j] | (count[cols[j]] >= min_count) << 31.
 * Pass min_count = INT64_MAX for plain 32-bit ids without hints. */
int pglb_pack_cols(const int64_t *cols, int64_t num_edges, int64_t n_src, int32_t *count,
                   int64_t min_count, uint32_t *packed, void *stream);

/* Narrow-row copy aggregation (sum / mean, D = 4..64 floats, D % 4 == 0): the same send_u_recv
 * (pgl/graph.py:860,886) for the 16..256-byte rows of a COLUMN-sharded feature matrix (every GPU holds the whole
 * CSR and D/R columns; reference precedent for the layout: examples/.../dist_feat.py:31-49).
 * pglb_narrow_plan builds, once per graph, what the kernel streams instead of cols/indptr:
 *   plan[E]        uint32: cols[j] | (slot j is the first of its row) << 30   (needs n_src < 2^30)
 *   nz_row[n_dst+2] int32: ids of the non-empty rows in order, padded with two copies of the last one
 *   blk_k[ceil(E/32)] int32: index into nz_row of the row that owns slot 32 b - 1 (-1 for b = 0)
 * ws: pglb_narrow_plan_ws(n_dst) / pglb_spmm_narrow_ws(E, D).  x and out rows 16-byte aligned (ldx, ldo % 4 == 0).
 * Row sums are formed in slot order inside 32-slot ranges and the ranges of a row added left to right:
 * deterministic, equal to the sequential loop up to fp32 rounding of the regrouping. */
int pglb_narrow_plan_ws(int64_t n_dst, size_t *ws_bytes);
/* cols_packed (nullable): the uint32 ids of pglb_pack_cols; its bit 31 (L2 residency hint) is carried into the plan */
int pglb_narrow_plan(const int64_t *indptr, const int64_t *cols, const uint32_t *cols_packed, int64_t n_dst,
                     int64_t n_src, int64_t num_edges, uint32_t *plan, int32_t *nz_row, int32_t *blk_k, void *ws,
                     size_t ws_bytes, void *stream);
int pglb_spmm_narrow_ws(int64_t num_edges, int64_t D, size_t *ws_bytes);
/* scale_src[n_src] (nullable): gathered per slot.  scale_slot[E] (nullable, wins over scale_src): the same values
 * already laid out per CSR slot (scale_slot[j] = scale_src[cols[j]], i.e. the edge values of the normalised adjacency),
 * streamed with the plan instead of gathered.  flags: PGLB_SPMM_L2_HINTS = honour bit 31 of the plan. */
int pglb_spmm_narrow_f32(const uint32_t *plan, const int32_t *nz_row, const int32_t *blk_k, const int64_t *indptr,
                         const float *x, int64_t ldx, float *out, int64_t ldo, int64_t n_dst, int64_t n_src,
                         int64_t num_edges, int64_t D, int reduce_op, const float *scale_src, const float *scale_slot,
                         const float *scale_dst, int flags, void *ws, size_t ws_bytes, void *stream);

/* One K-hop propagation step (APPNP, GCNII, SSGCConv, GPRConv; ChebNetII / BernNet recurrences) as one aggregation
 * with a row epilogue.  For every destination row d, with t[d] the row pglb_spmm_csr_slot_scale_f32 (copy message,
 * reduce SUM, the same scales) writes -- same route, slot order, hub / cut-row merging, and the same t for rows
 * without a slot:
 *   y[d]       = h ? a*t[d] + b*h[d] : a*t[d]
 *   out[d]     = y[d]
 *   acc_out[d] = acc_in[d] + cc*y[d]          (when acc_out is given; cc = c_dev ? *c_dev : c)
 * each product and sum rounded on its own (no FMA contraction): with a = (float)(1 - alpha), b = (float)alpha, h = h0
 * it is bit for bit torch's `alpha * h0 + (1 - alpha) * propagate(x)`.  c_dev (nullable, device float) lets a caller
 * take c from a device tensor without a host sync.  Arguments: pglb_spmm_csr_slot_scale_f32's without eid, y, ldy,
 * y_bcast, head_dim, msg_op and reduce_op, plus
 *   h [n_dst, ldh] (nullable; may be x itself), acc_in [n_dst, ld_acc_in] and acc_out [n_dst, ld_acc_out] (both or
 *   neither; acc_out == acc_in with the same stride updates in place).
 * ws: pglb_spmm_csr_ws(n_dst, E, D).  flags: PGLB_SPMM_L2_HINTS as above.  Refused before any CUDA call:
 *   PGLB_EINVAL   acc_out without acc_in (or the reverse); out overlapping x, h, acc_in or acc_out; acc_out
 *                 overlapping x, h, or acc_in other than as the same pointer and stride; scale_slot without scale_src
 *   PGLB_ESHAPE   ldh, ld_acc_in or ld_acc_out < D
 *   PGLB_EUNSUPPORTED  PGLB_SPMM_ACCUMULATE; a wide-row shape the copy-sum entry would send to spmm_stream (it has no
 *                 epilogue); h / acc rows that are not 16-byte aligned where x and out are (the vector kernels). */
int pglb_propagate_f32(const int64_t *indptr, const int64_t *cols, const float *x, int64_t ldx, float *out, int64_t ldo,
                       int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t D, const float *scale_src,
                       const float *scale_slot, const float *scale_dst, float a, float b, const float *h, int64_t ldh,
                       const float *acc_in, int64_t ld_acc_in, float *acc_out, int64_t ld_acc_out, float c,
                       const float *c_dev, const uint32_t *cols_packed, int64_t max_degree_hint, int flags, void *ws,
                       size_t ws_bytes, void *stream);
/* The same step over pglb_spmm_narrow_f32's plan (reduce SUM): its argument checks, then pglb_propagate_f32's on the
 * epilogue operands; h / acc rows must be 16-byte aligned (PGLB_EUNSUPPORTED).  t[d] is the row pglb_spmm_narrow_f32
 * writes.  ws: pglb_spmm_narrow_ws(E, D). */
int pglb_propagate_narrow_f32(const uint32_t *plan, const int32_t *nz_row, const int32_t *blk_k, const int64_t *indptr,
                              const float *x, int64_t ldx, float *out, int64_t ldo, int64_t n_dst, int64_t n_src,
                              int64_t num_edges, int64_t D, const float *scale_src, const float *scale_slot,
                              const float *scale_dst, float a, float b, const float *h, int64_t ldh,
                              const float *acc_in, int64_t ld_acc_in, float *acc_out, int64_t ld_acc_out, float c,
                              const float *c_dev, int flags, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Edge-parallel ops
 * ---------------------------------------------------------------------------------- */
/* out[e] = x[src[e]] (op) y[dst[e]] ; replaces paddle.geometric.send_uv (pgl/graph.py:965).
 * src/dst strided like pglb_csr_build.  x [n_src, D], y [n_dst, D], out [E, D]. */
int pglb_send_uv_f32(const float *x, const float *y, const int64_t *src, int64_t src_stride,
                     const int64_t *dst, int64_t dst_stride, int64_t num_edges, int64_t D,
                     int msg_op, float *out, void *stream);

/* out[i] = x[index[i]] ; paddle.gather(axis=0) at pgl/utils/op.py:45, pgl/message.py:157,
 * pgl/math.py:219,223.  index strided. */
int pglb_gather_rows_f32(const float *x, int64_t ldx, const int64_t *index,
                         int64_t index_stride, int64_t num_rows, int64_t D, float *out,
                         int64_t ldo, void *stream);
/* out[index[i]] = x[i] (unique indices) ; paddle.scatter(overwrite=True) at
 * pgl/graph.py:830, pgl/nn/functional/graph_op.py:122. */
int pglb_scatter_rows_f32(const float *x, int64_t ldx, const int64_t *index,
                          int64_t num_rows, int64_t D, float *out, int64_t ldo,
                          void *stream);

/* Per-row softmax over CSR rows, H columns; replaces pgl.math.segment_softmax
 * (pgl/math.py:216-224: 7 ops) and, with eid != NULL, GF.edge_softmax
 * (pgl/nn/functional/graph_op.py:117-123): slot j reads logits[eid[j]] and writes
 * out[eid[j]] (original edge order).  exp(x - rowmax) / rowsum, true division. */
int pglb_edge_softmax_csr_ws(int64_t num_edges, size_t *ws_bytes);
int pglb_edge_softmax_csr_f32(const int64_t *indptr, const int64_t *eid, const float *logits,
                              float *out, int64_t n_rows, int64_t num_edges, int64_t H,
                              void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Backward kernels.  The reference gets every gradient from Paddle autograd through the ops
 * above; sum / mean aggregation backward is pglb_spmm_csr_f32 on the reverse CSR, the rest:
 * ---------------------------------------------------------------------------------- */
/* out[e,h] = <a[ia[e],h,:], b[ib[e],h,:]>  (a, b rows of H*Dh floats; ia/ib strided like
 * pglb_csr_build).  Gradient of send_ue_recv(mul) wrt the edge operand [E,H,1] (pgl/graph.py:930
 * as used by GATConv, pgl/nn/conv.py:339) and of send_uv(mul). */
int pglb_sddmm_dot_f32(const float *a, const float *b, const int64_t *ia, int64_t ia_stride,
                       const int64_t *ib, int64_t ib_stride, int64_t num_edges, int64_t H,
                       int64_t Dh, float *out, void *stream);
/* gradient of pglb_edge_softmax_csr_f32: grad_logits = alpha * (grad - rowsum(alpha * grad)),
 * same row / eid convention as the forward (pgl/math.py:216-224 differentiated). */
int pglb_edge_softmax_bwd_csr_f32(const int64_t *indptr, const int64_t *eid, const float *alpha,
                                  const float *grad, float *grad_logits, int64_t n_rows,
                                  int64_t num_edges, int64_t H, void *stream);
/* gradient of send_u_recv(max|min) wrt x on the reverse (src-keyed) CSR: every source entry that
 * equals the reduced output receives the output's gradient (Paddle's send_u_recv grad contract).
 *   src_indptr[n_src+1], dst_of_slot[E]; x [n_src, D], out / grad_out [n_dst, D], grad_x [n_src, D] */
int pglb_maxmin_bwd_f32(const int64_t *src_indptr, const int64_t *dst_of_slot, const float *x,
                        const float *out, const float *grad_out, float *grad_x, int64_t n_src,
                        int64_t D, void *stream);

/* GAT attention in one launch (inference path of GATConv, pgl/nn/conv.py:333-335): for every dst row
 * d and head h, alpha[j,h] = softmax_j( leaky_relu(attn_src[cols[j],h] + attn_dst[d,h]) ) over the
 * row's slots j -- send_uv(add) + LeakyReLU + edge_softmax without materialising the [E,H] logits.
 * alpha_slots is in CSR SLOT order (row-contiguous), which is what pglb_spmm_csr_f32 reads
 * sequentially when eid == NULL.  ws as pglb_edge_softmax_csr_ws. */
int pglb_gat_attention_csr_f32(const int64_t *indptr, const int64_t *cols, const float *attn_src,
                               const float *attn_dst, float negative_slope, float *alpha_slots,
                               int64_t n_rows, int64_t num_edges, int64_t H, void *ws,
                               size_t ws_bytes, void *stream);

/* The whole GAT aggregation in ONE pass (inference path of GATConv, pgl/nn/conv.py:333-339):
 *   out[d,h,:] = sum_j softmax_j( leaky_relu(attn_src[cols[j],h] + attn_dst[d,h]) ) * f[cols[j],h,:]
 * send_uv + LeakyReLU + edge_softmax + send_ue_recv(mul,sum) with an online softmax inside the
 * wide-row aggregation kernel: neither the logits nor alpha are ever written.  f rows of
 * H*head_dim <= 128 floats (head_dim % 4 == 0, 16-byte aligned); ws as pglb_spmm_csr_ws(D = H*head_dim). */
int pglb_gat_fused_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                           const float *attn_src, const float *attn_dst, float negative_slope,
                           float *out, int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges,
                           int64_t H, int64_t head_dim, void *ws, size_t ws_bytes, void *stream);

/* GATConv's attention projections (pgl/nn/conv.py:323-326: paddle.sum(feature * weight_src, -1) and the same with
 * weight_dst -- two multiplies, two reductions, two [N, H, head_dim] temporaries) in one pass over f:
 *   attn_src[n,h] = <f[n,h,:], w_src[h,:]>,  attn_dst[n,h] = <f[n,h,:], w_dst[h,:]>.
 * f rows of H*head_dim <= 128 floats, 16-byte aligned; head_dim in {4, 8, ..., 128}. */
int pglb_head_dots_f32(const float *f, int64_t ldf, int64_t n, int64_t H, int64_t head_dim, const float *w_src,
                       const float *w_dst, float *attn_src, float *attn_dst, void *stream);
/* The same over bfloat16 / float16 f (`dtype`, ldf in elements, rows 16-byte aligned); w_src, w_dst, attn_src and
 * attn_dst are float32.  f is widened exactly and the products and adds are the fp32 entry's, in the same order: the
 * result equals pglb_head_dots_f32 on the widened f bit for bit.  Unknown dtype: PGLB_EINVAL. */
int pglb_head_dots_x16(const void *f, int64_t ldf, int64_t n, int64_t H, int64_t head_dim, int dtype,
                       const float *w_src, const float *w_dst, float *attn_src, float *attn_dst, void *stream);

/* Training forward of the same layer (GATConv under autograd, pgl/nn/conv.py:333-339; the reference gets the
 * backward from Paddle autograd over four ops): the same single launch, which also leaves
 *   lse[d,h] = log sum_j exp(leaky_relu(attn_src[cols[j],h] + attn_dst[d,h]))
 * for every row with at least one in-edge (other rows of lse are not written).  PGLB_EUNSUPPORTED when the shape is
 * outside the TMA kernel (H % 4 != 0, slope outside [0, 1], rows not 16-byte aligned): the caller keeps the
 * op-by-op path, every op of which has a backward. */
int pglb_gat_fused_train_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                 const float *attn_src, const float *attn_dst, float negative_slope,
                                 float *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src,
                                 int64_t num_edges, int64_t H, int64_t head_dim, void *ws, size_t ws_bytes,
                                 void *stream);

/* Per-edge part of that layer's backward.  rows[j] / cols[j] / eid[j] = destination, source and original edge id
 * of dst-CSR slot j (EdgeIndex.triples(); eid NULL = identity).  With z = attn_src[src,h] + attn_dst[dst,h]:
 *   alpha_e[e,h] = exp(leaky_relu(z) - lse[dst,h])                                   (the attention weight, rebuilt)
 *   dz_e[e,h]    = alpha * (<grad_out[dst,h,:], f[src,h,:]> - <grad_out[dst,h,:], out[dst,h,:]>) * leaky_relu'(z)
 * both [num_edges, H] in ORIGINAL edge order.  The caller finishes with reverse-CSR aggregations:
 * grad f = send_ue_recv(grad_out, alpha_e, mul, sum) over the src-keyed CSR, grad attn_src / grad attn_dst = segment
 * sums of dz_e over the src- / dst-keyed CSR.  head_dim in {4, 8, 16, 32, 64, 128}, H*head_dim <= 128. */
int pglb_gat_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                          int64_t ldf, const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                          const float *attn_src, const float *attn_dst, const float *lse,
                          float negative_slope, int64_t num_edges, int64_t H, int64_t head_dim,
                          float *alpha_e, float *dz_e, void *stream);

/* The fused GAT aggregation over bfloat16 / float16 features (`dtype`): the fp32 entries' arguments, f and out in
 * `dtype` (ldf / ldo in elements), attn_src, attn_dst and lse float32.
 *   - Shapes: H % 4 == 0, H <= 32, D = H * head_dim <= 128 with D % 8 == 0, 0 <= slope <= 1, the kernel's
 *     shared-memory budget, 16-byte aligned attn_src: otherwise PGLB_EUNSUPPORTED (there is no 16-bit fallback
 *     kernel).  f and out 16-byte aligned with ldf, ldo % 8 == 0: otherwise PGLB_ESHAPE.
 *   - Numerics: f is widened exactly; logits, LeakyReLU, the online softmax, rescales and accumulation are the fp32
 *     kernel's instructions in the same slot order; cut-row partials and (m, l) are fp32; each output element is
 *     rounded once, to nearest even.  So out == round16(pglb_gat_fused_csr_f32 on the widened f) bit for bit, and
 *     the train entry's lse equals the fp32 train entry's lse bit for bit, for every shape both run on the TMA kernel.
 *   - One shape only the 16-bit rings hold: H = 32 with head_dim = 4 (the halved feature rows leave room for 32
 *     attention floats per row).  There the fp32 inference entry runs its per-slot kernel and the fp32 train entry
 *     returns PGLB_EUNSUPPORTED, so nothing fp32 is bitwise comparable: out is within 2 u |ref32|_inf of the fp32
 *     inference entry's output on the widened f (u = 2^-8 bf16, 2^-11 fp16), and lse within the path's 1e-4
 *     relative bar of the exact log-sum-exp.
 *   - Unknown dtype: PGLB_EINVAL; NULL lse on the train entry (n_dst > 0): PGLB_EINVAL.  All argument checks precede
 *     any CUDA call.  ws as pglb_spmm_csr_ws(D = H*head_dim). */
int pglb_gat_fused_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                           const float *attn_src, const float *attn_dst, float negative_slope, void *out,
                           int64_t ldo, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim,
                           int dtype, void *ws, size_t ws_bytes, void *stream);
int pglb_gat_fused_train_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                 const float *attn_src, const float *attn_dst, float negative_slope, void *out,
                                 int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H,
                                 int64_t head_dim, int dtype, void *ws, size_t ws_bytes, void *stream);
/* pglb_gat_bwd_edge_f32 over bfloat16 / float16 f, grad_out and out (`dtype`, rows 16-byte aligned, ld in elements);
 * attn_src, attn_dst, lse, alpha_e and dz_e are float32.  The three row inputs are widened exactly and every value
 * after that is the fp32 kernel's: alpha_e and dz_e equal pglb_gat_bwd_edge_f32 on the widened inputs bit for bit.
 * In training, out is the forward's rounded 16-bit output, so delta = <grad_out, out> uses the rounded out.  Unknown
 * dtype: PGLB_EINVAL. */
int pglb_gat_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f, int64_t ldf,
                          const void *grad_out, int64_t ldg, const void *out, int64_t ldo, const float *attn_src,
                          const float *attn_dst, const float *lse, float negative_slope, int64_t num_edges, int64_t H,
                          int64_t head_dim, int dtype, float *alpha_e, float *dz_e, void *stream);

/* Training with attention dropout (pgl/nn/conv.py:337-339: dropout on the normalised attention, per edge and head):
 *   out[d,h,:] = sum_j s * m[j,h] * alpha[j,h] * f[cols[j],h,:],   m in {0, 1},  s = (float)(1 / (1 - attn_drop)).
 *   - The stream: the keep bit m of dst-CSR slot j (absolute slot index) and head h is word h % 4 of
 *     Philox4x32-10(counter = (j lo32, j hi32, h / 4, (uint32_t)(offset / 4)), key = (seed lo32, seed hi32)), kept iff
 *     word >= thresh = min(floor(attn_drop * 2^32), 2^32 - 1).  thresh and s are derived in double from the float
 *     attn_drop.  The forward and the backward recompute m in registers from (seed, offset); no mask is stored.
 *     pglb_attn_dropout_keep_host gives the same bits on the host.
 *   - Forward (pglb_gat_fused_train_drop_csr_*): the train entries' arguments plus attn_drop, seed, offset.  The
 *     online softmax's running sum keeps every slot and only the accumulator skips dropped ones, so lse is bitwise
 *     the train entry's lse; the row's quotient is multiplied by s once, after the division.
 *   - Backward (pglb_gat_bwd_edge_drop_*): the edge entries' arguments plus the forward's attn_drop, seed, offset.
 *     d alpha = s m <grad_out, f[src]>; delta = <grad_out, out> is unchanged; alpha_e holds the dropped attention
 *     beta = m ? fl(alpha * s) : 0, with which grad f is aggregated as before.
 *   - Bit anchors: attn_drop = 1e-12 (thresh 0, s = 1.0f) keeps every slot and gives out, lse, alpha_e and dz_e
 *     bitwise equal to the entries without dropout; the *_x16 siblings relate to the f32 ones as without dropout.
 *   - attn_drop outside (0, 1) (NaN included) or offset % 4 != 0: PGLB_EINVAL, checked before anything else and before
 *     any CUDA call.  H % 4 != 0 and the shapes the siblings refuse: PGLB_EUNSUPPORTED. */
int pglb_gat_fused_train_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                      const float *attn_src, const float *attn_dst, float negative_slope, float *out,
                                      int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                                      int64_t H, int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                      void *ws, size_t ws_bytes, void *stream);
int pglb_gat_fused_train_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                      const float *attn_src, const float *attn_dst, float negative_slope, void *out,
                                      int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                                      int64_t H, int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                      uint64_t offset, void *ws, size_t ws_bytes, void *stream);
int pglb_gat_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                               int64_t ldf, const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                               const float *attn_src, const float *attn_dst, const float *lse, float negative_slope,
                               int64_t num_edges, int64_t H, int64_t head_dim, float attn_drop, uint64_t seed,
                               uint64_t offset, float *alpha_e, float *dz_e, void *stream);
int pglb_gat_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                               int64_t ldf, const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                               const float *attn_src, const float *attn_dst, const float *lse, float negative_slope,
                               int64_t num_edges, int64_t H, int64_t head_dim, int dtype, float attn_drop,
                               uint64_t seed, uint64_t offset, float *alpha_e, float *dz_e, void *stream);
/* keep_words[i] = the keep word of dst-CSR slot slot0 + i (bit h = head h kept) of the stream above, computed on the
 * host by the kernels' own function.  H % 4 == 0, 4 <= H <= 32 (else PGLB_EUNSUPPORTED); attn_drop and offset as
 * above; n_slots = 0 does nothing. */
int pglb_attn_dropout_keep_host(uint64_t seed, uint64_t offset, float attn_drop, int64_t slot0, int64_t n_slots,
                                int64_t H, uint32_t *keep_words);

/* Dot-product attention of TransformerConv without edge features (pgl/nn/conv.py:808-847: send q[dst] * k[src] summed
 * over the head dim, softmax over the in-edges, weighted sum of v[src]) in ONE pass, the GAT kernel's online softmax:
 *   s_j = <q[d,h,:], k[cols[j],h,:]>,  lse[d,h] = log sum_j exp(s_j),  out[d,h,:] = sum_j exp(s_j - lse) v[cols[j],h,:]
 * over the dst-CSR slots j of row d (rows without in-edges: out = 0).  q is already scaled by 1 / sqrt(head_dim).  No
 * [E, H * head_dim] product and no [E, H] score is ever written.
 *   - q [n_dst, H * head_dim], k and v [n_src, H * head_dim], out [n_dst, ...] with row strides ldq, ldk, ldv, ldo in
 *     elements.  lse [n_dst, H] float32 is nullable (inference); when given, rows with at least one in-edge are
 *     written (others are not) -- all the edge backward needs.  ws as pglb_spmm_csr_ws(D = H * head_dim).
 *   - Shapes: D = H * head_dim <= 128 in 16-byte rows (D % 4 == 0 float32, D % 8 == 0 16-bit), head_dim in
 *     {4, 8, ..., 128}, n_src < 2^31 - 1: otherwise PGLB_EUNSUPPORTED.  q, k, v, out not 16-byte aligned, a row stride
 *     below D or not a multiple of 16 bytes: PGLB_ESHAPE.
 *   - _x16 (`dtype` bfloat16 / float16 q, k, v and out; lse float32): rows are widened exactly and every later operation
 *     is the float32 kernel's in the same slot order, rounded once on the store, so out == round16(pglb_dot_attn_csr_f32
 *     on the widened q, k, v) and lse equals its lse, bit for bit.  Unknown dtype: PGLB_EINVAL.
 *   - _drop_ (attention dropout): the arguments plus attn_drop, seed, offset, the stream and rules of the GAT dropout
 *     entries above (same keep word per dst-CSR slot and head, H % 4 == 0):
 *     out = sum_j s m_j exp(s_j - lse) v[cols[j]], and lse is bitwise the value without dropout.
 *   - All argument checks precede any CUDA call. */
int pglb_dot_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *q, int64_t ldq, const float *k,
                          int64_t ldk, const float *v, int64_t ldv, float *out, int64_t ldo, float *lse, int64_t n_dst,
                          int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, void *ws, size_t ws_bytes,
                          void *stream);
int pglb_dot_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq, const void *k,
                          int64_t ldk, const void *v, int64_t ldv, void *out, int64_t ldo, float *lse, int64_t n_dst,
                          int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, int dtype, void *ws,
                          size_t ws_bytes, void *stream);
int pglb_dot_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *q, int64_t ldq, const float *k,
                               int64_t ldk, const float *v, int64_t ldv, float *out, int64_t ldo, float *lse,
                               int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim,
                               float attn_drop, uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes, void *stream);
int pglb_dot_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *q, int64_t ldq, const void *k,
                               int64_t ldk, const void *v, int64_t ldv, void *out, int64_t ldo, float *lse,
                               int64_t n_dst, int64_t n_src, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                               float attn_drop, uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes, void *stream);

/* Per-edge part of that attention's backward.  rows / cols / eid as pglb_gat_bwd_edge_f32; lse from the forward;
 * grad_out = G.  With s and a = exp(s - lse[dst,h]) rebuilt (s bit for bit the forward's score):
 *   beta_e[e,h] = a,   ds_e[e,h] = a * (<G[dst,h,:], v[src,h,:]> - <G[dst,h,:], out[dst,h,:]>)
 * both [num_edges, H] float32 in ORIGINAL edge order.  The caller finishes with three aggregations:
 * grad q = send_ue_recv(k, ds_e, mul, sum) over the dst-keyed CSR, grad k = send_ue_recv(q, ds_e, mul, sum) and
 * grad v = send_ue_recv(grad_out, beta_e, mul, sum) over the src-keyed CSR.  head_dim in {4, 8, ..., 128},
 * H*head_dim <= 128, rows 16-byte aligned.
 *   - _x16: the row inputs in `dtype`, widened exactly; beta_e and ds_e equal the f32 entry's on the widened inputs
 *     bit for bit.
 *   - _drop_: the forward's attn_drop, seed, offset; da is multiplied by s m, and beta_e = m ? fl(a * s) : 0. */
int pglb_dot_attn_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *q,
                               int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv,
                               const float *grad_out, int64_t ldg, const float *out, int64_t ldo, const float *lse,
                               int64_t num_edges, int64_t H, int64_t head_dim, float *beta_e, float *ds_e,
                               void *stream);
int pglb_dot_attn_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *q,
                               int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                               const void *grad_out, int64_t ldg, const void *out, int64_t ldo, const float *lse,
                               int64_t num_edges, int64_t H, int64_t head_dim, int dtype, float *beta_e, float *ds_e,
                               void *stream);
int pglb_dot_attn_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *q,
                                    int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv,
                                    const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                    const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, float attn_drop,
                                    uint64_t seed, uint64_t offset, float *beta_e, float *ds_e, void *stream);
int pglb_dot_attn_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *q,
                                    int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                    const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                    const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                                    float attn_drop, uint64_t seed, uint64_t offset, float *beta_e, float *ds_e,
                                    void *stream);

/* Dot-product attention of TransformerConv WITH edge features (pgl/nn/conv.py:808-847 with edge_feat: the score of
 * q[dst] * (k[src] + e) summed over the head dim, the weighted sum of v[src] + e) in ONE pass, as pglb_dot_attn_csr_*:
 *   s_j = <q[d,h,:], k[cols[j],h,:] + e[eid[j],h,:]>,  lse[d,h] = log sum_j exp(s_j),
 *   out[d,h,:] = sum_j exp(s_j - lse) (v[cols[j],h,:] + e[eid[j],h,:])
 * (rows without in-edges: out = 0).  The add comes first, then the dot, both in float32, so e = 0 gives the
 * pglb_dot_attn_csr_* output and lse bit for bit.
 *   - The pglb_dot_attn_csr_* arguments, rules and return codes, plus eid [num_edges] (dst-CSR slot -> edge id, as the
 *     edge backward's eid), e [num_edges, H * head_dim] in EDGE-ID order in q's dtype, row stride lde in elements.
 *     NULL eid or e with edges: PGLB_EINVAL.  e not 16-byte aligned, lde below D or not a multiple of 16 bytes:
 *     PGLB_ESHAPE.
 *   - _x16 and _drop_: as pglb_dot_attn_csr_x16 / pglb_dot_attn_drop_csr_*; out == round16(the f32 entry on the
 *     widened q, k, v, e), and with dropout out = sum_j s m_j exp(s_j - lse) (v_j + e_j), lse the value without it.
 *   - All argument checks precede any CUDA call. */
int pglb_dot_attn_e_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const float *q, int64_t ldq,
                            const float *k, int64_t ldk, const float *v, int64_t ldv, const float *e, int64_t lde,
                            float *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                            int64_t H, int64_t head_dim, void *ws, size_t ws_bytes, void *stream);
int pglb_dot_attn_e_csr_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *q, int64_t ldq,
                            const void *k, int64_t ldk, const void *v, int64_t ldv, const void *e, int64_t lde,
                            void *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src, int64_t num_edges,
                            int64_t H, int64_t head_dim, int dtype, void *ws, size_t ws_bytes, void *stream);
int pglb_dot_attn_e_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const float *q,
                                 int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv, const float *e,
                                 int64_t lde, float *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src,
                                 int64_t num_edges, int64_t H, int64_t head_dim, float attn_drop, uint64_t seed,
                                 uint64_t offset, void *ws, size_t ws_bytes, void *stream);
int pglb_dot_attn_e_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *q,
                                 int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv, const void *e,
                                 int64_t lde, void *out, int64_t ldo, float *lse, int64_t n_dst, int64_t n_src,
                                 int64_t num_edges, int64_t H, int64_t head_dim, int dtype, float attn_drop,
                                 uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes, void *stream);

/* Per-edge part of that attention's backward: pglb_dot_attn_bwd_edge_* with k + e and v + e in place of k and v (s
 * rebuilt bit for bit from the forward's score), plus the edge-feature gradient
 *   grad_e[e,h,:] = ds_e[e,h] * q[dst,h,:] + beta_e[e,h] * G[dst,h,:]
 * in e's dtype, each edge's row written once, no atomics.  e [num_edges, H * head_dim] in edge-id order (row stride
 * lde); grad_e is nullable (e needs no gradient), row stride ldge.  The caller finishes grad q with one more
 * aggregation, send_ue_recv(e, ds_e, mul, sum) over the dst-keyed CSR with eid as its column array; grad k and grad v
 * are those of pglb_dot_attn_bwd_edge_*.  NULL e with edges: PGLB_EINVAL; e or grad_e not 16-byte aligned, lde or
 * ldge below D or not a multiple of 16 bytes: PGLB_ESHAPE.  _x16 / _drop_ as there; grad_e == round16(the f32
 * entry's on the widened inputs). */
int pglb_dot_attn_e_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *q,
                                 int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv, const float *e,
                                 int64_t lde, const float *grad_out, int64_t ldg, const float *out, int64_t ldo,
                                 const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, float *beta_e,
                                 float *ds_e, float *grad_e, int64_t ldge, void *stream);
int pglb_dot_attn_e_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *q,
                                 int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv, const void *e,
                                 int64_t lde, const void *grad_out, int64_t ldg, const void *out, int64_t ldo,
                                 const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                                 float *beta_e, float *ds_e, void *grad_e, int64_t ldge, void *stream);
int pglb_dot_attn_e_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *q,
                                      int64_t ldq, const float *k, int64_t ldk, const float *v, int64_t ldv,
                                      const float *e, int64_t lde, const float *grad_out, int64_t ldg, const float *out,
                                      int64_t ldo, const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                      float attn_drop, uint64_t seed, uint64_t offset, float *beta_e, float *ds_e,
                                      float *grad_e, int64_t ldge, void *stream);
int pglb_dot_attn_e_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *q,
                                      int64_t ldq, const void *k, int64_t ldk, const void *v, int64_t ldv,
                                      const void *e, int64_t lde, const void *grad_out, int64_t ldg, const void *out,
                                      int64_t ldo, const float *lse, int64_t num_edges, int64_t H, int64_t head_dim,
                                      int dtype, float attn_drop, uint64_t seed, uint64_t offset, float *beta_e,
                                      float *ds_e, void *grad_e, int64_t ldge, void *stream);

/* GATv2 attention (pgl/nn/conv.py:420-427: send_uv(feature, feature, add), LeakyReLU, the sum with attn over the head
 * dim, edge_softmax, attention dropout, send_ue_recv(mul, sum)) in ONE pass, the GAT kernel's online softmax:
 *   z_j = f[cols[j],h,:] + f[d,h,:],  s_j = sum_c a[h,c] lrelu(z_j,c),  lrelu(x) = max(x, slope x),
 *   lse[d,h] = log sum_j exp(s_j),  out[d,h,:] = sum_j exp(s_j - lse) f[cols[j],h,:]
 * over the dst-CSR slots j of row d (rows without in-edges: out = 0).  No [E, H * head_dim] tensor is ever written.
 *   - f [n, H * head_dim] with row stride ldf, out [n, ...] with row stride ldo, in elements; attn = a, H * head_dim
 *     float32.  lse [n, H] float32 is nullable (inference); when given, rows with at least one in-edge are written
 *     (others are not).  ws as pglb_spmm_csr_ws(n, num_edges, H * head_dim).
 *   - Shapes: D = H * head_dim <= 128 in 16-byte rows (D % 4 == 0 float32, D % 8 == 0 16-bit), head_dim in
 *     {4, 8, ..., 128}, 0 <= negative_slope <= 1, n < 2^31 - 1: otherwise PGLB_EUNSUPPORTED.  f, attn, out not 16-byte
 *     aligned, a row stride below D or not a multiple of 16 bytes: PGLB_ESHAPE.
 *   - _x16 (`dtype` bfloat16 / float16 f and out; attn and lse float32): rows are widened exactly and every later
 *     operation is the float32 kernel's in the same slot order, rounded once on the store, so out ==
 *     round16(pglb_gatv2_attn_csr_f32 on the widened f) and lse equals its lse, bit for bit.  Unknown dtype: PGLB_EINVAL.
 *   - _drop_ (attention dropout): attn_drop, seed, offset with the stream and rules of the GAT dropout entries above
 *     (same keep word per dst-CSR slot and head, H % 4 == 0): out = sum_j s m_j exp(s_j - lse) f[cols[j]], and lse is
 *     bitwise the value without dropout.
 *   - All argument checks precede any CUDA call. */
int pglb_gatv2_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf, const float *attn,
                            float negative_slope, float *out, int64_t ldo, float *lse, int64_t n, int64_t num_edges,
                            int64_t H, int64_t head_dim, void *ws, size_t ws_bytes, void *stream);
int pglb_gatv2_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *attn,
                            float negative_slope, void *out, int64_t ldo, float *lse, int64_t n, int64_t num_edges,
                            int64_t H, int64_t head_dim, int dtype, void *ws, size_t ws_bytes, void *stream);
int pglb_gatv2_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                                 const float *attn, float negative_slope, float *out, int64_t ldo, float *lse, int64_t n,
                                 int64_t num_edges, int64_t H, int64_t head_dim, float attn_drop, uint64_t seed,
                                 uint64_t offset, void *ws, size_t ws_bytes, void *stream);
int pglb_gatv2_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                                 const float *attn, float negative_slope, void *out, int64_t ldo, float *lse, int64_t n,
                                 int64_t num_edges, int64_t H, int64_t head_dim, int dtype, float attn_drop,
                                 uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes, void *stream);

/* Per-edge part of that attention's backward.  rows / cols / eid as pglb_gat_bwd_edge_f32; lse from the forward;
 * grad_out = G.  With s and a = exp(s - lse[dst,h]) rebuilt (s bit for bit the forward's score):
 *   beta_e[e,h] = a,   ds_e[e,h] = a * (<G[dst,h,:], f[src,h,:]> - <G[dst,h,:], out[dst,h,:]>)
 * both [num_edges, H] float32 in ORIGINAL edge order.  grad_attn (nullable, H * head_dim float32) receives
 * grad a[h,c] = sum_e ds_e[e,h] lrelu(z_e,c), reduced in a fixed order (bit-identical run to run) through ws
 * (pglb_gatv2_bwd_edge_ws bytes, 16-byte aligned; unused when grad_attn is NULL).  The caller finishes grad f with
 * pglb_gatv2_score_grad_* on the dst-keyed and the src-keyed CSR and send_ue_recv(grad_out, beta_e, mul, sum) over
 * the src-keyed CSR.  Shapes as the forward's: otherwise PGLB_EUNSUPPORTED.
 *   - _x16: f, grad_out and out in `dtype`, widened exactly; beta_e, ds_e and grad_attn equal the f32 entry's on the
 *     widened inputs bit for bit.
 *   - _drop_: the forward's attn_drop, seed, offset; da is multiplied by s m, and beta_e = m ? fl(a * s) : 0. */
int pglb_gatv2_bwd_edge_ws(int64_t num_edges, size_t *ws_bytes);
int pglb_gatv2_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f, int64_t ldf,
                            const float *attn, float negative_slope, const float *grad_out, int64_t ldg,
                            const float *out, int64_t ldo, const float *lse, int64_t num_edges, int64_t H,
                            int64_t head_dim, float *beta_e, float *ds_e, float *grad_attn, void *ws, size_t ws_bytes,
                            void *stream);
int pglb_gatv2_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f, int64_t ldf,
                            const float *attn, float negative_slope, const void *grad_out, int64_t ldg, const void *out,
                            int64_t ldo, const float *lse, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                            float *beta_e, float *ds_e, float *grad_attn, void *ws, size_t ws_bytes, void *stream);
int pglb_gatv2_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                                 int64_t ldf, const float *attn, float negative_slope, const float *grad_out,
                                 int64_t ldg, const float *out, int64_t ldo, const float *lse, int64_t num_edges,
                                 int64_t H, int64_t head_dim, float attn_drop, uint64_t seed, uint64_t offset,
                                 float *beta_e, float *ds_e, float *grad_attn, void *ws, size_t ws_bytes,
                                 void *stream);
int pglb_gatv2_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                                 int64_t ldf, const float *attn, float negative_slope, const void *grad_out,
                                 int64_t ldg, const void *out, int64_t ldo, const float *lse, int64_t num_edges,
                                 int64_t H, int64_t head_dim, int dtype, float attn_drop, uint64_t seed,
                                 uint64_t offset, float *beta_e, float *ds_e, float *grad_attn, void *ws,
                                 size_t ws_bytes, void *stream);

/* FAConv's self-gated aggregation (pgl/nn/conv.py:1306-1339: send_uv(g_src, g_dst, add), tanh, the product with
 * send_uv(norm, norm, mul), dropout, send_ue_recv(feature, alpha, mul, sum)) in ONE pass, no [E] tensor written:
 *   t_j = tanh(g_src[u] + g_dst[d]),  w_j = keep_j s ((t_j norm[u]) norm[d]),  out[d,:] = sum_j w_j f[u,:]
 * over the dst-CSR slots j = (u -> d) of row d (rows without in-edges: out = 0).  tanh is full-precision tanhf.
 *   - rec [n, 4] float32, 16-byte aligned: the node records (g_src[i], norm[i], g_dst[i], 0) -- one 16-byte bulk copy
 *     per slot.  f [n, D] with row stride ldf, out [n, D] with row stride ldo, in elements.  ws as
 *     pglb_spmm_csr_ws(n, num_edges, D).
 *   - Shapes: D <= 128 in 16-byte rows (D % 4 == 0 float32, D % 8 == 0 16-bit), n < 2^31 - 1: otherwise
 *     PGLB_EUNSUPPORTED.  f, rec, out not 16-byte aligned, a row stride below D or not a multiple of 16 bytes:
 *     PGLB_ESHAPE.
 *   - _x16 (`dtype` bfloat16 / float16 f and out; rec float32): rows are widened exactly and every later operation is
 *     the float32 kernel's in the same slot order, rounded once on the store: out == round16(pglb_fa_attn_csr_f32 on
 *     the widened f) bit for bit.  Unknown dtype: PGLB_EINVAL.
 *   - _drop_ (dropout on the edge weights): attn_drop in (0, 1), seed, offset (a multiple of 4) with the stream of the
 *     GAT dropout entries above: slot j is kept iff bit 0 of its 4-head keep word is set (pglb_attn_dropout_keep_host
 *     with H = 4, & 1), and s = (float)(1 / (1 - attn_drop)); without dropout keep_j s = 1.
 *   - All argument checks precede any CUDA call. */
int pglb_fa_attn_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf, const float *rec,
                         float *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D, void *ws, size_t ws_bytes,
                         void *stream);
int pglb_fa_attn_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf, const float *rec,
                         void *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D, int dtype, void *ws,
                         size_t ws_bytes, void *stream);
int pglb_fa_attn_drop_csr_f32(const int64_t *indptr, const int64_t *cols, const float *f, int64_t ldf,
                              const float *rec, float *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D,
                              float attn_drop, uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes, void *stream);
int pglb_fa_attn_drop_csr_x16(const int64_t *indptr, const int64_t *cols, const void *f, int64_t ldf,
                              const float *rec, void *out, int64_t ldo, int64_t n, int64_t num_edges, int64_t D,
                              int dtype, float attn_drop, uint64_t seed, uint64_t offset, void *ws, size_t ws_bytes,
                              void *stream);

/* Per-edge part of that aggregation's backward.  rows / cols / eid as pglb_gat_bwd_edge_f32 (eid nullable: identity);
 * rec the forward's node records; grad_out = G [n, D] with row stride ldg.  With t and w rebuilt by the forward's
 * function (w the forward's weight bit for bit):
 *   beta_e[e] = w,   dz_e[e] = keep s ((norm[u] norm[d]) (1 - t^2)) <G[d,:], f[u,:]>
 * both [num_edges] float32 in ORIGINAL edge order, no atomics.  The caller finishes the gradients on the existing
 * kernels: grad f = send_ue_recv(G, beta_e, mul, sum) over the src-keyed CSR, grad g_src / grad g_dst = segment sums of
 * dz_e over the src- / dst-keyed CSR.  Shapes and alignment as the forward's.
 *   - _x16: f and grad_out in `dtype`, widened exactly; beta_e and dz_e equal the f32 entry's on the widened inputs.
 *   - _drop_: the forward's attn_drop, seed, offset. */
int pglb_fa_bwd_edge_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f, int64_t ldf,
                         const float *rec, const float *grad_out, int64_t ldg, int64_t num_edges, int64_t D,
                         float *beta_e, float *dz_e, void *stream);
int pglb_fa_bwd_edge_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f, int64_t ldf,
                         const float *rec, const void *grad_out, int64_t ldg, int64_t num_edges, int64_t D, int dtype,
                         float *beta_e, float *dz_e, void *stream);
int pglb_fa_bwd_edge_drop_f32(const int64_t *rows, const int64_t *cols, const int64_t *eid, const float *f,
                              int64_t ldf, const float *rec, const float *grad_out, int64_t ldg, int64_t num_edges,
                              int64_t D, float attn_drop, uint64_t seed, uint64_t offset, float *beta_e, float *dz_e,
                              void *stream);
int pglb_fa_bwd_edge_drop_x16(const int64_t *rows, const int64_t *cols, const int64_t *eid, const void *f,
                              int64_t ldf, const float *rec, const void *grad_out, int64_t ldg, int64_t num_edges,
                              int64_t D, int dtype, float attn_drop, uint64_t seed, uint64_t offset, float *beta_e,
                              float *dz_e, void *stream);

/* The score-gradient aggregation of that backward:
 *   out[r, c] (+)= sum over the slots j of row r of ds[eid[j], h(c)] * attn[c] * lrelu'(f[r, c] + f[cols[j], c])
 * lrelu'(x) = 1 if x > 0 else negative_slope (torch's convention at 0).  On the dst-keyed CSR it is the dst term of
 * grad f, on the src-keyed CSR the src term; the [E, H * head_dim] dz is recomputed, never stored.  ds [E, H] float32
 * from pglb_gatv2_bwd_edge_*, eid nullable (identity).  out float32 [n_rows, H * head_dim], row stride ldo; accumulate:
 * add out's previous contents.  Every row's sum runs in slot order (rows longer than 1024 slots in fixed 1024-slot
 * chunks, summed in chunk order) with no atomics: bit-identical run to run.  ws as pglb_spmm_csr_ws(n_rows,
 * num_edges, H * head_dim).  D <= 128 in 16-byte rows, head_dim % 4 == 0, 0 <= negative_slope <= 1: otherwise
 * PGLB_EUNSUPPORTED; f, attn, out not 16-byte aligned: PGLB_ESHAPE.  _x16: f in `dtype`, widened exactly. */
int pglb_gatv2_score_grad_f32(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const float *f,
                              int64_t ldf, const float *attn, float negative_slope, const float *ds, float *out,
                              int64_t ldo, int64_t n_rows, int64_t num_edges, int64_t H, int64_t head_dim,
                              int accumulate, void *ws, size_t ws_bytes, void *stream);
int pglb_gatv2_score_grad_x16(const int64_t *indptr, const int64_t *cols, const int64_t *eid, const void *f,
                              int64_t ldf, const float *attn, float negative_slope, const float *ds, float *out,
                              int64_t ldo, int64_t n_rows, int64_t num_edges, int64_t H, int64_t head_dim, int dtype,
                              int accumulate, void *ws, size_t ws_bytes, void *stream);

/* out[M, N] = act(x[M, K] @ w[K, N] + bias[N]) -- the dense transform of the conv layers
 * (pgl/nn/conv.py:238-251 GCNConv: `self.linear(...)`, `+ self.bias`, activation; the same Linear in
 * GATConv :321 / GraphSageConv :107-108) on the tensor cores with 3xTF32 error compensation (fp32-level
 * accuracy, fp32 accumulate), bias and ReLU fused into the single write of out.
 * w is contiguous [K, N] (paddle.nn.Linear layout); K % 4 == 0, 4 <= K <= 128; N in {64, 128};
 * ldx % 4 == 0, x 16-byte aligned; bias may be NULL; act: 0 none, 1 relu. */
int pglb_linear_tf32x3_f32(const float *x, int64_t ldx, const float *w, const float *bias, float *out,
                           int64_t ldo, int64_t M, int64_t K, int64_t N, int act, void *stream);

/* ------------------------------------------------------------------------------------
 * RGCNConv's relation-typed aggregation (pgl/nn/conv.py:998-1024: sum_r send_recv(x @ W_r, mean) over the
 * relations' graphs), reassociated as out[d] = sum_r A_r[d] W_r with A_r[d] the mean of x[src] over the r-run of
 * row d.  The CSR is typed: the slots of every row are grouped by relation, ascending relation id, so a row's r-run
 * is one contiguous slot range; rel[slot] is its relation (int16).  fp32 only, 3xTF32 products with fp32
 * accumulation (the accuracy contract of pglb_linear_tf32x3_f32).  No floating-point atomics: outputs are
 * bit-identical run to run.  Every argument check returns PGLB_EINVAL before any CUDA call.
 * ---------------------------------------------------------------------------------- */

/* out[n_rows, N] (row stride ldo): out[d] = sum_r A_r[d] weight[r], weight contiguous [num_rels, K, N].
 * slot_w NULL: A_r[d] = mean over the r-run of x[cols[j]] (0 for an empty run) -- the forward on the typed dst-CSR.
 * slot_w non-NULL: A_r[d] = sum over the r-run of slot_w[j] x[cols[j]] -- grad x on the typed src-CSR with
 * slot_w[j] = 1 / cnt_r(dst_j) and weight = W^T [num_rels, O, D].  K, N multiples of 4 in [4, 128]; x 16-byte and
 * out 8-byte aligned, ldx % 4 == 0, ldo even; relation ids in [0, num_rels), num_rels <= 32767. */
int pglb_rgcn_agg_f32(const int64_t *indptr, const int64_t *cols, const int16_t *rel, const float *slot_w,
                      const float *x, int64_t ldx, const float *weight, int64_t num_rels, int64_t K, int64_t N,
                      float *out, int64_t ldo, int64_t n_rows, void *stream);

/* grad_weight[num_rels, D, O] = sum over the runs p of relation r of A_p^T grad_out[run_row[p]], A_p the mean of
 * x[cols[j]] over slots [run_beg[p], run_end[p]) of the typed dst-CSR.  The runs are sorted by relation: relation r
 * owns runs [run_off[r], run_off[r + 1]).  Work item i of relation r covers runs run_off[r] + (i - item_off[r]) * chunk
 * onward (chunk runs at most); item_off[num_rels + 1] is ascending with item_off[num_rels] = n_items.  Each item writes
 * an fp32 [D, O] partial into ws (pglb_rgcn_wgrad_ws bytes, 16-byte aligned), and a second launch adds a relation's
 * partials in item order (a relation without runs gets 0).  D, O multiples of 4 in [4, 128]; x and grad_out 16-byte
 * aligned with ldx, ldg multiples of 4. */
int pglb_rgcn_wgrad_ws(int64_t n_items, int64_t D, int64_t O, size_t *ws_bytes);
int pglb_rgcn_wgrad_f32(const int64_t *run_row, const int64_t *run_beg, const int64_t *run_end,
                        const int64_t *run_off, const int64_t *item_off, int64_t num_rels, int64_t n_items,
                        int64_t chunk, const int64_t *cols, const float *x, int64_t ldx, const float *grad_out,
                        int64_t ldg, int64_t D, int64_t O, float *grad_weight, void *ws, size_t ws_bytes,
                        void *stream);

/* ------------------------------------------------------------------------------------
 * Neighbour sampling + reindex for mini-batch GraphSAGE (SURVEY 8f rank 4).  Replace
 * paddle.geometric.sample_neighbors / reindex_graph as called by NeighborSampler.sample_neighbors
 * (pgl/sampling/sage.py:130-155) on the cached dst-CSR (row = adj_dst_index._sorted_v,
 * colptr = adj_dst_index._indptr).  Validated on hardware in round 2 (tests/test_gpu_sampling.py).
 * ---------------------------------------------------------------------------------- */
/* count[i] = min(deg(nodes[i]), sample_size)  (all neighbours when sample_size < 0);
 * offsets[0..n] = exclusive scan of count, offsets[n] = total (n + 1 entries). */
int pglb_sample_count(const int64_t *indptr, const int64_t *nodes, int64_t n, int64_t sample_size,
                      int64_t *count, int64_t *offsets, void *stream);
/* out_neighbors[offsets[i] + j] = j-th sampled in-neighbour of nodes[i]: the whole list in CSR order
 * when deg <= sample_size, else a uniform subset without replacement (Floyd), a pure function of
 * (seed, i).  out_eids (may be NULL) receives eid[slot] (or the CSR slot when eid is NULL).
 * sample_size <= 4096; degrees < 2^31. */
int pglb_sample_fill(const int64_t *indptr, const int64_t *row, const int64_t *eid, const int64_t *nodes,
                     int64_t n, int64_t sample_size, uint64_t seed, const int64_t *offsets,
                     int64_t *out_neighbors, int64_t *out_eids, void *stream);
/* Relation-typed sampling for HeteroNeighborSampler on a typed in-CSR: indptr / cols (src) / rel (int16 relation of
 * every slot) with the slots of every row grouped by relation in ascending relation id (heter_graph.typed_in_csr).
 * sample_sizes: HOST array of num_rels fan-outs k_r (negative = all neighbours, 0 = none, at most 4096), checked on
 * the host and copied to sizes_dev (device scratch of num_rels int32) on the stream; num_rels in [1, 32767].
 * Relation r's run of a row is found by binary search over rel: a row costs O(R log deg + sum k_r) however long
 * it is.  Relation ids outside [0, num_rels) are never sampled.
 * count[i] = sum_r min(deg_r(nodes[i]), k_r); offsets[0..n] = exclusive scan, offsets[n] = total. */
int pglb_sample_typed_count(const int64_t *indptr, const int16_t *rel, int64_t num_rels, const int64_t *sample_sizes,
                            int32_t *sizes_dev, const int64_t *nodes, int64_t n, int64_t *count, int64_t *offsets,
                            void *stream);
/* From out_neighbors[offsets[i]] on: the sampled in-neighbours of nodes[i], relation by relation in ascending order;
 * relation r's run whole in CSR order when deg_r <= k_r or k_r < 0, else a uniform k_r-subset without replacement
 * (Floyd) whose draw c is mix64(base(seed, i) + r 2^32 + c) -- with one relation, pglb_sample_fill's draws and
 * output.  out_rel receives the relation of every sampled slot; out_eids (may be NULL) eid[slot] (or the slot when
 * eid is NULL).  Degrees < 2^31. */
int pglb_sample_typed_fill(const int64_t *indptr, const int64_t *cols, const int16_t *rel, const int64_t *eid,
                           int64_t num_rels, const int64_t *sample_sizes, int32_t *sizes_dev, const int64_t *nodes,
                           int64_t n, uint64_t seed, const int64_t *offsets, int64_t *out_neighbors,
                           int16_t *out_rel, int64_t *out_eids, void *stream);
/* Dense lookup table for pglb_reindex_graph: num_nodes int64, filled with INT64_MAX ("empty"). */
int pglb_reindex_table_init(int64_t *table, int64_t num_nodes, void *stream);
int pglb_reindex_graph_ws(int64_t num_neighbors, size_t *ws_bytes);
/* paddle.geometric.reindex_graph(x, neighbors, count): out_nodes = x followed by the new ids among
 * neighbors in first-appearance order; reindex_src[p] = position of neighbors[p] in out_nodes;
 * reindex_dst[p] = i for the slots of x[i] (offsets as produced by pglb_sample_count, n + 1 entries).
 * x must hold distinct ids.  *num_out (device scalar) = number of entries written to out_nodes
 * (capacity n + m).  table: see pglb_reindex_table_init; left all-empty again on return. */
int pglb_reindex_graph(const int64_t *x, int64_t n, const int64_t *neighbors, const int64_t *offsets,
                       int64_t m, int64_t *table, int64_t *reindex_src, int64_t *reindex_dst,
                       int64_t *out_nodes, int64_t *num_out, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Random walks (csrc/walk.cu).  Replace pgl.sampling.random_walk / node2vec_walk / node2vec_walk_plus
 * (pgl/sampling/walk.py:23-183, graph_kernel.pyx:142-224) on the src-keyed CSR (indptr = adj_src_index._indptr,
 * cols = adj_src_index._sorted_v): one walker per thread, the whole walk in one launch.
 *   - Walker i starts at nodes[i] and writes row i of out (row-major, L columns): the walk, then -1 after it ends.
 *     A walk ends early exactly when its current node has no successors.  A start outside [0, num_nodes) gives a row
 *     of -1.  Successor ids are not range-checked (the graph build checks them).
 *   - Every draw is Philox4x32-10(counter = (i lo32, i hi32, step, trial), key = (seed lo32, seed hi32)): the walks
 *     are a pure function of (graph, nodes, seed).  A uniform slot of a row of deg slots is mulhi64(r64, deg) with
 *     r64 = (word1 << 32) | word0.
 *   - random_walk: at most max_depth nodes (max_depth - 1 steps), L = max_depth; each step takes the uniform slot of
 *     trial 0.
 *   - node2vec: up to max_depth steps, L = max_depth + 1 (the reference's count).  A step from cur with previous node
 *     prev takes slot s with probability proportional to w = 1/p if cols[s] == prev, 1 if cols[s] is a successor of
 *     prev (plus != 0: of any earlier node of the walk), 1/q otherwise; the first step (no prev) is the uniform slot of
 *     trial 0.  Rejection sampling: trial k proposes the uniform slot of trial k and accepts it iff
 *     word2 < floor(w / max(1/p, 1, 1/q) * 2^32); after cap = max(16, deg) rejected trials the step is an exact
 *     float64 inverse CDF over the row in slot order, with u = (r64 of trial cap >> 11) * 2^-53.  Membership is a binary search in
 *     sorted_cols: the successor columns with every row ascending by id (same indptr).  Cost per trial:
 *     O(log deg(prev)); plus: O(t log d) at step t.  stats (device, 2 uint64, may be NULL; the caller zeroes it)
 *     accumulates {candidate draws, fallback steps}.
 *   - max_depth outside [1, 2^31 - 1), p or q not positive and finite (or with an infinite reciprocal), a negative
 *     size or a NULL pointer with n > 0: PGLB_EINVAL before any CUDA call. */
int pglb_random_walk(const int64_t *indptr, const int64_t *cols, int64_t num_nodes, const int64_t *nodes, int64_t n,
                     int64_t max_depth, uint64_t seed, int64_t *out, void *stream);
int pglb_node2vec_walk(const int64_t *indptr, const int64_t *cols, const int64_t *sorted_cols, int64_t num_nodes,
                       const int64_t *nodes, int64_t n, int64_t max_depth, double p, double q, int plus,
                       uint64_t seed, int64_t *out, uint64_t *stats, void *stream);
/* The same walks on the host over host arrays, by the kernels' own step function, blocking: mode 0 = random_walk,
 * 1 = node2vec, 2 = node2vec_plus (p, q and sorted_cols are ignored in mode 0).  stats (host, may be NULL) receives
 * {candidate draws, fallback steps}.  For tests and small graphs. */
int pglb_walk_host(const int64_t *indptr, const int64_t *cols, const int64_t *sorted_cols, int64_t num_nodes,
                   const int64_t *nodes, int64_t n, int64_t max_depth, double p, double q, int mode, uint64_t seed,
                   int64_t *out, uint64_t *stats);
/* Metapath walks on a heterogeneous graph (replace the reference's examples/metapath2vec/datasets/sampling.py
 * metapath_randomwalk).  indptrs / cols are host arrays of m pointers, 1 <= m <= 64: position k of the metapath is a
 * relation's src-keyed CSR (indptrs[k], cols[k]) over the same num_nodes nodes; a relation may fill several positions.
 * Pass indptrs[k] in place of a relation's empty cols (it is never read).
 *   - Walker i starts at nodes[i] and writes row i of out (row-major, L = walk_length columns): at most walk_length
 *     nodes, then -1.  Step t (t = 0, 1, ...) goes from cur to the uniform slot of cur's row in relation position
 *     t % m, drawn as a random_walk step: mulhi64(r64, deg) with r64 from Philox4x32-10(counter = (i lo32, i hi32, t,
 *     0), key = (seed lo32, seed hi32)).  So m = 1 gives pglb_random_walk's walks bit for bit.
 *   - A walk ends early exactly when cur has no out-edge in the step's relation.  A start outside [0, num_nodes) gives
 *     a row of -1.  Nothing checks that the relations chain by node type.
 *   - m outside [1, 64], walk_length outside [1, 2^31 - 1), a negative size, or a NULL pointer with n > 0 (indptrs,
 *     cols, any of their first m entries, nodes, out): PGLB_EINVAL before any CUDA call.
 * pglb_metapath_walk: device pointers in indptrs / cols, nodes and out; one launch on `stream`.
 * pglb_metapath_walk_host: the same walks over host arrays by the kernel's own walk function, one walker after
 * another, blocking.  For tests and small graphs. */
int pglb_metapath_walk(const int64_t *const *indptrs, const int64_t *const *cols, int m, int64_t num_nodes,
                       const int64_t *nodes, int64_t n, int64_t walk_length, uint64_t seed, int64_t *out,
                       void *stream);
int pglb_metapath_walk_host(const int64_t *const *indptrs, const int64_t *const *cols, int m, int64_t num_nodes,
                            const int64_t *nodes, int64_t n, int64_t walk_length, uint64_t seed, int64_t *out);

/* ------------------------------------------------------------------------------------
 * Skip-gram pairs and alias-table sampling (csrc/skipgram.cu; alias build in csrc/host.cpp).  Replace the reference's
 * graph_kernel.skip_gram_gen_pair (graph_kernel.pyx:343-365) called once per walk, and the host negative sampling of
 * its walk examples (graph_kernel.alias_sample_build_table, graph_kernel.pyx:368-393, and alias_sample,
 * examples/metapath2vec/datasets/sampling.py:133-146).
 *
 * Counter tags: the fourth Philox counter word of the two streams below.  The walk kernels put a trial number there,
 * at most max(16, deg) for a row of deg slots, so no row shorter than 2^32 - 2 slots shares a counter with them. */
#define PGLB_SKIPGRAM_TAG 0xFFFFFFFFu
#define PGLB_ALIAS_TAG 0xFFFFFFFEu
/* Skip-gram pairs.  walks: int64 [B, L] row-major, each row a walk padded with -1 (the walk entries' layout).
 *   - Walk b has length n_b: the index of the first entry < 0 in its row, or L if there is none.
 *   - Centre i < n_b has the window w = 1 + mulhi32(word0, win_size), in [1, win_size], where word0..3 =
 *     Philox4x32-10(counter = (b lo32, b hi32, i, PGLB_SKIPGRAM_TAG), key = (seed lo32, seed hi32)).
 *   - The centre emits (walk[b][i], walk[b][j]) for every j from max(0, i - w) to min(n_b - 1, i + w) ascending,
 *     skipping each j with walk[b][j] == walk[b][i] (by node id, not position: a revisited node never pairs with
 *     itself).  Output order: walk, then centre, then j -- the reference's per-walk outputs concatenated.  Given the
 *     same windows the output is the reference's.
 *   - win_size in [1, 2^31), L in [0, 2^31 - 1), B >= 0; a NULL pointer with B > 0: PGLB_EINVAL before any CUDA call.
 *     B = 0 is a no-op (offsets is not written).  Pair offsets are int64; the total may exceed 2^32.
 * pglb_skipgram_count: offsets[0..B] = exclusive scan of the per-walk pair counts, offsets[B] = total (B + 1 device
 *   entries): one counting launch and the three launches of the multi-block int64 scan.  ws: device scratch of
 *   pglb_skipgram_count_ws(B) bytes (too small: PGLB_EWORKSPACE).
 * pglb_skipgram_fill: src[offsets[b] ..] / pos[offsets[b] ..] = the pairs of walk b (offsets from the count with the
 *   same walks, win_size and seed); one launch, a warp per walk.
 * pglb_skipgram_host: both over host arrays, blocking, by the kernels' own window and emit functions; src and pos may
 *   both be NULL to count only.  For tests and small batches. */
int pglb_skipgram_count_ws(int64_t B, size_t *ws_bytes);
int pglb_skipgram_count(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed, int64_t *offsets,
                        void *ws, size_t ws_bytes, void *stream);
int pglb_skipgram_fill(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed,
                       const int64_t *offsets, int64_t *src, int64_t *pos, void *stream);
int pglb_skipgram_host(const int64_t *walks, int64_t B, int64_t L, int64_t win_size, uint64_t seed, int64_t *offsets,
                       int64_t *src, int64_t *pos);
/* Alias table build, on the host: graph_kernel.pyx:368-393 exactly -- alias = probs * n in float64, the indices with
 * alias > 1 and < 1 on two stacks, and while both are non-empty: s = top of smaller (popped), l = top of larger,
 * events[s] = l, alias[l] -= (1 - alias[s]), pop l if alias[l] <= 1, push l on smaller if alias[l] < 1.  Output
 * equals the reference's bit for bit (compiled without FMA contraction), including the entries whose events stay 0
 * after rounding.  probs is used as given (no normalisation).  n = 0: no-op; n < 0 or a NULL pointer: PGLB_EINVAL. */
int pglb_alias_build_host(const double *probs, int64_t n, double *alias, int64_t *events);
/* Alias sampling: out[k], k < count, is draw k of the table (alias float64 [n], events int64 [n]):
 * word0..3 = Philox4x32-10(counter = (k lo32, k hi32, 0, PGLB_ALIAS_TAG), key = (seed lo32, seed hi32));
 * slot = mulhi64(word1 << 32 | word0, n); u = ((word2 << 32 | word3) >> 11) * 2^-53; out[k] = slot if u < alias[slot],
 * else events[slot] (the reference's alias_sample rule: uni >= alias[idx] takes the event).  n in [1, 2^32), count >= 0,
 * NULL pointers with count > 0: PGLB_EINVAL before any CUDA call; count = 0 is a no-op.
 * pglb_alias_sample: device arrays, one launch.  pglb_alias_sample_host: host arrays by the kernel's own draw. */
int pglb_alias_sample(const double *alias, const int64_t *events, int64_t n, int64_t count, uint64_t seed,
                      int64_t *out, void *stream);
int pglb_alias_sample_host(const double *alias, const int64_t *events, int64_t n, int64_t count, uint64_t seed,
                           int64_t *out);

/* Skip-gram negative-sampling loss, forward (csrc/sgns.cu).  Replaces the training step of the reference's walk models
 * (SkipGramModel.forward of examples/deepwalk/model.py and examples/metapath2vec/model.py: two embedding lookups, two
 * matmuls and BCEWithLogitsLoss on each), which materialises the [P, 1 + K, D] context rows.
 *   emb [n_emb, ld_emb] and ctx [n_ctx, ld_ctx] float32 tables (first D columns used; ctx == emb for a shared table),
 *   src[P] and dsts[P, 1 + K] int64 row ids (column 0 the positive, 1..K the negatives), every id inside its table
 *   (not checked here).  With s[p, j] = <emb[src[p]], ctx[dsts[p, j]]>:
 *     *loss   = ( mean_p softplus(-s[p, 0]) + mean_{p, k >= 1} softplus(s[p, k]) ) / 2
 *     c[p, 0] = -sigmoid(-s[p, 0]) / (2P),  c[p, k] = sigmoid(s[p, k]) / (2PK)     (float32 [P, 1 + K], = d loss / d s)
 *     w[p]    = sum_j c[p, j] ctx[dsts[p, j]]                                  (float32 [P, ldw], first D columns)
 *   softplus(x) = max(x, 0) + log1p(exp(-|x|)); saturated logits give finite values.  c and w are both given (training)
 *   or both NULL (loss only).  The loss is the sum of fixed-order per-block partials, then a one-block fixed-order sum:
 *   bit-identical run to run.  Two launches.  Any D >= 1; rows are read 16 bytes at a time when D, ld_emb, ld_ctx (and
 *   ldw) are multiples of 4 and the tables (and w) are 16-byte aligned, and held in registers up to D = 512 (256 when
 *   read 4 bytes at a time); wider rows stream through a warp per pair.
 *   Refused before any CUDA call: a NULL table, id array, loss or workspace (PGLB_EINVAL); P, K, D, n_emb or n_ctx < 1
 *   (PGLB_EINVAL); ld_emb, ld_ctx or (training) ldw < D (PGLB_ESHAPE); only one of c and w (PGLB_EINVAL); an output
 *   overlapping an input or another output (PGLB_EINVAL); ws below pglb_sgns_fwd_ws(P) bytes or not 8-byte aligned
 *   (PGLB_EWORKSPACE).
 * The gradients are segment sums of these by node id, and run on the aggregation entries: d emb[n] = g sum over pairs
 * with src[p] = n of w[p]; d ctx[m] = g sum over (p, j) with dsts[p, j] = m of c[p, j] emb[src[p]]. */
int pglb_sgns_fwd_ws(int64_t P, size_t *ws_bytes);
int pglb_sgns_fwd_f32(const float *emb, int64_t n_emb, int64_t ld_emb, const float *ctx, int64_t n_ctx, int64_t ld_ctx,
                      const int64_t *src, const int64_t *dsts, int64_t P, int64_t K, int64_t D, float *loss, float *c,
                      float *w, int64_t ldw, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Graph-level readouts (csrc/readout.cu).  Every entry is keyed by a segment CSR indptr[B + 1] (device int64,
 * non-decreasing, indptr[0] = 0, indptr[B] = N): segment g is the contiguous rows indptr[g] .. indptr[g + 1] - 1 (a
 * batched graph's _graph_node_index).  Every output element has exactly one writer, there are no atomics, and the
 * results are the same from run to run.  Bad arguments return PGLB_EINVAL before any CUDA call.
 *
 * Fused attention readout (GlobalAttention, Set2Set; reference pgl/nn/pool.py:121-179):
 *   out[g] = sum_{i in g} softmax_g(s)_i * x_i,  lse[g] = log sum_{i in g} exp(s_i)
 * with s_i = gate[i] (gate, [N]) or s_i = <x_i, query[g]> (query, [B, D]); pass exactly one of the two.  x [N, D], out
 * [B, D] row-major float32, 1 <= D <= 16384.  One pass over x with an online max and sum.  An empty segment gives a
 * zero row and lse = -inf.  Segments are split into chunks of 2048 rows (boundaries depend on the segment's length
 * only, so a segment's output is bit-identical wherever it sits in the batch); a longer segment's chunks write
 * partials to the workspace that a second launch merges in chunk order.  max_len: the longest segment.  With
 * max_len <= 2048 no workspace is needed (pglb_attn_readout_ws gives 0) and the call is one launch.  A max_len below
 * the true longest segment still gives correct results, but such a segment is then read as one chunk.
 * Backward (one launch when max_len <= 2048; a second merges grad_query otherwise): with a_i = exp(s_i - lse_g),
 *   ds_i = a_i (<x_i, grad_out_g> - <out_g, grad_out_g>),  grad_x_i = a_i grad_out_g (+ ds_i query_g),
 *   grad_gate_i = ds_i (gate given; grad_gate may be NULL),  grad_query_g = sum_i ds_i x_i (query given). */
int pglb_attn_readout_ws(int64_t num_segments, int64_t num_rows, int64_t dim, int64_t max_len, size_t *ws_bytes);
int pglb_attn_readout_f32(const float *x, int64_t num_rows, int64_t dim, const int64_t *indptr, int64_t num_segments,
                          int64_t max_len, const float *gate, const float *query, float *out, float *lse, void *ws,
                          size_t ws_bytes, void *stream);
int pglb_attn_readout_bwd_f32(const float *x, int64_t num_rows, int64_t dim, const int64_t *indptr,
                              int64_t num_segments, int64_t max_len, const float *gate, const float *query,
                              const float *out, const float *lse, const float *grad_out, float *grad_x,
                              float *grad_gate, float *grad_query, void *ws, size_t ws_bytes, void *stream);

/* Segmented top-k (segment_topk / SAGPool; reference pgl/math.py:299-364), two calls:
 *   count: k_g = min(k, n_g) when k > 0, else ceilf(ratio * (float)n_g) computed in fp32 as the reference does
 *          (ratio in (0, 1], otherwise PGLB_EINVAL); offsets[0 .. B] (device int64, B + 1) = exclusive prefix of k_g;
 *          info (device int64[2]) = {offsets[B] (total kept), longest segment}.  One launch.
 *   fill : perm[offsets[g] + r] = the node of rank r of segment g, r < k_g.  Ranks follow a total order: score
 *          descending, -0.0 == +0.0, NaN after every number, ties by ascending node index.  max_len = info[1]:
 *          segments of at most 2048 nodes are ranked in shared memory (one CTA per segment, one launch, no
 *          workspace); a longer max_len sorts (segment, score) keys with the stable radix sort of pglb_csr_build and
 *          needs pglb_segment_topk_ws bytes.  Both paths give the same perm.  A max_len below the longest segment
 *          still gives the same perm: a segment longer than the shared array is then ranked from global memory
 *          (quadratic in its length). */
int pglb_segment_topk_count(const int64_t *indptr, int64_t num_segments, float ratio, int64_t k, int64_t *offsets,
                            int64_t *info, void *stream);
int pglb_segment_topk_ws(int64_t num_segments, int64_t num_rows, int64_t max_len, size_t *ws_bytes);
int pglb_segment_topk_fill(const float *scores, int64_t num_rows, const int64_t *indptr, int64_t num_segments,
                           const int64_t *offsets, int64_t max_len, int64_t *perm, void *ws, size_t ws_bytes,
                           void *stream);

/* Dense batching (to_dense_batch / segment_padding; reference pgl/utils/transform.py:101-135, pgl/math.py:227-272),
 * copies by element size (2, 4 or 8 bytes), so exact in every dtype.  Rows are D contiguous elements.
 *   pad  : out[b, p] (out [B, max_len, D]) = x[indptr[b] + p] for p < n_b, else D copies of the element whose bits are
 *          the low elem_size bytes of fill_bits.  Each output row is written once; rows of a segment beyond max_len
 *          are dropped (the caller passes max_len >= the longest segment).
 *   unpad: out[i] = padded[b, i - indptr[b]] for every row i (the adjoint gather; zeros where i - indptr[b] >= max_len). */
int pglb_segment_pad(const void *x, int64_t num_rows, int64_t dim, int elem_size, const int64_t *indptr,
                     int64_t num_segments, int64_t max_len, uint64_t fill_bits, void *out, void *stream);
int pglb_segment_unpad(const void *padded, int64_t num_segments, int64_t max_len, int64_t dim, int elem_size,
                       const int64_t *indptr, int64_t num_rows, void *out, void *stream);

/* norm[i] = clip(float(degree[i]), 1)^-0.5 ; GF.degree_norm (graph_op.py:46-55) */
int pglb_degree_norm_f32(const int64_t *degree, int64_t n, float *norm, void *stream);

/* Strided host<->device copy on `stream` (cudaMemcpy2DAsync): moves a column block of a row-major
 * matrix without staging.  kind: 1 = host->device, 2 = device->host.  Used by the host-buffer
 * entry of the aggregation (features in pinned host memory): column chunks are independent for a
 * copy-message aggregation, so chunk c+1's upload, chunk c's kernel and chunk c-1's download
 * overlap (PCIe is full duplex). */
int pglb_memcpy2d_async(void *dst, size_t dst_pitch, const void *src, size_t src_pitch,
                        size_t width_bytes, size_t height, int kind, void *stream);

/* ------------------------------------------------------------------------------------
 * Peer-mappable device buffers for the multi-GPU halo pull (NVLink P2P, one process per GPU).
 * The only place the library allocates: cudaMalloc'ed buffers whose CUDA IPC handle (64 bytes)
 * other ranks open under THEIR device with pglb_ipc_open; kernels such as pglb_gather_rows_f32
 * then read the owner's HBM directly.  No reference counterpart (the reference replicates all
 * features on every GPU, pgl/graph.py:1410-1553).
 * ---------------------------------------------------------------------------------- */
int pglb_ipc_alloc(size_t bytes, void **dev_ptr, void *handle64);
int pglb_ipc_free(void *dev_ptr);
int pglb_ipc_open(const void *handle64, void **peer_ptr);
int pglb_ipc_close(void *peer_ptr);

/* Debug aid (scripts/task_trace.py): while `buffer` (device, capacity_tasks x 4 int64) is armed, the wide-row
 * aggregation kernels record (start ns, end ns, SM id, warp slot) for every task of a launch with at most
 * capacity_tasks tasks.  buffer = NULL disarms.  Process-global; not for concurrent use. */
int pglb_debug_task_trace(void *buffer, int64_t capacity_tasks);

/* ------------------------------------------------------------------------------------
 * Partition -> local-graph pipeline on the device (SURVEY.md section 8f rank 3; csrc/localgraph.cu).
 * ---------------------------------------------------------------------------------- */
/* graph_kernel.map_nodes(nodes, reindex) (pgl/graph_kernel.pyx:123-138) with the dict as a dense table
 * new_id[old_id] (table_size entries): out[i] = table[nodes[i]].  An id outside [0, table_size) gives -1 and
 * sets *bad_flag (device int, may be NULL; the caller zeroes it) -- the reference's unordered_map would
 * silently insert 0. */
int pglb_map_nodes(const int64_t *nodes, int64_t n, const int64_t *table, int64_t table_size,
                   int64_t *out, int32_t *bad_flag, void *stream);
/* graph_kernel.map_edges(eid, edges, reindex) (pgl/graph_kernel.pyx:104-120): out[i, :] = table[edges[eid[i], :]];
 * eid NULL = all edges in order.  edges / out contiguous [*, 2] int64. */
int pglb_map_edges(const int64_t *eid, int64_t n, const int64_t *edges, int64_t num_edges,
                   const int64_t *table, int64_t table_size, int64_t *out, int32_t *bad_flag, void *stream);
/* inverse[perm[j]] = j.  With perm = sorted_eid of pglb_csr_build(u = part) -- the stable sort of the nodes by
 * part -- inverse is the `new id of every node` of apps/GNNAutoScale/graph_partition.py:94-101 and the build's
 * indptr is its offsets array. */
int pglb_invert_perm(const int64_t *perm, int64_t n, int64_t *inverse, void *stream);
/* One rank's local graph of a 1-D node partition whose parts are contiguous id ranges (this rank owns
 * [lo, hi)).  Two calls, because the output sizes are data dependent:
 *   count: counts[0] = E_local (edges whose destination is owned), counts[1] = H (distinct remote sources);
 *          *bad_flag (device int, zeroed by the caller) is set when an endpoint lies outside [0, num_nodes).
 *   fill : eid[E_local]       ascending global edge ids of the local edges,
 *          dst_local[E_local] destination - lo,
 *          col_local[E_local] source - lo when owned, else (hi - lo) + position of the source in halo_ids,
 *          halo_ids[H]        ascending distinct remote source ids (= grouped by owner),
 *          recv_counts[K]     how many of them lie in [offsets[p], offsets[p+1])  (offsets: device, K + 1 entries).
 * The same workspace (pglb_halo_plan_ws bytes, 256-byte aligned) must be passed to both calls, untouched between. */
int pglb_halo_plan_ws(int64_t num_edges, int64_t num_nodes, size_t *ws_bytes);
int pglb_halo_plan_count(const int64_t *edges, int64_t num_edges, int64_t num_nodes, int64_t lo, int64_t hi,
                         int64_t *counts, int32_t *bad_flag, void *ws, size_t ws_bytes, void *stream);
int pglb_halo_plan_fill(const int64_t *edges, int64_t num_edges, int64_t num_nodes, int64_t lo, int64_t hi,
                        const int64_t *offsets, int64_t num_parts, int64_t *eid, int64_t *dst_local,
                        int64_t *col_local, int64_t *halo_ids, int64_t *recv_counts, void *ws, size_t ws_bytes,
                        void *stream);

/* ------------------------------------------------------------------------------------
 * Host: METIS K-way behind the same call shape as graph_kernel.metis_partition
 * (pgl/graph_kernel.pyx:434-472 <- pgl/partition.py:83-90).  libmetis (IDXTYPEWIDTH 64) is
 * dlopen()ed from `libmetis_path` (NULL = default search); returns PGLB_ENOLIB if absent.
 * ---------------------------------------------------------------------------------- */
int pglb_metis_partition(const char *libmetis_path, int64_t num_nodes, const int64_t *indptr,
                         const int64_t *adjncy, int64_t nparts, const int64_t *node_weights,
                         const int64_t *edge_weights, int recursive, int64_t *part);

#ifdef __cplusplus
}
#endif
#endif /* PGLB_H_ */
