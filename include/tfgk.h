/*
 * tfgk.h - C ABI of the H100 (sm_90a) message-passing kernel backend for tf_geometric's hot path.
 *
 * The reference (CrawlScript/tf_geometric @4539f11) has NO native FFI: its "operator API" for this path is a set
 * of Python functions built on stock TensorFlow ops and the tf_sparse package.  Each entry point below therefore
 * cites the reference Python interface (file:line, relative to tf_geometric/ of the reference, CrawlScript/tf_geometric) whose arithmetic it
 * replaces; INTEGRATION.md shows the ctypes binding a tf_geometric maintainer would add at each of those sites.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch's allocator in this repo); the library never
 *     allocates or frees device memory: scratch space is queried (`*_workspace_bytes`) and passed in;
 *   - `stream` is a cudaStream_t cast to void* (NULL = default stream); all launches are asynchronous, except
 *     tfgk_csr_build which synchronises `stream` once to report out-of-range node ids;
 *   - outputs are fully overwritten; no global mutable state (calls on distinct streams are thread-safe);
 *   - return value 0 = TFGK_OK, otherwise an error code with a thread-local message in tfgk_last_error();
 *   - float data is IEEE fp32, node ids int32, edge offsets (rowptr) int64; one call handles < 2^31 edges;
 *   - "row" = aggregation target (destination), "col" = neighbour (source): nn/kernel/map_reduce.py:60-70.
 */
#ifndef TFGK_H_
#define TFGK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Raised when an existing entry point, struct layout or enum value changes meaning.  New symbols, new structs and new
 * enum values leave a binding written against an earlier header working, so they keep the version (the bf16 and fp8
 * entries were added under 7). */
#define TFGK_ABI_VERSION 7

enum tfgk_status {
    TFGK_OK = 0,
    TFGK_ERR_INVALID_ARGUMENT = 1,
    TFGK_ERR_CUDA = 2,
    TFGK_ERR_WORKSPACE = 3,
    TFGK_ERR_UNSUPPORTED = 4,
    TFGK_ERR_INDEX_OUT_OF_RANGE = 5
};

enum tfgk_reduce { TFGK_REDUCE_SUM = 0, TFGK_REDUCE_MEAN = 1, TFGK_REDUCE_MAX = 2 };
enum tfgk_act { TFGK_ACT_NONE = 0, TFGK_ACT_RELU = 1 };
enum tfgk_deg_power { TFGK_POW_INV_SQRT = 0, TFGK_POW_INV = 1 };
enum tfgk_heads_mode { TFGK_HEADS_SPLIT = 0, TFGK_HEADS_BROADCAST = 1, TFGK_HEADS_REDUCE = 2 };
enum tfgk_edge_flag { TFGK_FLAG_ALL = 0, TFGK_FLAG_UPPER = 1, TFGK_FLAG_MAPPED = 2 };
enum tfgk_bernoulli { TFGK_BERNOULLI_NONE = 0, TFGK_BERNOULLI_DROPOUT = 1, TFGK_BERNOULLI_KEEP = 2 };
enum tfgk_sample_padding { TFGK_SAMPLE_NO_PADDING = 0, TFGK_SAMPLE_PADDING = 1, TFGK_SAMPLE_HEAD = 2 };
enum tfgk_gcn_norm { TFGK_GCN_NORM_BOTH = 0, TFGK_GCN_NORM_LEFT = 1, TFGK_GCN_NORM_RIGHT = 2 };
enum tfgk_gcn_loop { TFGK_GCN_LOOP_NONE = 0, TFGK_GCN_LOOP_NORMED = 1, TFGK_GCN_LOOP_FILL = 2 };
/* element type of a bf16-capable buffer; bf16 and fp16 data are passed as their 16-bit patterns (uint16_t), fp8 data as
 * bytes.  TFGK_DTYPE_F16 (IEEE binary16) is taken only by the 16-bit host-table gathers. */
enum tfgk_dtype { TFGK_DTYPE_F32 = 0, TFGK_DTYPE_BF16 = 1, TFGK_DTYPE_FP8_E4M3 = 2, TFGK_DTYPE_F16 = 3 };

/* fp8 message rows (inference storage of the rows GCN and GAT gather along edges):
 *   element   OCP e4m3fn bytes (torch.float8_e4m3fn): max 448, no infinities, NaN = 0x7F / 0xFF;
 *   scale     one int8 exponent k per row and group of 128 columns (group g = columns [128 g, 128 g + 128)), in a separate
 *             [N, ceil(D / 128)] array (row stride ceil(D / 128) unless stated otherwise);
 *   exponent  m = max |x| over the group's finite entries; k = the smallest integer with m 2^-k <= 448, clamped to
 *             [-126, 127]; k = 0 when m = 0 or the group has no finite entry;
 *   value     q = RNE-to-e4m3fn(x 2^-k) (never saturates); +-inf and NaN are stored as NaN with their sign; -0.0 stays;
 *   dequant   x^ = float(q) 2^k, exact in fp32 (except that a value rounded up past FLT_MAX, possible only within 2^-4
 *             of FLT_MAX, becomes inf), so "the fp32 kernel over x^" is a bit-level reference;
 *   rows      16-byte aligned (ld % 16 == 0) with zeroed pad columns.
 * |x^ - x| <= max(2^-4 |x|, 2^(k-10)) per element. */

int tfgk_version(void);
const char *tfgk_last_error(void);
/* SM count and compute capability of the current device. */
int tfgk_device_info(int *sm_count, int *cc_major, int *cc_minor);

/* ---- integer edge preprocessing (bit-exact) ------------------------------------------------------------------ */

/* utils/graph_utils.py:350-366 add_self_loop_edge: out[2,E+N] = concat(edge_index[2,E], [[0..N-1],[0..N-1]]). */
int tfgk_self_loops_i32(const int32_t *edge_index, int64_t E, int32_t N, int32_t *out, void *stream);
/* same function, weight half: out[E+N] = concat(w (ones if NULL), fill). */
int tfgk_self_loop_weights_f32(const float *w, int64_t E, int32_t N, float fill, float *out, void *stream);
/* nn/kernel/segment.py:36-40 segment_count: int32 histogram of ids (negative ids dropped like
 * tf.math.unsorted_segment_sum; ids >= N are an error reported by tfgk_csr_build, ignored here). */
int tfgk_segment_count_i32(const int32_t *ids, int64_t E, int32_t N, int32_t *out, void *stream);

/* Destination-sorted CSR of a COO edge list: a STABLE sort by row, so that a left-to-right walk of a row
 * visits its edges in input order (= tf.math.unsorted_segment_sum's CPU summation order).
 *   rowptr[N+1] int64, col_sorted[E] = col[perm], perm[E] (position in the input list).
 * Replaces the implicit scatter of tf.math.unsorted_segment_* (nn/kernel/map_reduce.py:16,28,41) and of
 * tf_sparse.SparseMatrix.matmul (nn/conv/gcn.py:280, gat.py:89, appnp.py:86). */
int tfgk_csr_workspace_bytes(int64_t E, int32_t N, size_t *out_bytes);
int tfgk_csr_build(const int32_t *row, const int32_t *col, int64_t E, int32_t N_rows, int32_t N_cols,
                   int64_t *rowptr, int32_t *col_sorted, int32_t *perm,
                   void *workspace, size_t workspace_bytes, void *stream);
/* The same CSR without the id check, so without its synchronisation: for edge lists whose ids are in range by
 * construction (a sampled block's transposed structure).  An id outside the range is undefined behaviour. */
int tfgk_csr_build_in_range(const int32_t *row, const int32_t *col, int64_t E, int32_t N_rows, int32_t N_cols,
                            int64_t *rowptr, int32_t *col_sorted, int32_t *perm,
                            void *workspace, size_t workspace_bytes, void *stream);

/* utils/graph_utils.py:67-125 merge_duplicated_edge, index half: duplicates of (row, col) collapse onto their FIRST occurrence
 * (tf.unique order on the hash num_nodes*row + col, num_nodes = N).  unique_index is [2, E] row-major with the first
 * *n_unique_host columns valid; unique_of_edge[e] = column of edge e's representative (the segment id the edge properties
 * are merged with).  Bit-exact; synchronises `stream`. */
int tfgk_edge_unique_workspace_bytes(int64_t E, int32_t N, size_t *out_bytes);
int tfgk_edge_unique(const int32_t *row, const int32_t *col, int64_t E, int32_t N, int32_t *unique_index,
                     int32_t *unique_of_edge, int32_t *n_unique_host, void *workspace, size_t workspace_bytes, void *stream);

/* utils/graph_utils.py:181-190 convert_edge_to_directed, index half: out[2, out_ld] = upper edges followed by the mirrored
 * non-self-loop upper edges (in order); lower_src[j] = column of the upper edge mirrored into column U + j (to copy its
 * properties).  upper_index is [2, ld] row-major with U valid columns.  Bit-exact; synchronises `stream`. */
int tfgk_directed_workspace_bytes(int64_t U, size_t *out_bytes);
int tfgk_directed_edges(const int32_t *upper_index, int64_t U, int64_t ld, int32_t *out, int64_t out_ld,
                        int32_t *lower_src, int32_t *n_lower_host, void *workspace, size_t workspace_bytes, void *stream);

/* Work plan of a CSR for the streaming kernels (K1, K3): destination rows are grouped into tasks of at most
 * `rows_per_task` consecutive rows (one warp each), and every row with more than `hub_threshold` edges is cut into slices
 * of `chunk` edges that are reduced by separate warps into `scratch` and merged by a fix-up kernel in slice order
 * (deterministic; a hub row is therefore summed slice by slice instead of strictly left to right).  Without hub rows the
 * kernels need no plan (pass NULL).  The reference has no counterpart: tf.math.unsorted_segment_sum is one sequential loop. */
typedef struct tfgk_plan {
    int32_t n_tasks, n_hubs, n_slots, chunk;
    const int32_t *task_row;    /* [n_tasks] first destination row                                   */
    const int32_t *task_nrows;  /* [n_tasks] number of rows (1 for a hub slice)                      */
    const int64_t *task_e0;     /* [n_tasks] first CSR edge                                          */
    const int64_t *task_e1;     /* [n_tasks] one past the last CSR edge                              */
    const int32_t *task_slot;   /* [n_tasks] -1: whole rows; >= 0: hub slice -> partial in scratch   */
    const int32_t *hub_row;     /* [n_hubs]                                                          */
    const int32_t *hub_slot0;   /* [n_hubs] first scratch slot of the row                            */
    const int32_t *hub_nslots;  /* [n_hubs]                                                          */
    float *scratch;             /* K1: n_slots * D floats;  K3: n_slots * (H*dv + 64) floats         */
    size_t scratch_bytes;
} tfgk_plan;

/* Upper bounds for the plan arrays of a CSR with E edges and N rows. */
int tfgk_plan_capacity(int64_t E, int32_t N, int32_t hub_threshold, int32_t chunk, int32_t rows_per_task,
                       int64_t *max_tasks, int64_t *max_hubs);
int tfgk_plan_workspace_bytes(int32_t N, size_t *out_bytes);
/* Fills the arrays; counts_host[3] = {n_tasks, n_hubs, n_slots} (synchronises `stream` once). */
int tfgk_plan_build(const int64_t *rowptr, int32_t N, int32_t hub_threshold, int32_t chunk, int32_t rows_per_task,
                    int32_t *task_row, int32_t *task_nrows, int64_t *task_e0, int64_t *task_e1, int32_t *task_slot,
                    int32_t *hub_row, int32_t *hub_slot0, int32_t *hub_nslots, int64_t cap_tasks, int64_t cap_hubs,
                    int32_t *counts_host, void *workspace, size_t workspace_bytes, void *stream);

/* dst[i*width + j] = src[perm[i]*width + j]   (COO order -> CSR order) and the inverse scatter. */
int tfgk_permute_f32(const float *src, const int32_t *perm, int64_t E, int32_t width, float *dst, void *stream);
int tfgk_unpermute_f32(const float *src, const int32_t *perm, int64_t E, int32_t width, float *dst, void *stream);

/* ---- feature tables in host memory (utils.HostFeatureTable) --------------------------------------------------------
 * _register   page-locks [ptr, ptr + bytes) in place (cudaHostRegister, portable | mapped) and returns the address the
 *             device reads it through.  A range that overlaps a registered one fails (one registration per range).
 * _unregister waits for the current device's work (so no gather in flight reads the range), then releases a
 *             registration made by _register (ptr is the same host address).
 * Both return TFGK_ERR_CUDA with CUDA's message on failure and leave no CUDA error pending. */
int tfgk_host_register(void *ptr, size_t bytes, void **dev_ptr);
int tfgk_host_unregister(void *ptr);
/* out[i*ldo + j] = table[index[i]*ld + j] for j < F, where `table` is host memory the device reads over the host link
 * (a mapped pointer from tfgk_host_register, or pinned memory under unified addressing).  An id outside [0, n_rows)
 * writes a row of NaN and reads nothing, so a bad id never touches memory past the registered range.  One warp per
 * output row, grid-strided over 16 warps per SM; 16-byte accesses when F, ld, ldo and both base pointers allow them,
 * 4-byte accesses otherwise.  Asynchronous.  Bytes over the link: n * F * 4. */
int tfgk_gather_rows_mapped_f32(const float *table, int64_t ld, int64_t n_rows, int32_t F, const int32_t *index,
                                int64_t n, float *out, int64_t ldo, void *stream);
/* The same gather with a device cache of some rows (HostFeatureTable(x, device_rows=...)): slot is an int32 [n_rows]
 * device map, and slot[r] = s >= 0 means row r is cache[s*ldc + j] for j < F (device memory, ldc >= F), read instead of
 * the host row; slot[r] = -1 reads the host table.  An id outside [0, n_rows) writes a row of NaN and reads neither the
 * map nor either table.  One launch serves hits and misses; 16-byte accesses need ldc % 4 == 0 and a 16-byte-aligned
 * cache as well.  Asynchronous.  Bytes: misses * F * 4 over the host link, hits * F * 4 from device memory. */
int tfgk_gather_rows_cached_f32(const float *table, int64_t ld, int64_t n_rows, int32_t F, const float *cache,
                                int64_t ldc, const int32_t *slot, const int32_t *index, int64_t n, float *out,
                                int64_t ldo, void *stream);
/* The two gathers above from a 16-bit table: dtype is TFGK_DTYPE_BF16 or TFGK_DTYPE_F16, and ld, ldc and ldo count
 * elements.  The rows are those of the float32 entries, each element widened to float32 exactly (bf16 by a 16-bit shift,
 * fp16 by the hardware conversion), so out is the gather of the widened table bit for bit; an id outside [0, n_rows)
 * writes a float32 NaN row and reads nothing.  The cache holds rows in the table's dtype.
 * out_dtype (mapped entry): TFGK_DTYPE_F32, or the table's dtype to copy the 16-bit patterns unchanged (NaN payloads
 * included; a bad id then writes the 16-bit NaN 0x7FC0 / 0x7E00), which fills a 16-bit device cache without a float32
 * staging buffer.  Any other dtype or out_dtype: TFGK_ERR_INVALID_ARGUMENT.
 * Loads carry 8, 4, 2 or 1 elements (16, 8, 4 or 2 bytes): the widest that F, the strides and the base pointers allow
 * (F = 100 rows at 8-byte alignment take 8 bytes; F = 104 at 16-byte alignment take 16).  Asynchronous, no host
 * synchronisation.  Bytes over the link: misses * F * 2. */
int tfgk_gather_rows_mapped_16(const uint16_t *table, int32_t dtype, int64_t ld, int64_t n_rows, int32_t F,
                               const int32_t *index, int64_t n, void *out, int32_t out_dtype, int64_t ldo,
                               void *stream);
int tfgk_gather_rows_cached_16(const uint16_t *table, int32_t dtype, int64_t ld, int64_t n_rows, int32_t F,
                               const uint16_t *cache, int64_t ldc, const int32_t *slot, const int32_t *index,
                               int64_t n, float *out, int64_t ldo, void *stream);

/* ---- a CSR built from an edge list in host memory (utils.HostNeighborSampler) -----------------------------------------
 * row, col [E] int32 (and w [E] float32) are device-readable pointers to page-locked host memory (tfgk_host_register);
 * E may be 2^31 or more.  Every entry streams them in edge order, 16 bytes per load where the array is 16-byte aligned.
 * _id_range   range_host[4] = {min row, max row, min col, max col}, from one pass over both arrays (E > 0).  The
 *             workspace is at least 16 bytes of device memory.  Synchronises `stream`.
 * _rowptr     rowptr int64 [n_rows + 1] = exclusive scan of the per-row edge counts; rows outside [0, n_rows) are not
 *             counted.  Equal to tfgk_csr_build's rowptr of the same edges.  Counts are int64, so a row of 2^31 edges
 *             or more is counted exactly (the caller refuses it).  Asynchronous.
 * _select_rows the edges with r0 <= row < r1, in edge order: out_row = row - r0, out_col = col, out_w = w (w may be NULL:
 *             out_w is then untouched), at most cap < 2^31 of them (the caller knows the count from rowptr).  A stable
 *             compaction in tiles of 1024 edges: int offsets within a tile, int64 tile offsets.  Sorting its output with
 *             tfgk_csr_build_in_range(out_row, out_col, count, r1 - r0, ...) gives rows [r0, r1) of the CSR of the whole
 *             edge list (the selection keeps edge order and the sort is stable).  Asynchronous. */
int tfgk_mapped_id_range_i32(const int32_t *row, const int32_t *col, int64_t E, int32_t *range_host, void *workspace,
                             size_t workspace_bytes, void *stream);
int tfgk_mapped_rowptr_workspace_bytes(int32_t n_rows, size_t *out_bytes);
int tfgk_mapped_rowptr_i32(const int32_t *row, int64_t E, int32_t n_rows, int64_t *rowptr, void *workspace,
                           size_t workspace_bytes, void *stream);
int tfgk_mapped_select_rows_workspace_bytes(int64_t E, size_t *out_bytes);
int tfgk_mapped_select_rows_i32(const int32_t *row, const int32_t *col, const float *w, int64_t E, int32_t r0,
                                int32_t r1, int32_t *out_row, int32_t *out_col, float *out_w, int64_t cap,
                                void *workspace, size_t workspace_bytes, void *stream);

/* ---- GCN normalisation (nn/conv/gcn.py:32-130, utils/graph_utils.py:914-943) -------------------------------- */

/* SparseMatrix.segment_sum(axis=-1) on CSR-ordered values: out[r] = sum of w[rowptr[r]..rowptr[r+1]) in order. */
int tfgk_csr_rowsum_f32(const int64_t *rowptr, const float *w_csr, int32_t N, float *out, void *stream);
/* tf.pow(deg, -0.5 | -1) followed by _remove_inf_and_nan (gcn.py:23-29,81-82,104-105,114-115). */
int tfgk_deg_inv_f32(const float *deg, int32_t N, int power, float *out, void *stream);
/* (diags(dl) @ A) @ diags(dr) on the value array, COO order: out[e] = (dl[row[e]] * w[e]) * dr[col[e]];
 * dl or dr may be NULL (gcn.py:94,109,119). */
int tfgk_scale_edges_f32(const int32_t *row, const int32_t *col, const float *w, int64_t E,
                         const float *dl, const float *dr, float *out, void *stream);

/* ---- K1: gather - edge-apply - segment-reduce ---------------------------------------------------------------- */

/* out[r,:] = epilogue( REDUCE_{e in row r} ( w[e] * h[col[e],:] ) )            r in [0, n_dst)
 *   reduce = SUM  : tf.math.unsorted_segment_sum  (map_reduce.py:15-16), tf_sparse matmul (gcn.py:280)
 *            MEAN : tf.math.unsorted_segment_mean (map_reduce.py:27-28; graph_sage.py:41), empty row -> 0
 *            MAX  : tf.math.unsorted_segment_max  (map_reduce.py:38-42), empty row -> -FLT_MAX
 *   w NULL = identity_mapper (map_reduce.py:7-8), else gcn_mapper (gcn.py:221-222); CSR order.
 *   epilogue: v = agg*alpha + addend*beta (addend NULL -> v = agg; APPNP appnp.py:86-87, sum_updater
 *   map_reduce.py:19-20), then + bias[D] (NULL ok), then activation  (gcn.py:284-288).
 * Deterministic (no atomics); per-row accumulation is sequential in CSR order, except for the hub rows of `plan`
 * (NULL = none), which are accumulated slice by slice. */
int tfgk_spmm_f32(const int64_t *rowptr, const int32_t *col, const float *w,
                  const float *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                  float alpha, const float *addend, int64_t ld_addend, float beta,
                  const float *bias, int act,
                  float *out, int64_t ldo, const tfgk_plan *plan, void *stream);
/* Aggregate, then project (GCN inference when the input is narrower than the layer):
 *   out[r, :] = act( (SUM_{e in row r} w[e] * x[col[e], :]) . W + bias )          r in [0, n_dst)
 * x [n, F] fp32 with 16-byte aligned rows and ldx % 4 == 0, W [F, U] row-major, bias [U] or NULL, act NONE or RELU;
 * 4 <= F < U <= 128 and F % 4 == 0, anything else returns TFGK_ERR_UNSUPPORTED.  The aggregate of each row (never
 * stored) is bit-identical to tfgk_spmm_f32's SUM over x with the same plan, which it takes where tfgk_spmm_f32 does
 * (F >= 32; the plan's hub scratch takes F floats per slot).  Each output is then an fmaf chain over k = 0 .. F-1 from
 * +0, then + bias[c] (rounded), then the activation.  Algorithmic bytes: E*(4*F + 4 [+4 weighted]) + N*(4*U + 8). */
int tfgk_spmm_proj_f32(const int64_t *rowptr, const int32_t *col, const float *w,
                       const float *x, int64_t ldx, int32_t n_dst, int32_t F, const float *W, int32_t U,
                       const float *bias, int act, float *out, int64_t ldo, const tfgk_plan *plan, void *stream);
/* The same with bf16 rows h (w, addend, bias, the accumulators and out stay fp32).  Bf16 -> fp32 widening is exact, and
 * the kernels widen each element and run the fp32 arithmetic in the same order with the same plan, so the output is
 * bit-identical to tfgk_spmm_f32 over the widened table with the same leading dimension and alignment in elements.  Rows
 * with D % 8 == 0, 32 <= D <= 256 and 16-byte aligned rows take the TMA ring (2 D bytes per row); D % 4 == 0 up to 512
 * with 8-byte aligned rows a cp.async ring; both use the plan, as tfgk_spmm_f32 does for 16-byte aligned fp32 rows.  Any
 * other D or leading dimension takes a scalar path without the plan (hub rows summed strictly in order), as in fp32: a
 * dense widened copy of such a view would take the plan, so callers comparing against one pass a dense copy of h
 * (ops.spmm does when the plan has hub rows).  Algorithmic bytes: E*(2*D + 4 [+4 weighted]) + N*(4*D + 8). */
int tfgk_spmm_bf16(const int64_t *rowptr, const int32_t *col, const float *w,
                   const uint16_t *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                   float alpha, const float *addend, int64_t ld_addend, float beta,
                   const float *bias, int act,
                   float *out, int64_t ldo, const tfgk_plan *plan, void *stream);
/* tfgk_spmm_bf16 that stores its fp32 result (after alpha / addend / bias / activation) in `out` and/or, rounded to
 * nearest even, in the bf16 table `out_bf16` ([n_dst, D], leading dimension ldob): either may be NULL, not both.  `out`
 * is bit-identical to what tfgk_spmm_bf16 writes with the same arguments, and out_bf16 to tfgk_round_bf16 of it (inf and
 * NaN stay inf and NaN, finite values beyond the bf16 range become inf); with out == NULL, to tfgk_spmm_bf16 into a dense
 * fp32 out.  A multi-hop chain thus writes its intermediate hops as 2 bytes per element, ready for the next gather.
 * Padded tables: rows 16-byte aligned with ldh % 8 == 0 and ldh >= D rounded up to 8 (8-byte aligned, ldh >= D rounded
 * up to 4) may be read with their pad columns, so that the TMA (cp.async) ring runs for any D; pad columns are computed
 * and never stored, and do not interact with the first D.  A plan is used exactly where tfgk_spmm_bf16 uses it.  h and
 * out_bf16 must be 2-byte aligned and out 4-byte aligned.  Algorithmic bytes: E*(2*D + 4 [+4 weighted]) + N*(4*D + 8)
 * with both outputs, N*(2*D + 8) for the output side of a bf16-only store. */
int tfgk_spmm_bf16_dual(const int64_t *rowptr, const int32_t *col, const float *w,
                        const uint16_t *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                        float alpha, const float *addend, int64_t ld_addend, float beta,
                        const float *bias, int act,
                        float *out, int64_t ldo, uint16_t *out_bf16, int64_t ldob,
                        const tfgk_plan *plan, void *stream);

/* The same with fp8 rows h and exponents h_exp ([N, ceil(D / 128)] int8, 2-byte aligned when D > 128); w, addend, bias,
 * the accumulators and out stay fp32.  Each element is widened and multiplied by 2^k of its row's group, then the fp32
 * arithmetic runs in the same order; the plan is used exactly where tfgk_spmm_f32 uses it over the dequantised table with
 * the same leading dimension, and rows without the plan are summed strictly in CSR order, so the output is bit-identical
 * to tfgk_spmm_f32 over x^ wherever both use the plan or neither does.  Rows 16-byte aligned with ldh % 16 == 0 and
 * ldh >= D rounded up to 16, up to 256 columns, take the TMA ring (read with their pad columns, which are computed and
 * never stored; the plan's scratch holds D rounded up to 16 floats per slot); every other shape takes a scalar path
 * without the plan (a hub row of a table wider than 256 columns is then summed in order, unlike in fp32).
 * Algorithmic bytes: E*(D + 1 [+1 for D > 128] + 4 [+4 weighted]) + N*(4*D + 8). */
int tfgk_spmm_fp8(const int64_t *rowptr, const int32_t *col, const float *w,
                  const uint8_t *h, int64_t ldh, const int8_t *h_exp, int32_t n_dst, int32_t D, int reduce,
                  float alpha, const float *addend, int64_t ld_addend, float beta,
                  const float *bias, int act,
                  float *out, int64_t ldo, const tfgk_plan *plan, void *stream);

/* ---- K3: edge softmax and fused GAT ------------------------------------------------------------------------- */

/* nn/kernel/segment.py:26-33 segment_softmax over CSR segments, H interleaved score columns:
 * score/out are [E, H] row-major in CSR order; per (segment, h): exp(s - max) / (sum + 1e-8). */
int tfgk_segment_softmax_f32(const int64_t *rowptr, const float *score, int32_t n_seg, int32_t H,
                             float *out, void *stream);

/* nn/conv/gat.py:73-114 fused: per destination r and head h
 *     s_e = <Q[r,h,:], K[col_e,h,:]> / scale  (scale = sqrt(dqk), gat.py:78-79) ;  a_e = softmax_e(s_e)  (gat.py:83-84,
 *     segment.py:26-33) ;  out[r,h,:] = sum_e a_e V[col_e,h,:]  (gat.py:87-89)
 * Q,K: [N, H*dqk]; V: [N, H*dv]. split_value_heads=1: out[N, H*dv] heads concatenated (gat.py:112);
 * 0: out[N, dv] = mean over heads (gat.py:114).  Then + bias, activation (gat.py:116-120).
 * att: [E, H] CSR order, REQUIRED scratch (raw scores, then exp(s - max)); with write_att != 0 it holds the
 * attention coefficients a_e on return.  The CSR must already contain the self loops gat.py:43 appends. */
int tfgk_gat_fused_f32(const int64_t *rowptr, const int32_t *col,
                       const float *Q, int64_t ldq, const float *K, int64_t ldk, const float *V, int64_t ldv,
                       int32_t N, int32_t H, int32_t dqk, int32_t dv, float scale, int split_value_heads,
                       const float *bias, int act, float *att, int write_att, float *out, int64_t ldo,
                       const tfgk_plan *plan, void *stream);
/* The same with bf16 K and V (Q, bias, att and out fp32), inference only: write_att != 0 returns TFGK_ERR_UNSUPPORTED.
 * Heads concatenated with dqk == dv, H * dqk <= 128 and V == K + H*dqk in one [N, 2A] buffer (ldk == ldv, a multiple of 8,
 * 16-byte aligned) take the TMA ring, one bulk copy of 4A bytes per neighbour; other shapes with heads concatenated,
 * dqk == dv and A <= 512 (8-byte aligned rows) the register-staged single-pass kernel.  Both give the output of
 * tfgk_gat_fused_f32 over the widened K and V where it runs the same kernel.  Every other shape (averaged heads, dqk != dv)
 * takes the two-pass generic kernel, which needs att ([E, H] scratch).  Only the TMA ring reads K and V faster than fp32 does;
 * the single-pass kernel with bf16 rows is latency-bound and slower than with fp32 rows (DESIGN.md section 4). */
int tfgk_gat_fused_bf16(const int64_t *rowptr, const int32_t *col,
                        const float *Q, int64_t ldq, const uint16_t *K, int64_t ldk, const uint16_t *V, int64_t ldv,
                        int32_t N, int32_t H, int32_t dqk, int32_t dv, float scale, int split_value_heads,
                        const float *bias, int act, float *att, int write_att, float *out, int64_t ldo,
                        const tfgk_plan *plan, void *stream);
/* The same with fp8 K | V in ONE [N, 2A]-byte buffer KV (K in bytes [0, A), V in [A, 2A) of a row; ldkv % 16 == 0,
 * 16-byte aligned) with kv_exp [N, 2] int8 (K group, V group; 2-byte aligned), inference only: heads concatenated,
 * dqk == dv, H a power of two, dqk / 4 a power of two, A = H * dqk <= 128.  Q, bias and out are fp32, 16-byte aligned.
 * The TMA ring copies 2A bytes (rounded up to 16) per neighbour and reads its two exponents; each element is widened
 * and scaled by 2^k, then the fp32 ring's arithmetic runs with its lane mapping, so the output is bit-identical to
 * tfgk_gat_fused_f32 over Q, K^, V^ wherever that takes its TMA ring.  Every other shape returns TFGK_ERR_UNSUPPORTED (no
 * attention coefficients are returned).  The plan's hub scratch takes A + 64 floats per slot.
 * Algorithmic bytes: E*(2A + 2 + 4) + N*(8A + 8). */
int tfgk_gat_fused_fp8(const int64_t *rowptr, const int32_t *col, const float *Q, int64_t ldq,
                       const uint8_t *KV, int64_t ldkv, const int8_t *kv_exp, int32_t N, int32_t H, int32_t dqk,
                       float scale, const float *bias, int act, float *out, int64_t ldo,
                       const tfgk_plan *plan, void *stream);
/* Packed keys: a table of one slot of ldt floats per node (ldt a multiple of 16, at least 2A + 4; A = H * dqk <= 128):
 *     [0, A) V[n] | [A, A + 4) zero mask, bit c set <=> the bits of K[n, c] are not 0x00000000 |
 *     [A + 4, ...) the entries of K[n] whose bit is set, in column order, zero-padded to a multiple of four floats
 * and ksize[n] = 16-byte units of the slot a neighbour's copy reads, (A + 4 + padded count) / 4.  The caller writes V into the
 * slots; tfgk_gat_pack_keys_f32 writes the mask, the packed keys and ksize from K [N, A] (16-byte aligned rows). */
int tfgk_gat_pack_keys_f32(const float *K, int64_t ldk, int32_t N, int32_t A, float *table, int64_t ldt, uint8_t *ksize,
                           void *stream);
/* tfgk_gat_fused_f32 with heads concatenated and dqk == dv over a packed table: the TMA ring copies 16 * ksize[c] bytes per
 * neighbour c instead of 8A and rebuilds K[c] from the mask.  Only the bit pattern 0x00000000 is left out of the table, so
 * the output is bit-identical to tfgk_gat_fused_f32 over the same Q, K, V (for the shapes that take its TMA ring) for any
 * K.  H a power of two <= 32, dqk / 4 a power of two, A <= 128, 16-byte aligned Q, out, bias and table rows; other shapes
 * return TFGK_ERR_UNSUPPORTED.  The plan's hub scratch takes A + 64 floats per slot, as for tfgk_gat_fused_f32. */
int tfgk_gat_fused_packed_f32(const int64_t *rowptr, const int32_t *col, const float *Q, int64_t ldq,
                              const float *table, int64_t ldt, const uint8_t *ksize, int32_t N, int32_t H, int32_t dqk,
                              float scale, const float *bias, int act, float *out, int64_t ldo,
                              const tfgk_plan *plan, void *stream);

/* ---- K4: dense projections (gcn.py:272, gat.py:52,61,70, graph_sage.py:43-44, appnp.py:69) ------------------- */

/* C[M,N] = act( op(A) @ op(B) + bias[N] + beta * C ),  op = transpose when the flag is set (backward passes).
 * fp32 in/out. workspace is needed only for split-K (tall-skinny reductions); NULL/0 disables split-K. */
int tfgk_gemm_workspace_bytes(int32_t M, int32_t N, int32_t K, size_t *out_bytes);
int tfgk_gemm_f32(const float *A, int64_t lda, int transA, const float *B, int64_t ldb, int transB,
                  const float *bias, int act, float beta, int32_t M, int32_t N, int32_t K,
                  float *C, int64_t ldc, void *workspace, size_t workspace_bytes, void *stream);

/* Several projections of the same input in ONE launch (round 2): for every column block b < n_blocks
 *   C_b[M, ncols_b] = act_b( A[M, K] @ B_b[K, ncols_b] + bias_b ),   ncols_b <= 128, n_blocks <= 4,
 * e.g. the three projections of gat.py:52,61,70 (Q | K | V) or gcn.py:272 next to them; A is read from HBM once.
 * Same 3xTF32 wgmma arithmetic as tfgk_gemm_f32's tensor-core path (bit-identical results).
 * A may live in n_parts <= 8 row blocks of part_rows rows each (a multiple of 128 when n_parts > 1), part i at
 * A_parts[i]: with the other ranks' buffers mapped through tfgk_peer_open this is the fused all-gather -> GEMM of the
 * partitioned path (rows are pulled over NVLink tile by tile while earlier tiles are multiplied); the walk starts at
 * part first_part so that concurrent ranks read from different peers.  max_ctas > 0 bounds the grid (to share the GPU
 * with a kernel on another stream).  Returns TFGK_ERR_UNSUPPORTED when the shape does not qualify (K > 184, where W no
 * longer fits in shared memory; lda not a multiple of 4 or A not 16-byte aligned; ncols > 128): the caller then uses
 * tfgk_gemm_f32 per block. */
typedef struct tfgk_proj_block {
    const float *B; int64_t ldb;       /* [K, ncols] row-major weights ([ncols, K] row-major when transB != 0) */
    int32_t ncols;
    int32_t transB;                    /* 0: C = A @ B;  1: C = A @ B^T  (the dX = dY W^T products of the backward pass) */
    const float *bias;                 /* [ncols] or NULL */
    int act;                           /* tfgk_act */
    float *C; int64_t ldc;             /* [M, ncols] output (may be a column slice of a wider buffer) */
} tfgk_proj_block;
int tfgk_gemm_proj_f32(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                       int32_t M, int32_t K, const tfgk_proj_block *blocks, int32_t n_blocks,
                       int32_t first_part, int32_t max_ctas, void *stream);
/* tfgk_gemm_proj_f32 with a per-block output type: a TFGK_DTYPE_BF16 block stores the fp32 result of its epilogue
 * (bias, activation) rounded to nearest even, bit-identical to rounding tfgk_gemm_proj_f32's output (inf and NaN stay
 * inf and NaN, finite values beyond the bf16 range become inf).  GAT's fp32 Q and bf16 K | V thus still come from one
 * launch that reads x once.  Only n_parts == 1 (TFGK_ERR_UNSUPPORTED otherwise); the other shape limits are those of
 * tfgk_gemm_proj_f32, and tfgk_round_bf16 rounds the output of tfgk_gemm_f32 for the shapes it refuses. */
typedef struct tfgk_proj_block_out {
    const float *B; int64_t ldb;       /* as in tfgk_proj_block */
    int32_t ncols;
    int32_t transB;
    const float *bias;
    int act;
    void *C; int64_t ldc;              /* [M, ncols] output of type c_dtype (may be a column slice) */
    int32_t c_dtype;                   /* tfgk_dtype */
} tfgk_proj_block_out;
int tfgk_gemm_proj_mixed(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                         int32_t M, int32_t K, const tfgk_proj_block_out *blocks, int32_t n_blocks,
                         int32_t first_part, int32_t max_ctas, void *stream);
/* dst[r, c] = bf16(src[r, c]) rounded to nearest even, r < rows, c < cols. */
int tfgk_round_bf16(const float *src, int64_t lds, int32_t rows, int32_t cols, uint16_t *dst, int64_t ldd, void *stream);
/* tfgk_gemm_proj_mixed with fp8 blocks as well: a TFGK_DTYPE_FP8_E4M3 block stores the fp32 result of its epilogue (bias,
 * activation) in the fp8 format above, one exponent per row (a block is at most 128 columns: one group) written to
 * E[row * lde] (e.g. column g of a [N, G] exponent array).  The bytes and exponents are those of tfgk_quantize_fp8 over
 * tfgk_gemm_proj_f32's output.  In the m64n128 accumulator layout a row's columns sit in the four threads of a quad: two
 * xor-shuffles give the row maximum, each thread scales its values and packs pairs with cvt.rn.satfinite.e4m3x2.f32.  GAT's
 * fp32 Q and fp8 K | V thus come from one launch that reads x once.  Only n_parts == 1; other limits as tfgk_gemm_proj_f32. */
typedef struct tfgk_proj_block_fp8 {
    const float *B; int64_t ldb;       /* as in tfgk_proj_block */
    int32_t ncols;
    int32_t transB;
    const float *bias;
    int act;
    void *C; int64_t ldc;              /* [M, ncols] output of type c_dtype (may be a column slice) */
    int32_t c_dtype;                   /* tfgk_dtype */
    int8_t *E; int64_t lde;            /* TFGK_DTYPE_FP8_E4M3 only: the row exponents, E[row * lde] */
} tfgk_proj_block_fp8;
int tfgk_gemm_proj_fp8(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                       int32_t M, int32_t K, const tfgk_proj_block_fp8 *blocks, int32_t n_blocks,
                       int32_t first_part, int32_t max_ctas, void *stream);
/* dst = the fp8 format above of src [rows, cols] (leading dimension lds), exps[r * lde + g] for group g < ceil(cols / 128):
 * for tables tfgk_gemm_proj_fp8 refuses (K > 184), the same bytes it would write from the same fp32 values.  Only the
 * first cols bytes of a row are written. */
int tfgk_quantize_fp8(const float *src, int64_t lds, int32_t rows, int32_t cols, uint8_t *dst, int64_t ldd,
                      int8_t *exps, int64_t lde, void *stream);

/* ---- K5: peer memory for the partitioned path (SURVEY.md 8e) ---------------------------------------------------
 * The ONE exception to "the library never allocates": buffers that other ranks on the same node read over NVLink
 * must come from cudaMalloc so that they can be exported with CUDA IPC (PyTorch's caching allocator sub-allocates).
 *   tfgk_peer_alloc / _free    device buffer on the current device (zero-initialised)
 *   tfgk_peer_export           64-byte IPC handle of a buffer from tfgk_peer_alloc (sent to the other ranks by the host)
 *   tfgk_peer_open / _close    map another process's buffer into this process (peer access enabled lazily)
 *   tfgk_peer_barrier          device-side barrier over NVLink on `stream`: thread j stores `value` into slot `rank` of
 *                              rank j's flag array (flags[j], uint32[world], from tfgk_peer_open) after a system-scope
 *                              fence, then waits until slot j of the local array reaches `value` (values grow by one per
 *                              barrier).  Traps instead of hanging if a peer does not arrive within timeout_ms.
 * The reference has no counterpart (its multi-GPU demos replicate the graph, demo/demo_distributed_gcn.py:37-57). */
#define TFGK_PEER_HANDLE_BYTES 64
int tfgk_peer_alloc(size_t bytes, void **ptr);
int tfgk_peer_free(void *ptr);
int tfgk_peer_export(void *ptr, void *handle_out);
int tfgk_peer_open(const void *handle, void **ptr);
int tfgk_peer_close(void *ptr);
/* Copies `bytes` (a multiple of 16, both pointers 16-byte aligned) from a peer-mapped buffer into local memory.
 * max_ctas > 0: copy kernel with that many CTAs (wide contiguous loads);  max_ctas = 0: the copy kernel on one CTA per SM
 * of the current device;  max_ctas < 0: the copy engine (cudaMemcpyAsync on `stream`; takes no SMs). */
int tfgk_peer_pull(const void *src, void *dst, int64_t bytes, int32_t max_ctas, void *stream);
int tfgk_peer_barrier(uint32_t *const *flags, int32_t rank, int32_t world, uint32_t value, int32_t timeout_ms, void *stream);

/* out[c] = sum_r x[r, c]: the bias gradients db = 1^T dY of the backward passes (TensorFlow autodiff's BiasAddGrad under
 * gcn.py:283-284, gat.py:116-117, graph_sage.py:51-52).  Deterministic: per-block partial sums added in block order. */
int tfgk_colsum_workspace_bytes(int64_t n_rows, int32_t D, size_t *out_bytes);
int tfgk_colsum_f32(const float *x, int64_t ldx, int64_t n_rows, int32_t D, float *out, void *workspace,
                    size_t workspace_bytes, void *stream);

/* tf.nn.l2_normalize(x, axis=-1) (graph_sage.py:57-58): out = x * rsqrt(max(sum(x^2), 1e-12)). */
int tfgk_l2_normalize_f32(const float *x, int64_t ldx, int32_t N, int32_t D, float *out, int64_t ldo, void *stream);

/* ---- training-mode extras (SURVEY.md 8(f)4) -------------------------------------------------------------------
 * Randomness is counter-based (Philox4x32-10): draw i of (seed, rng_stream) is a pure function of its arguments,
 * u_i = (philox(counter = (i >> 2, rng_stream, 0), key = seed)[i & 3] >> 8) * 2^-24.  Parity with TensorFlow's own
 * generator is statistical only; parity with oracle/tfg_oracle.py (same generator) is bit-exact. */

/* tf.nn.dropout (gcn.py:262 via tf_sparse dropout on the adjacency values, gat.py:85 on the attention coefficients):
 * out[i] = u_i >= rate ? x[i] * (1 / (1 - rate)) : 0.   x NULL = ones (a scaled keep mask). */
int tfgk_dropout_f32(const float *x, int64_t n, float rate, uint64_t seed, uint32_t rng_stream, float *out, void *stream);

/* Aggregation with one weight per (edge, head): the value half of gat.py:87-114 when the coefficients are already
 * known (attention dropout), and the three scatter-shaped gradients of the fused GAT kernel when run on the
 * transposed CSR.  weight(e, h) = w[pos*H + h] * dropout(pos*H + h), pos = emap ? emap[e] : e.
 *   TFGK_HEADS_SPLIT     out[r, h*dh+u] = alpha * sum_e weight(e,h) * src[col_e, h*dh+u]
 *   TFGK_HEADS_BROADCAST out[r, h*dh+u] = alpha * sum_e weight(e,h) * src[col_e, u]            (src has dh columns)
 *   TFGK_HEADS_REDUCE    out[r, u]      = alpha * sum_h sum_e weight(e,h) * src[col_e, h*dh+u]  (out has dh columns)
 * then + bias, activation.  Sequential in CSR order per row (deterministic). */
int tfgk_spmm_heads_f32(const int64_t *rowptr, const int32_t *col, const int32_t *emap, const float *w,
                        const float *src, int64_t lds, int32_t n_dst, int32_t H, int32_t dh, int mode,
                        float drop_rate, uint64_t seed, uint32_t rng_stream, float alpha,
                        const float *bias, int act, float *out, int64_t ldo, void *stream);

/* Gradient of gat.py:83-114 w.r.t. the scaled scores, given G = dL/d(aggregated rows before bias/activation):
 *   da_e,h = <G[r,h,:], V[col_e,h,:]> * dropout(e*H+h)   (split_value_heads=0: <G[r,:], V[col_e,h,:]> / H)
 *   ds_e,h = a_e,h * (da_e,h - sum_f a_f,h da_f,h)
 * att: [E, H] softmax coefficients BEFORE dropout, CSR order (tfgk_gat_fused_f32 with write_att); ds: [E, H] out.
 * The 1e-8 in segment.py:31 makes d a/d max non-zero by ~1e-8 relative in TF autodiff; that term is dropped. */
int tfgk_gat_softmax_bwd_f32(const int64_t *rowptr, const int32_t *col, const float *att,
                             const float *G, int64_t ldg, const float *V, int64_t ldv,
                             int32_t n_dst, int32_t H, int32_t dv, int split_value_heads,
                             float drop_rate, uint64_t seed, uint32_t rng_stream, float *ds, void *stream);

/* ---- device keys: the three entries above for CUDA-graph capture ------------------------------------------------
 * A captured graph replays its launches with the arguments they were captured with, so a key passed by value would draw
 * the same mask on every replay.  The _devkey entries take (key_base, slot) in place of `seed`: key_base points at one
 * uint64 in device memory, the base, and the kernel uses
 *     key = splitmix64(*key_base + 0x9E3779B97F4A7C15 * (slot + 1))
 * with splitmix64(z) = z ^= z >> 30, z *= 0xBF58476D1CE4E5B9, z ^= z >> 27, z *= 0x94D049BB133111EB, z ^ (z >> 31)
 * (the output function only; the Weyl step is the + above).  That is the host key sequence of tf_geometric_b200/_rng.py:
 * its (slot + 1)-th key after set_seed(base) is the key of `slot` here, so a captured run can be repeated eagerly.
 * Every other argument, and the mask as a function of (key, rng_stream, element), is that of the entry with a seed.
 * Epochs: tfgk_rng_advance replaces the base by splitmix64(base) on `stream` and, when `epoch` is not NULL, copies the new
 * base into *epoch.  The host enqueues it once per captured region, before its first keyed launch (slot 0), with an
 * epoch word of that region's own, and the region's launches take that word as key_base.  Every replay then draws new
 * masks, and a backward that regenerates a forward's masks reads the value its forward read, even when other graphs that
 * draw keys replay in between (make_graphed_callables over several modules replays every forward before any backward).
 * A graph that draws no key (a backward captured on its own) neither advances the base nor owns a word.
 * tfgk_capture_id: *id = the capture sequence id of `stream` (cudaStreamGetCaptureInfo), 0 when it is not capturing. */
int tfgk_dropout_devkey_f32(const float *x, int64_t n, float rate, const uint64_t *key_base, uint64_t slot,
                            uint32_t rng_stream, float *out, void *stream);
int tfgk_spmm_heads_devkey_f32(const int64_t *rowptr, const int32_t *col, const int32_t *emap, const float *w,
                               const float *src, int64_t lds, int32_t n_dst, int32_t H, int32_t dh, int mode,
                               float drop_rate, const uint64_t *key_base, uint64_t slot, uint32_t rng_stream, float alpha,
                               const float *bias, int act, float *out, int64_t ldo, void *stream);
int tfgk_gat_softmax_bwd_devkey_f32(const int64_t *rowptr, const int32_t *col, const float *att,
                                    const float *G, int64_t ldg, const float *V, int64_t ldv,
                                    int32_t n_dst, int32_t H, int32_t dv, int split_value_heads,
                                    float drop_rate, const uint64_t *key_base, uint64_t slot, uint32_t rng_stream,
                                    float *ds, void *stream);
int tfgk_rng_advance(uint64_t *key_base, uint64_t *epoch, void *stream);
int tfgk_capture_id(void *stream, uint64_t *id);

/* Training without the [E, H] coefficient table (round 2).  The forward pass is the same streaming kernel as
 * tfgk_gat_fused_f32 (heads concatenated, dqk == dv, H * dqk <= 128) and additionally keeps stats[N, 2H]: per (row, head)
 * the softmax maximum and the denominator (+1e-8).  The backward pass recomputes every coefficient from Q, K and stats:
 *   _prepare: GS[N, H*dqk + 32] = [ G * act'(Y) | max (8) | denominator (8) | delta = <G, Y - bias> per head (8) | pad (8) ]
 *   _dst    : dQ[r] = (1/scale) sum_{e in row r} ds_e K[col_e]                     forward CSR
 *   _src    : dK[c] = (1/scale) sum ds_e Q[row_e],  dV[c] = sum a_e G[row_e]       transposed CSR (rows = sources)
 * with a_e = exp(<Q_r, K_c>/scale - max_r) / den_r and ds_e = a_e (<G_r, V_c> - delta_r) per head.  Replaces TensorFlow
 * autodiff over gat.py:73-114.  The forward and the three backward entry points take the same (H, dqk): H a power of two
 * <= 8, dqk / 4 a power of two, H * dqk <= 128; TFGK_ERR_UNSUPPORTED for any other shape or unaligned operands, and the
 * caller keeps the coefficient table instead. */
int tfgk_gat_fused_stats_f32(const int64_t *rowptr, const int32_t *col,
                             const float *Q, int64_t ldq, const float *K, int64_t ldk, const float *V, int64_t ldv,
                             int32_t N, int32_t H, int32_t dqk, int32_t dv, float scale,
                             const float *bias, int act, float *out, int64_t ldo, float *stats,
                             const tfgk_plan *plan, void *stream);
int tfgk_gat_bwd_prepare_f32(const float *G, int64_t ldg, const float *Y, int64_t ldy, const float *bias, int act,
                             const float *stats, int32_t N, int32_t H, int32_t dqk, float *GS, int64_t ldgs, void *stream);
int tfgk_gat_bwd_dst_f32(const int64_t *rowptr, const int32_t *col, const float *Q, int64_t ldq,
                         const float *K, int64_t ldk, const float *V, int64_t ldv, const float *GS, int64_t ldgs,
                         int32_t N, int32_t H, int32_t dqk, float scale, float *dQ, int64_t lddq, void *stream);
int tfgk_gat_bwd_src_f32(const int64_t *rowptr_t, const int32_t *col_t, const float *Q, int64_t ldq,
                         const float *K, int64_t ldk, const float *V, int64_t ldv, const float *GS, int64_t ldgs,
                         int32_t N, int32_t H, int32_t dqk, float scale, float *dK, int64_t lddk, float *dV, int64_t lddv,
                         void *stream);

/* ---- device-side edge sampling (SURVEY.md 8(f)3) -------------------------------------------------------------- */

/* flag[e] = structural(e) && bernoulli(e):
 *   structural: ALL | UPPER row<col (drop_edge.py:35 force_undirected) | MAPPED row_map[row]>=0 && col_map[col]>=0
 *               (graph_utils.py:826-832 virtual node filter)
 *   bernoulli : NONE | DROPOUT u_e >= prob (drop_edge.py:36,41: tf.nn.dropout(ones, rate) > 0) | KEEP u_e <= prob
 *               (graph_utils.py:808-809,841-842 UniformNeighborSampler) */
int tfgk_edge_flags_i32(const int32_t *row, const int32_t *col, int64_t E, int mode,
                        const int32_t *row_map, const int32_t *col_map,
                        int bernoulli, float prob, uint64_t seed, uint32_t rng_stream, int32_t *flag, void *stream);

/* tf.boolean_mask(tf.range(n), flag): ascending positions of the non-zero flags; *n_out_host = how many.
 * Synchronises the stream. */
int tfgk_select_workspace_bytes(int64_t n, size_t *out_bytes);
int tfgk_select_flagged_i32(const int32_t *flag, int64_t n, int32_t *out_index, int64_t *n_out_host,
                            void *workspace, size_t workspace_bytes, void *stream);

/* Building blocks of nn/pool/topk_pool.py:31-58 (tf.argsort by source, per-source descending tf.argsort of the scores):
 * keys[i] = order-preserving 32-bit pattern of score[i] (complemented for descending; -0.0 ties with +0.0), and a
 * stable LSD radix argsort of 32-bit patterns read as unsigned numbers (only the low key_bits are examined):
 * perm_out[j] = position of the j-th smallest key, equal keys in input order. */
int tfgk_sort_keys_f32(const float *score, int64_t n, int descending, int32_t *keys, void *stream);
int tfgk_argsort_workspace_bytes(int64_t n, size_t *out_bytes);
int tfgk_stable_argsort_u32(const int32_t *keys, int64_t n, int key_bits, int32_t *perm_out,
                            void *workspace, size_t workspace_bytes, void *stream);

/* RandomNeighborSampler.sample (graph_utils.py:669-776) on a CSR whose rows are the source nodes in ascending order
 * with neighbours in edge order (= the reference's neighbor_dict).  k < 0 and ratio < 0: every neighbour; ratio < 0:
 * k per row (all of them in order when k >= degree and !padding; k draws WITH replacement when padding and
 * k >= degree); otherwise ceil(degree * ratio) without replacement.  Rows without neighbours emit nothing.
 * _count writes the [n_rows + 1] offsets of the sampled edges and their total (synchronises); _fill writes, per sampled
 * edge, its row and the CSR position it was taken from (gather col / weights with tfgk_permute_f32).  Without
 * replacement = reservoir sampling with draws (seed, rng_stream, row << 32 | i).
 * padding = TFGK_SAMPLE_HEAD is the deterministic rule of nn/pool/topk_pool.py:59-82: the FIRST min(k, degree) (or
 * ceil(float(degree) * float(ratio)), float32 like the reference) entries of every row, in order. */
int tfgk_neighbor_sample_workspace_bytes(int32_t n_rows, size_t *out_bytes);
int tfgk_neighbor_sample_count(const int64_t *rowptr, int32_t n_rows, int32_t k, double ratio, int padding,
                               int64_t *out_rowptr, int64_t *total_host, void *workspace, size_t workspace_bytes,
                               void *stream);
int tfgk_neighbor_sample_fill(const int64_t *rowptr, int32_t n_rows, int32_t k, double ratio, int padding,
                              uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                              int32_t *out_row, int32_t *out_pos, void *stream);

/* K13: the same sampler over a list of n_list rows of an existing CSR (rowptr with n_rows rows, not copied).  Listed row t
 * is global row rows[t]; its sampled positions are exactly those tfgk_neighbor_sample_fill writes for that global row with
 * the same k / ratio / padding / seed / rng_stream, in the same order, so a node's sample depends on the node and the key
 * only.  Rows may repeat.  _count takes the workspace of tfgk_neighbor_sample_workspace_bytes(n_list), writes the
 * [n_list + 1] offsets and their total (synchronises) and fails with TFGK_ERR_INDEX_OUT_OF_RANGE for a listed row outside
 * [0, n_rows).  _fill writes out_pos and, unless out_row is null, the LIST position t of every sampled edge's row.
 * Work is proportional to the listed rows' degrees: rows of degree <= 128 take one thread, longer rows a CTA of 256. */
int tfgk_neighbor_sample_rows_count(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list, int32_t k,
                                    double ratio, int padding, int64_t *out_rowptr, int64_t *total_host, void *workspace,
                                    size_t workspace_bytes, void *stream);
int tfgk_neighbor_sample_rows_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list, int32_t k,
                                   double ratio, int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                   int32_t *out_row, int32_t *out_pos, void *stream);

/* Relabelling through an int32 [N] id -> position map that holds -1 everywhere before and after each call (the caller
 * fills it with -1 once and may keep it; calls that share a map must be ordered on one stream).  Node ids outside
 * [0, N) fail with TFGK_ERR_INDEX_OUT_OF_RANGE; *n_dup_host counts the node-list entries that repeat an earlier id (the
 * output is then meaningless and the caller reports the error).  Both synchronise `stream`.
 * tfgk_reindex_i32: out[e] = position of ids[e] in nodes[0, n_nodes), -1 when absent or outside [0, N).
 * tfgk_frontier_i32: nodes[0, n_nodes) is the current list and has room for S more ids.  The ids of cols[0, S) that are
 * not in the list are appended in first-occurrence order (*n_new_host of them) and local_col[e] = the position of
 * cols[e] in the grown list.  Deterministic: first occurrences are found with atomicMin and placed by a scan. */
int tfgk_relabel_workspace_bytes(int64_t n_ids, size_t *out_bytes);
int tfgk_reindex_i32(const int32_t *nodes, int32_t n_nodes, const int32_t *ids, int64_t n_ids, int32_t N, int32_t *map,
                     int32_t *out, int32_t *n_dup_host, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_frontier_i32(const int32_t *cols, int64_t S, int32_t N, int32_t *nodes, int32_t n_nodes, int32_t *map,
                      int32_t *local_col, int32_t *n_new_host, int32_t *n_dup_host, void *workspace, size_t workspace_bytes,
                      void *stream);

/* Block sampler: the mini-batch neighbourhood of tfgk_neighbor_sample_rows_* + tfgk_frontier_i32, with every size kept on
 * the device so that a batch synchronises once, at its end.  Bit for bit, the node list and every hop's edges are those
 * of the K13 + frontier route with the same keys (hop h samples every listed row, new ids are appended in first-occurrence
 * order).  state is int32 [4 + 2 L] for L hops: [0] seeds outside [0, N), [1] repeated seeds, [2] unused,
 * [3 + h] list length after hop h (h = 0: the seeds), [4 + L + h] edges of hop h.  map is the relabelling map of
 * tfgk_frontier_i32 (-1 everywhere before begin and after end); it stays populated across the hops of a batch.  Calls
 * of one batch must be ordered on one stream.
 * _begin: nodes[0, n_seeds) = seeds, map[seed] = position, the seed counters; reads nothing back.
 * _count: K13's count and scan for hop `hop` (< n_hops, the L of state) over cap_list >= the list length (read from
 *   state): out_rowptr int64 [cap_list + 1], zero-count rows past the list, so out_rowptr[cap_list] is the hop's edge
 *   total.  Asynchronous.
 * A batch that fails between _begin and _end leaves the map populated: the caller resets it (ops.block_sample does).
 * _read_total: the list length and out_rowptr[cap_list] to the host (synchronises); the fallback for hops whose edge
 *   capacity is unknown (every neighbour) or not below 2^31.
 * _fill: K13's fill (out_row = list position, out_gcol = col[pos], out_w = w_csr[pos]; cap_edges >= the edge total),
 *   then the frontier: new ids appended to nodes (room for them is the caller's), out_local = position of out_gcol in
 *   the grown list, and state's sizes for the hop.  Asynchronous.  The workspace is that of
 *   tfgk_block_sample_workspace_bytes(cap_list, cap_edges), shared with _count.
 * _end: resets map over the final list (cap_nodes >= its length), then copies state to state_host and synchronises. */
int tfgk_block_sample_workspace_bytes(int32_t cap_list, int64_t cap_edges, size_t *out_bytes);
int tfgk_block_sample_begin(const int32_t *seeds, int32_t n_seeds, int32_t N, int32_t *nodes, int32_t *map,
                            int32_t *state, int32_t n_hops, void *stream);
int tfgk_block_sample_count(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                            int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding, int64_t *out_rowptr,
                            void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_read_total(const int32_t *state, int32_t hop, const int64_t *out_rowptr, int32_t cap_list,
                                 int32_t *n_list_host, int64_t *total_host, void *stream);
int tfgk_block_sample_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr, int32_t N,
                           int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                           int64_t cap_edges, int32_t k, int padding, uint64_t seed, uint32_t rng_stream,
                           const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local, int32_t *out_gcol,
                           float *out_w, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_end(const int32_t *nodes, int32_t cap_nodes, int32_t N, int32_t *map, const int32_t *state,
                          int32_t n_hops, int32_t *state_host, void *stream);
/* _fill over a CSR in host memory: col (and w_csr) are device-readable pointers to page-locked host memory, and w_csr may
 * be NULL (every weight is then 1.0f and nothing is read).  CSR positions are int64, so the CSR may hold 2^31 edges or
 * more; rowptr stays on the device.  Same rule, same draws and same outputs as tfgk_block_sample_fill over the same CSR.
 * Each sampled edge reads one 4-byte column (and one 4-byte weight) over the host link.  The workspace is that of
 * tfgk_block_sample_mapped_workspace_bytes(cap_list, cap_edges), which also serves _count; _begin, _count, _read_total
 * and _end are shared with the device CSR. */
int tfgk_block_sample_mapped_workspace_bytes(int32_t cap_list, int64_t cap_edges, size_t *out_bytes);
int tfgk_block_sample_fill_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                  int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                  int32_t cap_list, int64_t cap_edges, int32_t k, int padding, uint64_t seed,
                                  uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                  int32_t *out_gcol, float *out_w, void *workspace, size_t workspace_bytes,
                                  void *stream);

/* A block's self loops (GAT on a sampled block, utils.SelfLoopBlock): the block's CSR (rowptr int64 [n_dst + 1], and for
 * each of its S edges in CSR order the row row[p] < n_dst and column col[p]) with the edge (r, r) appended after the
 * sampled edges of every row r < n_dst, where a block's output row r is its input row r.
 * out_rowptr [n_dst + 1]: out_rowptr[r] = rowptr[r] + r.  out_row / out_col [S + n_dst]: edge p of row r moves to p + r,
 * and row r's self edge goes to rowptr[r + 1] + r.  row must agree with rowptr (rowptr[row[p]] <= p < rowptr[row[p] + 1]).
 * One launch, grid-strided over S + n_dst + 1 items; no atomics, no host synchronisation.  S + n_dst >= 2^31 returns
 * TFGK_ERR_UNSUPPORTED. */
int tfgk_block_self_loops_i32(const int64_t *rowptr, const int32_t *row, const int32_t *col, int64_t S, int32_t n_dst,
                              int64_t *out_rowptr, int32_t *out_row, int32_t *out_col, void *stream);

/* A row block (layer-wise inference, utils.RandomNeighborSampler.row_block / HostNeighborSampler.row_block): the block
 * sampler's batch for the seeds r0, ..., r1 - 1 and one hop of fan-out None, bit for bit, from the range's columns.
 * rowptr int64 [N + 1] (device) is the graph's CSR row pointer; cols int32 [S] (device) its columns
 * [rowptr[r0], rowptr[r1]), staged by the caller, S = rowptr[r1] - rowptr[r0] < 2^31.  map is the int32 [N] relabelling
 * map of tfgk_frontier_i32 (-1 everywhere before and after).  Writes, with n = r1 - r0:
 *   nodes [n + S at most]: nodes[i] = r0 + i, then the columns outside the range in first-occurrence order;
 *   out_rowptr int64 [n + 1] = rowptr[r0 .. r1] - rowptr[r0];  out_row [S]: each edge's output row;
 *   out_local [S]: each column's position in nodes;  *num_src_host: the length of nodes.
 * The range's ids are distinct and in range by construction, so the seeds get no duplicate or bad-id pass; the columns
 * are relabelled by tfgk_frontier_i32's kernels and scan.  Workspace: tfgk_relabel_workspace_bytes(S).  One host read-back
 * (the list length) when S > 0, none when S == 0.  A column id outside [0, N) fails with TFGK_ERR_INDEX_OUT_OF_RANGE. */
int tfgk_row_block_i32(const int64_t *rowptr, int32_t N, int32_t r0, int32_t r1, const int32_t *cols, int64_t S,
                       int32_t *nodes, int32_t *map, int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                       int32_t *num_src_host, void *workspace, size_t workspace_bytes, void *stream);
/* cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, stream): asynchronous between device memory and page-locked host
 * memory (tfgk_host_register's ranges, or pinned allocations), whatever a framework knows of the host buffer. */
int tfgk_copy_async(void *dst, const void *src, size_t bytes, void *stream);

/* GCN's normalised values on a sampled block (utils.GcnBlock): every row normalised with its FULL-graph degree, and each
 * output row's sampled edges rescaled so that their sum is an unbiased estimate of the full graph's row.
 * The block: rowptr int64 [n_dst + 1] (rowptr[0] = 0, rowptr[n_dst] = S), gcol int32 [S] (the global id of every edge's
 * column), w float32 [S] (NULL: all ones), dst int32 [n_dst] (the global id of every output row).  The full graph:
 * g_rowptr int64 and g_rowsum float32, indexed by global id: the sampler's CSR rowptr and the sequential fp32 row sums of
 * its weights (tfgk_csr_rowsum_f32).  For output row r with global id g, k_r = rowptr[r + 1] - rowptr[r] sampled edges
 * and n_g = g_rowptr[g + 1] - g_rowptr[g] edges in the full graph:
 *   f(v) = d^-1/2 (norm BOTH) or d^-1 (LEFT, RIGHT) of d = g_rowsum[v] + deg_fill, as tfgk_deg_inv_f32 (inf, nan -> 0)
 *   edge p of row r:  s_r * (f(g) * w[p] * f(gcol[p]))  BOTH,  s_r * (f(g) * w[p])  LEFT,  s_r * (w[p] * f(gcol[p]))  RIGHT
 *                     with s_r = (float)n_g / (float)k_r, each product rounded in that order (tfgk_scale_edges_f32's,
 *                     then s_r; s_r = 1 changes no bit)
 *   self loop of r:   fill scaled like an edge (g, g) without s_r (loop = TFGK_GCN_LOOP_NORMED), or fill as it is (_FILL)
 * out: with a loop mode, [S + n_dst] in tfgk_block_self_loops_i32's layout (edge p of row r at p + r, row r's loop at
 * rowptr[r + 1] + r); with TFGK_GCN_LOOP_NONE, [S] in the block's order.
 * One launch, grid-strided over S (+ n_dst) items; no atomics, no host synchronisation.  An edge finds its row by binary
 * search over rowptr.  Algorithmic bytes: 12 per edge (gcol, w, out) plus a 4-byte g_rowsum gather per edge for BOTH and
 * RIGHT, and 40 per output row (rowptr, dst, g_rowptr, g_rowsum, the loop).  S + n_dst >= 2^31 returns
 * TFGK_ERR_UNSUPPORTED. */
int tfgk_block_gcn_values_f32(const int64_t *rowptr, const int32_t *gcol, const float *w, int64_t S, const int32_t *dst,
                              int32_t n_dst, const int64_t *g_rowptr, const float *g_rowsum, int norm, int loop,
                              float deg_fill, float fill, float *out, void *stream);

/* Link prediction on sampled blocks (utils.LinkBlocks): a block batch seeded by the endpoints of node pairs, with the
 * batch's target edges optionally excluded from the CSR rows their endpoints sample.
 * _begin_pairs: tfgk_block_sample_begin for the endpoint list pair_row[0], pair_col[0], pair_row[1], ... of n_pairs pairs:
 *   the frontier of an empty list over those 2 n_pairs ids, so nodes[0, n_seeds) holds the distinct endpoints in
 *   first-occurrence order, map[id] their positions and state[3] = n_seeds (on the device).  Endpoints outside [0, N) are
 *   counted in state[0] and relabelled -1.  local int32 [2, n_pairs]: the pairs relabelled (sources, then destinations).
 *   Hop 0's capacity is 2 n_pairs.  Workspace: tfgk_block_pairs_workspace_bytes(n_pairs).  Asynchronous; _count, _fill
 *   and _end follow as for _begin.
 * tfgk_link_tail_negatives_i32: out_row[i] = src[i / q], out_col[i] = random_below64(seed, rng_stream, i, N) for
 *   i < n_src * q (tail corruption, uniform over [0, N) to within N / 2^64).  One launch, asynchronous.
 * Exclusion lists, for the cap >= n_seeds first rows of the list `nodes`: target_src / target_dst [n_targets] are the
 *   (local row, global column) pairs to exclude, sorted by (source, destination) (sources outside [0, cap) are
 *   skipped).  Row t's list is every position p of CSR row nodes[t] whose column col[p] is a target of t, ascending; a
 *   position is listed once however many targets match it.  col may be device memory or page-locked host memory; each
 *   targeted row reads its deg columns once per pass.
 *   _count writes excl_off int64 [cap + 1] (exclusive offsets) and the total to *total_host (synchronises).  _fill
 *   (int32 positions) and _fill_mapped (int64 positions, a CSR in host memory) then write excl_pos [total], with the
 *   workspace _count used: tfgk_block_exclusion_workspace_bytes(cap).
 * _count_excl, _fill_excl, _fill_mapped_excl: _count, _fill and _fill_mapped where list row t < n_excl skips the
 *   x_t = excl_off[t + 1] - excl_off[t] positions excl_pos[excl_off[t], excl_off[t + 1]) of its CSR row: the rule and
 *   the draws run over the deg - x_t kept entries in CSR order, so the hop equals that of the same call on the CSR with
 *   those entries deleted.  Rows without exclusions take the plain path.
 * tfgk_block_gcn_values_excl_f32: tfgk_block_gcn_values_f32 where output row r < n_excl scales its edges by
 *   s_r = (n_g - x_r) / k_r. */
int tfgk_block_pairs_workspace_bytes(int32_t n_pairs, size_t *out_bytes);
int tfgk_block_sample_begin_pairs(const int32_t *pair_row, const int32_t *pair_col, int32_t n_pairs, int32_t N,
                                  int32_t *nodes, int32_t *map, int32_t *state, int32_t n_hops, int32_t *local,
                                  void *workspace, size_t workspace_bytes, void *stream);
int tfgk_link_tail_negatives_i32(const int32_t *src, int32_t n_src, int32_t q, int32_t N, uint64_t seed,
                                 uint32_t rng_stream, int32_t *out_row, int32_t *out_col, void *stream);
int tfgk_block_exclusion_workspace_bytes(int32_t cap, size_t *out_bytes);
int tfgk_block_exclusion_count(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                               int32_t cap, const int32_t *target_src, const int32_t *target_dst, int64_t n_targets,
                               int64_t *excl_off, int64_t *total_host, void *workspace, size_t workspace_bytes,
                               void *stream);
int tfgk_block_exclusion_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                              int32_t cap, const int32_t *target_dst, const int64_t *excl_off, int32_t *excl_pos,
                              void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_exclusion_fill_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                     int32_t cap, const int32_t *target_dst, const int64_t *excl_off, int64_t *excl_pos,
                                     void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_count_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                                 int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding,
                                 const int64_t *excl_off, int32_t n_excl, int64_t *out_rowptr, void *workspace,
                                 size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                int32_t cap_list, int64_t cap_edges, int32_t k, int padding, uint64_t seed,
                                uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                int32_t *out_gcol, float *out_w, const int64_t *excl_off, const int32_t *excl_pos,
                                int32_t n_excl, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                       int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                       int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, int padding,
                                       uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                       int32_t *out_local, int32_t *out_gcol, float *out_w, const int64_t *excl_off,
                                       const int64_t *excl_pos, int32_t n_excl, void *workspace, size_t workspace_bytes,
                                       void *stream);

/* Weighted block sampler: fan-outs drawn in proportion to the CSR's float32 weights w_csr (utils.RandomNeighborSampler /
 * HostNeighborSampler with weighted=True).  The draw rule, for listed row t of global row r under hop key `seed`:
 *   Candidates: the row's kept entries (all of them, or those the _excl lists leave), numbered by virtual position v as
 *     the _excl entries number them; only entries of weight > 0 can be drawn, and d+ counts them.
 *   Key: E(v, j) = -ln(u) / w in double, w the float32 weight widened, u = ((u64 >> 11) + 1) 2^-53 in (0, 1] where u64 is
 *     lanes 0 | 1 << 32 of one Philox4x32-10 block with counter (v, r, rng_stream, j) and key `seed`.  ln is rng.cuh's
 *     log_rn (exact exponent extraction, a fixed polynomial in explicitly rounded double operations), not the libm.
 *   Integer fan-out k, padding 0, or padding 1 with k < d+: the min(k, d+) candidates of smallest (E(v, 0), v), without
 *     replacement (successive sampling, Efraimidis-Spirakis), written in ascending CSR position.
 *   Padding 1 with k >= d+ > 0: k draws with replacement, P(entry) = w / W; draw j is the candidate of smallest
 *     (E(v, j + 1), v) (an exponential race: no prefix sums, so no bit depends on a summation order); draws in order.
 *   d+ = 0: nothing.  Fan-out None is not a weighted rule (it takes every kept entry, zero weights included: the caller
 *   uses the unweighted entries), and neither is the head rule; both are refused.
 * pos_deg int32 [n_rows]: the positive degree of every CSR row, from tfgk_csr_positive_degree_f32.
 * tfgk_csr_positive_degree_f32: pos_deg[r] = the entries of weight > 0 (and finite) of rows [0, n_rows) of rowptr, whose
 *   weights are w[p - w_base] (w_base: the CSR position of w[0], so a range of rows staged on the device takes the
 *   range's slice of rowptr and its first position); adds the count of negative, NaN and infinite weights to *n_invalid
 *   (device).  One warp per row; asynchronous.
 * _count_weighted / _count_weighted_excl / _count_weighted_mapped_excl: _count / _count_excl by the rule above (the _excl
 *   forms read the weights at the excluded positions, int32 or, over a host CSR, int64).
 * _fill_weighted, _fill_weighted_excl, _fill_weighted_mapped, _fill_weighted_mapped_excl: the _fill entries by the rule
 *   above, same outputs otherwise (positions, then global columns and weights, then the frontier).  A row of at most 128
 *   entries is drawn by one warp, which reads its weights once in 128-byte segments; a longer row by the CTA, with a
 *   radix select of the k smallest keys (8 bits a pass, keys recomputed from the counter each pass, so no workspace grows
 *   with the degree) or one CTA argmin per draw with replacement.  Over a host CSR every candidate's weight crosses the
 *   link: once for a warp row, once per pass for a CTA row.
 * tfgk_neighbor_sample_rows_count_weighted / _fill_weighted: K13's count and fill by the same rule, for
 *   sample_neighborhood (device CSR, int32 positions). */
int tfgk_csr_positive_degree_f32(const int64_t *rowptr, int32_t n_rows, const float *w, int64_t w_base,
                                 int32_t *pos_deg, int32_t *n_invalid, void *stream);
int tfgk_neighbor_sample_rows_count_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list,
                                             int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                             int64_t *out_rowptr, int64_t *total_host, void *workspace,
                                             size_t workspace_bytes, void *stream);
int tfgk_neighbor_sample_rows_fill_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list,
                                            int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                            uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                            int32_t *out_row, int32_t *out_pos, void *stream);
int tfgk_block_sample_count_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                                     int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding,
                                     const int32_t *pos_deg, const float *w_csr, int64_t *out_rowptr, void *workspace,
                                     size_t workspace_bytes, void *stream);
int tfgk_block_sample_count_weighted_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes,
                                          const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                          int padding, const int32_t *pos_deg, const float *w_csr,
                                          const int64_t *excl_off, const int32_t *excl_pos, int32_t n_excl,
                                          int64_t *out_rowptr, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_count_weighted_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes,
                                                 const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                                                 int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                                 const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                                 int64_t *out_rowptr, void *workspace, size_t workspace_bytes,
                                                 void *stream);
int tfgk_block_sample_fill_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                    const int32_t *pos_deg, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                    int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                    int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                    int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                    void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_weighted_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                         const int32_t *pos_deg, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                         int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                         int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                         int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                         const int64_t *excl_off, const int32_t *excl_pos, int32_t n_excl,
                                         void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_weighted_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                           const float *w_csr, const int32_t *pos_deg, int32_t N, int32_t *nodes,
                                           int32_t *map, int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                                           int64_t cap_edges, int32_t k, int padding, uint64_t seed, uint32_t rng_stream,
                                           const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                           int32_t *out_gcol, float *out_w, void *workspace, size_t workspace_bytes,
                                           void *stream);
int tfgk_block_sample_fill_weighted_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                                const float *w_csr, const int32_t *pos_deg, int32_t N, int32_t *nodes,
                                                int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                                int32_t cap_list, int64_t cap_edges, int32_t k, int padding,
                                                uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                                int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                                const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                                void *workspace, size_t workspace_bytes, void *stream);

/* LABOR block sampler: layer-neighbour sampling (LABOR-0; Balin & Catalyurek, NeurIPS 2023), the rule of
 * utils.RandomNeighborSampler / HostNeighborSampler with labor=True.  For listed row t of global row r under hop key
 * `seed` (the hop's _batch_seed key, or hop 0's at every hop with layer dependency) and integer fan-out k >= 0:
 *   Candidates: the row's kept entries (all of them, or those the _excl lists leave); d counts them.
 *   Variate: u_c = lane 0 of one Philox4x32-10 block with counter (c, 0, rng_stream, 0) and key `seed`, c the entry's
 *     column (a global node id); rng_stream is RNG_STREAM_LABOR = 4.  u_c depends on c and the key only: not on the row,
 *     the CSR position or the exclusions.
 *   Rule: d <= k keeps every candidate (no column is read to count it); otherwise candidate (t, c) is kept iff
 *     (uint64) u_c * d < (uint64) k << 32, exact integer arithmetic.  k = 0 keeps nothing.  Kept entries are written in
 *     ascending CSR position, with their global columns and their weights w_csr[p] (1.0f when w_csr is null).
 *   Properties, with pi(k, d) = ceil(k 2^32 / d) / 2^32 for d > k and 1 otherwise: each candidate is kept with
 *     probability pi; given its count m, a row's kept set is uniform over the m-subsets of its distinct columns (repeated
 *     columns are kept or dropped together); two rows of one hop sharing c both keep it with probability min(pi_1, pi_2),
 *     so c is reached with probability max pi over the listed rows holding it; a row with d > k keeps nothing with
 *     probability (1 - pi)^(distinct columns).  A row keeps k entries in expectation and up to d, so no capacity bounds a
 *     LABOR hop: the caller reads its edge total back (tfgk_block_sample_read_total), as for fan-out None.
 *   Fan-out None and padding are not LABOR rules (refused: the caller uses the uniform entries for None).
 * _count_labor / _count_labor_excl / _count_labor_mapped_excl: _count / _count_excl by this rule (col: the CSR's int32
 *   columns, on the device or page-locked in host memory; the _excl forms take int32 or, over a host CSR, int64
 *   excluded positions).  _fill_labor, _fill_labor_excl, _fill_labor_mapped, _fill_labor_mapped_excl: the _fill entries
 *   by this rule, same outputs otherwise.  Both passes visit a row of d > k (and the fill every row) with the same
 *   predicate: one warp for a row of at most 128 entries, its columns read 32 at a time (128-byte segments over the host
 *   link) and its kept entries placed by a ballot prefix; the whole CTA for a longer row, 256 columns at a time and a
 *   block-wide prefix count.  Every candidate column of a row of d > k is read twice (count, fill). */
int tfgk_block_sample_count_labor(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                  const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                  uint64_t seed, uint32_t rng_stream, int64_t *out_rowptr, void *workspace,
                                  size_t workspace_bytes, void *stream);
int tfgk_block_sample_count_labor_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                       const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                       uint64_t seed, uint32_t rng_stream, const int64_t *excl_off,
                                       const int32_t *excl_pos, int32_t n_excl, int64_t *out_rowptr, void *workspace,
                                       size_t workspace_bytes, void *stream);
int tfgk_block_sample_count_labor_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                              const int32_t *nodes, const int32_t *state, int32_t hop, int32_t n_hops,
                                              int32_t cap_list, int32_t k, uint64_t seed, uint32_t rng_stream,
                                              const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                              int64_t *out_rowptr, void *workspace, size_t workspace_bytes,
                                              void *stream);
int tfgk_block_sample_fill_labor(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                 int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                 int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed, uint32_t rng_stream,
                                 const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local, int32_t *out_gcol,
                                 float *out_w, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_labor_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                      int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                      int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed,
                                      uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                      int32_t *out_local, int32_t *out_gcol, float *out_w, const int64_t *excl_off,
                                      const int32_t *excl_pos, int32_t n_excl, void *workspace, size_t workspace_bytes,
                                      void *stream);
int tfgk_block_sample_fill_labor_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                        int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                        int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed,
                                        uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                        int32_t *out_local, int32_t *out_gcol, float *out_w, void *workspace,
                                        size_t workspace_bytes, void *stream);
int tfgk_block_sample_fill_labor_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                             const float *w_csr, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                             int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                             uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                             int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                             const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                             void *workspace, size_t workspace_bytes, void *stream);
int tfgk_block_gcn_values_excl_f32(const int64_t *rowptr, const int32_t *gcol, const float *w, int64_t S,
                                   const int32_t *dst, int32_t n_dst, const int64_t *g_rowptr, const float *g_rowsum,
                                   int norm, int loop, float deg_fill, float fill, const int64_t *excl_off,
                                   int32_t n_excl, float *out, void *stream);

/* ---- link prediction (SURVEY.md 8(f)5, demo/demo_gae.py) -------------------------------------------------------- */

/* K6, predict_edge of demo/demo_gae.py:53-60: out[e] = sum_d h[row_e, d] * h[col_e, d] in fp32, COO order.
 * h is [N, D] with leading dimension ldh.  An edge's result depends only on that edge and h (same bits whatever E,
 * the launch or the edge's position); an id outside [0, N) gives NaN and is never read.  Asynchronous.
 * Algorithmic bytes: E * (8 D + 12). */
int tfgk_edge_dot_f32(const float *h, int64_t ldh, int32_t N, const int32_t *row, const int32_t *col, int64_t E, int32_t D,
                      float *out, void *stream);

/* Exact negative sampling over an implicit candidate list (utils/graph_utils.py:369-452).  The caller passes a CSR
 * (rowptr int64 [N+1], col int32) whose row i holds X_i, the sorted DISTINCT columns row i must not pair with:
 *   TFGK_NEG_UPPER  X_i = upper neighbours j > i of the undirected edge set; row i's candidates are the j in (i, N) not
 *                   in X_i, and the rows concatenated are np.nonzero(np.triu(adj, 1)) of the reference (row-major);
 *   TFGK_NEG_START  X_a = out-neighbours of a together with a itself; a's candidates are [0, N) minus X_a.
 * _offsets: offsets[i] = candidates before row i (int64 prefix sum), *total_host = C (synchronises `stream`).
 * _draw: k[s] = random_below64(seed, rng_stream, round << 32 | s, C) for s = index[t] (index NULL: s = t < n).
 * _dup_flags: flag[order[p]] = 1 when k[order[p]] == k[order[p-1]] (order = a stable argsort of k: later duplicates).
 * _decode: candidate k[s] -> (out_row[s], out_col[s]) by two binary searches; k outside [0, C) gives (-1, -1).
 * _sample_start: out_col[s] = candidate random_below64(seed, rng_stream, s, count) of row start[s] (TFGK_NEG_START
 *                structure); -1 for a start id outside [0, N) or a row without candidates. */
enum tfgk_neg_mode { TFGK_NEG_UPPER = 0, TFGK_NEG_START = 1 };
int tfgk_neg_offsets_workspace_bytes(int32_t N, size_t *out_bytes);
int tfgk_neg_offsets(const int64_t *rowptr, int32_t N, int mode, int64_t *offsets, int64_t *total_host, void *workspace,
                     size_t workspace_bytes, void *stream);
int tfgk_neg_draw(int64_t C, const int32_t *index, int64_t n, uint64_t seed, uint32_t rng_stream, int32_t round, int64_t *k,
                  void *stream);
int tfgk_neg_dup_flags(const int64_t *k, const int32_t *order, int64_t S, int32_t *flag, void *stream);
int tfgk_neg_decode(const int64_t *rowptr, const int32_t *col, const int64_t *offsets, int32_t N, int mode, const int64_t *k,
                    int64_t S, int32_t *out_row, int32_t *out_col, void *stream);
int tfgk_neg_sample_start(const int64_t *rowptr, const int32_t *col, int32_t N, const int32_t *start, int64_t S,
                          uint64_t seed, uint32_t rng_stream, int32_t *out_col, void *stream);
/* np.random.randint(0, N, [2, S]) with the counter-based generator: out[0, s] = random_below64(seed, rng_stream, 2 s, N),
 * out[1, s] = random_below64(seed, rng_stream, 2 s + 1, N), one Philox block per pair and uniform over [0, N) to within
 * N / 2^64  (negative_sampling without edge_index, graph_utils.py:384-386). */
int tfgk_random_pairs_i32(int32_t N, int64_t S, uint64_t seed, uint32_t rng_stream, int32_t *out, void *stream);

/* ---- edge-weight gradients ------------------------------------------------------------------------------------ */

/* K7, sampled dense-dense product over a destination-sorted CSR: for every slot p of every row r,
 *     out[perm ? perm[p] : p] = (alpha * row_scale[r]) * sum_d G[r, d] * X[col[p], d]
 * (row_scale NULL: 1).  It is the gradient of K1's output with respect to its edge weights: G = d loss / d out, X the
 * aggregated rows, row_scale = 1 / max(cnt, 1) for the mean reducer; with perm (the CSR's slot -> edge map) the result
 * lands in the caller's edge order.  G is [N_rows, D] with leading dimension ldg, X [*, D] with ldx; column slices are
 * fine.  The slots are cut into warp tasks of equal size (TFGK_SDDMM_TASK_EDGES, default 512), so a hub row is spread
 * over several warps; each output is one edge, written once, without atomics.  An edge's bits depend only on G[r],
 * X[col[p]], row_scale[r] and alpha (not on the task size, the grid or perm).  Asynchronous.
 * Algorithmic bytes: E * (4 D + 12) + N_rows * (4 D + 8). */
int tfgk_sddmm_csr_f32(const int64_t *rowptr, const int32_t *col, const int32_t *perm, int32_t N_rows,
                       const float *G, int64_t ldg, const float *X, int64_t ldx, int32_t D,
                       const float *row_scale, float alpha, float *out, void *stream);

/* ---- DiffPool / MinCutPool: per-graph dense algebra (nn/pool/cluster_pool.py:32-44) -------------------------------
 * A batch of G graphs whose nodes are each assigned to C clusters of their own graph; block layout: row g*C + c of a
 * [G*C, *] matrix belongs to cluster c of graph g. */

/* K8a, per-graph transposed product: out[g*C + c, d] = sum_{n in graph g} S[n, c] * Y[n, d], fp32, for c < C, d < D.
 * Graph g's nodes are the node-list positions p in [gptr[g], gptr[g+1]), node id gnodes[p] (gnodes NULL: p itself, i.e.
 * graph-major nodes).  S is [N, C] (lds), Y [N, D] (ldy), out [G*C, D] (ldo); column slices are fine.  S^T X, S^T (A S)
 * and S^T S are one launch each.  Every graph is cut into chunks of 1024 positions; a graph with several chunks sums
 * them into the workspace and a fix-up adds the partial blocks in chunk order.  Within a chunk the rows are summed in
 * node-list order with fmaf, so a graph's bits depend only on its own rows (not on G, the grid or the other graphs); no
 * atomics.  A node id outside [0, N), or a graph whose positions reach past N, makes its graph's block NaN.  Asynchronous (the chunk plan is computed on the device).
 * Algorithmic bytes: N * 4 (C + D) + G * C * D * 4 + G * 8. */
int tfgk_graph_tmm_workspace_bytes(int32_t G, int32_t N, int32_t C, int32_t D, size_t *out_bytes);
int tfgk_graph_tmm_f32(const float *S, int64_t lds, const float *Y, int64_t ldy, int32_t N, int32_t C, int32_t D,
                       const int64_t *gptr, const int32_t *gnodes, int32_t G, float *out, int64_t ldo, void *workspace,
                       size_t workspace_bytes, void *stream);

/* K8b, row times its graph's block: with g = node_graph[n] and B [G*C, K] (ldb) in block layout,
 *   trans = 0: out[n, k] = beta * out[n, k] + sum_{c < C} Y[n, c] * B[g*C + c, k]     Y [N, C], out [N, K]
 *   trans = 1: out[n, c] = beta * out[n, c] + sum_{k < K} Y[n, k] * B[g*C + c, k]     Y [N, K], out [N, C]
 * (beta = 0 never reads out).  The backward of K8a and of S^T A S: dX = S dP, dS = X dP^T + T dQ^T + U dQ, and S dQ for
 * the edge-weight gradient.  One output element per thread, summed in ascending order with fmaf: bits independent of the
 * grid.  A graph id outside [0, G) gives NaN.  Asynchronous.  Algorithmic bytes: N * 4 (C + K + 1) + G * C * K * 4. */
int tfgk_graph_rmm_f32(const float *Y, int64_t ldy, const int32_t *node_graph, int32_t N, const float *B, int64_t ldb,
                       int32_t G, int32_t C, int32_t K, int trans, float beta, float *out, int64_t ldo, void *stream);

/* ---- K9: padded row gather (nn/conv/graph_sage.py:319-337 lstm_graph_sage, utils/graph_utils.py:215-249
 * convert_x_to_3d): the rows of every CSR row r, in slot order, zero-padded to a width of K --------------------------- */

enum tfgk_pad_layout { TFGK_PAD_ROW_MAJOR = 0, TFGK_PAD_STEP_MAJOR = 1 };

/* out[r, j, :] = X[src[rowptr[r] + j], :] for j < min(deg r, K), zeros for every other j < K; r < R, D columns.
 * layout TFGK_PAD_ROW_MAJOR: out is [R, K, D]; TFGK_PAD_STEP_MAJOR: out is [K, R, D] (the input order of a sequence-major
 * recurrence).  out is dense (leading dimension D); X is [NX, D] with leading dimension ldx (column slices are fine).
 * src is csr.col (neighbour rows) or csr.perm (the data rows of a segment-id CSR).  A padded slot is never read; a src
 * id outside [0, NX) gives its output row NaN.  slot_out (may be NULL) receives, for every slot p of row r with
 * j = p - rowptr[r], the flat output row of that slot: r * K + j (row-major) or j * R + r (step-major), -1 for j >= K;
 * it needs K * R < 2^31.  A pure copy: bit-exact.  16-byte loads and stores when X, ldx, D and out are aligned, scalar
 * otherwise.  Asynchronous.  Algorithmic bytes: R * K * D * 4 written, kept * (4 D + 4) read, R * 8 for rowptr. */
int tfgk_pad_rows_f32(const int64_t *rowptr, const int32_t *src, int32_t R, int32_t K, int layout, const float *X,
                      int64_t ldx, int32_t NX, int32_t D, float *out, int32_t *slot_out, void *stream);

/* Backward of the convert_x_to_3d case (src = perm): for every slot p of row r, j = p - rowptr[r],
 *   out[perm[p], :] = j < K ? G[r * K + j, :] : 0          G [R, K, D] row-major, out [nnz, D], both dense.
 * Every output row whose index appears in perm is written exactly once (truncated rows become 0); no atomics.  A perm
 * entry outside [0, n_out) is skipped.  Asynchronous.  Algorithmic bytes: kept * 8 D + (nnz - kept) * 4 D + nnz * 4. */
int tfgk_unpad_rows_f32(const int64_t *rowptr, const int32_t *perm, int32_t R, int32_t K, const float *G, int32_t D,
                        float *out, int64_t n_out, void *stream);

/* ---- K10: sparse x sparse product C = A B of two CSR matrices (nn/pool/cluster_pool.py:32-34, S^T A S) --------------
 * A is [M, K] and B [K, Ncol], both CSR (rowptr int64, col int32, val f32; columns in any order, duplicates allowed).
 * C is CSR with ascending columns in every row, duplicates merged, every structurally present entry kept (exact zeros
 * too).  C[i, j] is the fp32 sum of the products a_ik * b_kj in production order (A's row i left to right, then B's row k
 * left to right): ((p_0 + p_1) + p_2) + ..., no fused multiply-add, no atomics, so the bits depend only on the inputs
 * (not on the grid, the chunking or the tier).  One CTA per row expands the products, sorts them stably by column and
 * sums every run.  A row with more than TFGK_SPGEMM_SHARED_PRODUCTS products is "big": its expansion goes to the caller's
 * workspace instead of shared memory.
 *   _plan      prod_ptr[M+1] = exclusive scan of the products per row, big_ptr[M+1] = the same over big rows only (0 for
 *              the others); both are also copied to the host arrays.  Synchronises once.  A column id of A outside
 *              [0, K) or of B outside [0, Ncol) returns TFGK_ERR_INDEX_OUT_OF_RANGE (nothing is read through it); a row
 *              with 2^31 or more products TFGK_ERR_UNSUPPORTED.
 *   _count     c_count[i] = distinct columns of C's row i for the rows [row0, row1).  Asynchronous.
 *   _rowptr    c_rowptr[M+1] = exclusive scan of c_count; *nnz_host = nnz(C).  Synchronises once.
 *   _fill_f32  C's columns and values of the rows [row0, row1).  Asynchronous.
 * _count and _fill_f32 take the big-row products of their row range, big_products = big_ptr[row1] - big_ptr[row0], and a
 * workspace of tfgk_spgemm_rows_workspace_bytes(big_products); the caller cuts the rows into ranges whose expansion fits
 * its budget (a single row larger than the budget is a range on its own).
 * Algorithmic bytes of _fill_f32: A (8 per row, 8 per entry) + B's row offsets (16 per A entry) + B's column and value
 * (8 per product) + C (8 per row read, 8 per entry written). */
#define TFGK_SPGEMM_SHARED_PRODUCTS 2048
int tfgk_spgemm_plan_workspace_bytes(int32_t M, size_t *out_bytes);
int tfgk_spgemm_plan(const int64_t *a_rowptr, const int32_t *a_col, int32_t M, int32_t K, const int64_t *b_rowptr,
                     const int32_t *b_col, int32_t Ncol, int64_t *prod_ptr, int64_t *big_ptr, int64_t *prod_ptr_host,
                     int64_t *big_ptr_host, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_spgemm_rows_workspace_bytes(int64_t big_products, size_t *out_bytes);
int tfgk_spgemm_count(const int64_t *a_rowptr, const int32_t *a_col, const int64_t *b_rowptr, const int32_t *b_col,
                      int32_t row0, int32_t row1, const int64_t *prod_ptr, const int64_t *big_ptr, int64_t big_products,
                      int64_t *c_count, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_spgemm_rowptr(const int64_t *c_count, int32_t M, int64_t *c_rowptr, int64_t *nnz_host, void *workspace,
                       size_t workspace_bytes, void *stream);
int tfgk_spgemm_fill_f32(const int64_t *a_rowptr, const int32_t *a_col, const float *a_val, const int64_t *b_rowptr,
                         const int32_t *b_col, const float *b_val, int32_t row0, int32_t row1, const int64_t *prod_ptr,
                         const int64_t *big_ptr, int64_t big_products, const int64_t *c_rowptr, int32_t *c_col,
                         float *c_val, void *workspace, size_t workspace_bytes, void *stream);

/* ---- K12: the gradient of K10's C = A B with respect to A's and B's values ------------------------------------------
 * A is [M, K], B [K, N], C [M, N] with ascending, unique columns in every row (K10's output), dC its upstream gradient in
 * C's value order.  For every CSR entry p of X, one row of Y is walked and dC is looked up in C:
 *   TFGK_SPGEMM_GRAD_LEFT   X = A, Y = B:    dA[p = (i, k)] = sum_{q in B.row(k)}   B.val[q]  * dC(i, B.col[q])
 *   TFGK_SPGEMM_GRAD_RIGHT  X = B, Y = A^T:  dB[p = (k, j)] = sum_{q in A^T.row(k)} At.val[q] * dC(At.col[q], j)
 * dC(r, c) is found by binary search over C's row r; a column the row does not hold contributes 0 (nothing is added).
 * Summation order, part of the contract: every product Y.val[q] * dC is rounded once (no fused multiply-add); a Y row is
 * cut into consecutive slices of TFGK_SPGEMM_GRAD_SLICE entries; a slice sums its products from +0 in Y's CSR order and
 * the entry sums its slice sums from +0 in slice order.  The bits therefore depend only on the inputs (not on the grid
 * or on which threads take the slices); no atomics; out[x_perm ? x_perm[p] : p] is written exactly once per entry
 * (x_perm, X's CSR slot -> COO position map, lands the gradient in X's COO order).
 *   _plan  slice_ptr[nnz_x + 1] = exclusive scan over X's entries of their slice counts, 0 for an entry whose Y row has
 *          at most TFGK_SPGEMM_GRAD_SLICE entries (one thread takes it whole) and ceil(len / SLICE) otherwise (the slices
 *          are spread over threads); *n_slices_host = their total.  Decided from row lengths alone.  A column id of X
 *          outside [0, K) (left) / [0, N) (right), or of Y outside [0, N) / [0, M), returns TFGK_ERR_INDEX_OUT_OF_RANGE.
 *          Synchronises once.
 *   _f32   the gradient, given the plan and `partial`, a scratch of n_slices floats.  Asynchronous.
 * X's rowptr must end at nnz_x.  Nothing per product is stored.  Algorithmic bytes of _f32 (products = sum over X's
 * entries of their Y row lengths): X (8 per row, 16 per entry: col, slice_ptr, out, [+4 perm]) + Y's row offsets (16 per
 * entry) + Y's column and value and the matching C column and dC (16 per product) + C's row offsets (16 per entry left,
 * 16 per product right) + 8 per hub slice. */
#define TFGK_SPGEMM_GRAD_SLICE 64
enum tfgk_spgemm_grad_mode { TFGK_SPGEMM_GRAD_LEFT = 0, TFGK_SPGEMM_GRAD_RIGHT = 1 };
int tfgk_spgemm_grad_workspace_bytes(int64_t nnz_x, size_t *out_bytes);
int tfgk_spgemm_grad_plan(int mode, const int64_t *x_rowptr, const int32_t *x_col, int64_t nnz_x, const int64_t *y_rowptr,
                          const int32_t *y_col, int32_t M, int32_t K, int32_t N, int64_t *slice_ptr,
                          int64_t *n_slices_host, void *workspace, size_t workspace_bytes, void *stream);
int tfgk_spgemm_grad_f32(int mode, const int64_t *x_rowptr, const int32_t *x_col, const int32_t *x_perm, int64_t nnz_x,
                         const int64_t *y_rowptr, const int32_t *y_col, const float *y_val, int32_t M, int32_t K, int32_t N,
                         const int64_t *c_rowptr, const int32_t *c_col, const float *dC, const int64_t *slice_ptr,
                         int64_t n_slices, float *partial, float *out, void *stream);

/* ---- K11: max aggregation with tie counts, and its backward over the transposed CSR --------------------------------
 * (max_pool_graph_sage and aggregate_neighbors(max_reducer) training, ASAP's query; graph_sage.py:228-287) */

/* K11a.  out[r,d] = max_{e in row r} w[e] * h[col[e],d]   (w NULL = 1; an empty row gives -FLT_MAX)
 *        cnt[r,d] = #{e in row r : w[e] * h[col[e],d] == out[r,d]}, int32, IEEE equality: +0 and -0 are ties, NaN never
 *        counts, and -inf is no tie of an empty row's -FLT_MAX.
 * out is bit-identical to tfgk_spmm_f32(reduce = MAX, alpha = 1, no epilogue) with the same CSR, weights and plan: fmaxf
 * in CSR order from -FLT_MAX, products rounded once, and the plan taken exactly where tfgk_spmm_f32 takes it for the same
 * h and out (16-byte aligned rows, D % 4 == 0, 32 <= D <= 512), its hub slices merged as (max, count) pairs in slice order.
 * Any D; rows that are not 16-byte aligned or D % 4 != 0 take a scalar path.  The plan's scratch must hold
 * n_slots * D * 8 bytes.  Counts are exact up to 2^31 - 1 ties.  No atomics.  Asynchronous.
 * Algorithmic bytes: E*(4*D + 4 [+4 weighted]) + N*(8*D + 8). */
int tfgk_spmm_max_f32(const int64_t *rowptr, const int32_t *col, const float *w, const float *h, int64_t ldh,
                      int32_t n_dst, int32_t D, float *out, int64_t ldo, int32_t *cnt, int64_t ldc,
                      const tfgk_plan *plan, void *stream);
/* K11b.  The gradient of K11a's out with respect to h, given g = dL/dout, over the TRANSPOSED CSR: row c of rowptr_t lists
 * the edges leaving source c in stable edge order, dst_t[p] their destination rows and w_t[p] their weights (NULL = 1):
 *     dh[c,d] = sum_p ((Gn[r,d] * sel) * w_t[p]),   r = dst_t[p],  sel = (w_t[p] * h[c,d] == out[r,d]) ? 1 : 0,
 *     Gn = g / max(cnt, 1)   (fp32, correctly rounded; written with out into pk = [out | Gn], [n_dst, 2D] contiguous).
 * Every edge adds its term, selected or not, so an inf or NaN in g reaches every neighbour of its row (0 * inf = NaN),
 * as the product of the gradient with the 0/1 selection does.  Sums start at 0 and run in edge order with separate
 * roundings; sources with hub out-degree are summed in the plan's slices (plan taken where tfgk_spmm_f32 takes it for a
 * dense [E, D] table: D % 4 == 0, 32 <= D <= 512; scratch n_slots * D * 4 bytes) and merged in slice order.  dh is
 * therefore bit-identical to gathering h, reducing with SegmentReduce(max) and summing the message gradient with K1
 * (TakeRows).  Every dh row of [0, n_src) is written once; no atomics.  Asynchronous.
 * Algorithmic bytes: E*(8*D + 4 [+4 weighted]) + N*(8*D + 8), plus 20*D*N for the pass writing pk. */
int tfgk_spmm_max_bwd_f32(const int64_t *rowptr_t, const int32_t *dst_t, const float *w_t, const float *h, int64_t ldh,
                          int32_t n_src, int32_t n_dst, int32_t D, const float *out, int64_t ldo, const int32_t *cnt,
                          int64_t ldc, const float *g, int64_t ldg, float *pk, float *dh, int64_t lddh,
                          const tfgk_plan *plan, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* TFGK_H_ */
