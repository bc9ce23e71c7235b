// K10, the product of two CSR matrices C = A B (the S^T A S of nn/pool/cluster_pool.py:32-34, which the reference
// computes by densifying the N x N adjacency of the whole batch).
//
// Gustavson order, made deterministic by sorting instead of hashing.  Every output row i is computed by one CTA in three
// steps:
//   expand   : the products a_ik * b_kj in the order they are produced (A's row i left to right, then B's row k left to
//              right), each with the 64-bit key (j << 32 | position);
//   sort     : a bitonic sort of the keys.  The position in the low half makes every key distinct, so the sorted order
//              is the stable order by column: equal columns keep their production order;
//   compress : the first slot of every run of equal columns sums the run left to right in fp32 (__fadd_rn, no
//              contraction) and writes one output entry.
// So C[i, j] = ((p_0 + p_1) + p_2) + ... over the products of (i, j) in production order, whatever the grid, the chunking or
// the tier; no atomics.  The row's expansion lives in shared memory when it has at most TFGK_SPGEMM_SHARED_PRODUCTS
// products, and otherwise in the caller's workspace (the rows are then "big"; the workspace holds 2 x the products of
// the big rows of one launch, as the sort pads to a power of two).  Both tiers run the same code on generic pointers.
//
// The product runs in four calls: _plan (products per row, validation, one synchronisation), _count per chunk of rows
// (distinct columns per row), _rowptr (C's row offsets and nnz, one synchronisation) and _fill_f32 per chunk.  The caller
// cuts the rows into chunks whose expansion fits its budget, which bounds the workspace of the chunk's big rows.
#include "common.cuh"
#include "scan.cuh"

namespace tfgk {
namespace {

constexpr int kRowThreads = 256;
constexpr int kShared = TFGK_SPGEMM_SHARED_PRODUCTS;
constexpr int64_t kMaxRowProducts = 1ll << 31;      // the position must fit the low half of the key

// products per row of A, big-row products (0 for rows that fit shared memory), and the validation of A's column ids
__global__ void spgemm_rowprod_kernel(const int64_t *__restrict__ a_rowptr, const int32_t *__restrict__ a_col, int32_t M,
                                      int32_t K, const int64_t *__restrict__ b_rowptr, int64_t *__restrict__ prod,
                                      int64_t *__restrict__ big, int32_t *__restrict__ flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t s = 0;
        bool bad = false;
        for (int64_t ka = a_rowptr[i]; ka < a_rowptr[i + 1]; ++ka) {
            const int32_t k = a_col[ka];
            if (k < 0 || k >= K) { bad = true; continue; }
            s += b_rowptr[k + 1] - b_rowptr[k];
        }
        if (bad) { flag[0] = 1; s = 0; }
        if (s >= kMaxRowProducts) { flag[1] = 1; s = 0; }
        prod[i] = s;
        big[i] = s > kShared ? s : 0;
    }
}

__global__ void spgemm_check_cols_kernel(const int64_t *__restrict__ b_rowptr, int32_t K, const int32_t *__restrict__ b_col,
                                         int32_t Ncol, int32_t *__restrict__ flag) {
    const int64_t nnz = b_rowptr[K];
    for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t j = b_col[e];
        if (j < 0 || j >= Ncol) flag[0] = 1;
    }
}

// exclusive prefix count of `v` over the CTA; `total` receives the CTA's count.  `buf` holds kRowThreads / 32 ints.
__device__ __forceinline__ int block_exclusive_count(bool v, int *buf, int &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned mask = __ballot_sync(0xffffffffu, v);
    if (lane == 0) buf[wid] = __popc(mask);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < kRowThreads / 32; ++w) {
        const int c = buf[w];
        if (w < wid) before += c;
        sum += c;
    }
    __syncthreads();                                 // buf is reused by the next call
    total = sum;
    return before + __popc(mask & ((1u << lane) - 1u));
}

template <bool FILL>
__global__ void __launch_bounds__(kRowThreads) spgemm_rows_kernel(
    const int64_t *__restrict__ a_rowptr, const int32_t *__restrict__ a_col, const float *__restrict__ a_val,
    const int64_t *__restrict__ b_rowptr, const int32_t *__restrict__ b_col, const float *__restrict__ b_val,
    int32_t row0, const int64_t *__restrict__ prod_ptr, const int64_t *__restrict__ big_ptr,
    int64_t *__restrict__ c_count, const int64_t *__restrict__ c_rowptr, int32_t *__restrict__ c_col,
    float *__restrict__ c_val, uint64_t *ws_keys, float *ws_vals) {
    __shared__ uint64_t s_keys[kShared];
    __shared__ float s_vals[FILL ? kShared : 1];
    __shared__ int s_buf[kRowThreads / 32];
    const int32_t i = row0 + (int32_t)blockIdx.x;
    const int64_t n = prod_ptr[i + 1] - prod_ptr[i];
    if (n == 0) {
        if (!FILL && threadIdx.x == 0) c_count[i] = 0;
        return;
    }
    int64_t m = 1;
    while (m < n) m <<= 1;
    uint64_t *keys = s_keys;
    float *vals = s_vals;
    if (n > kShared) {
        const int64_t off = 2 * (big_ptr[i] - big_ptr[row0]);
        keys = ws_keys + off;
        vals = ws_vals + off;
    }

    // expand in production order
    int64_t off = 0;
    for (int64_t ka = a_rowptr[i]; ka < a_rowptr[i + 1]; ++ka) {
        const int32_t k = a_col[ka];
        const float av = FILL ? a_val[ka] : 0.0f;
        const int64_t b0 = b_rowptr[k], len = b_rowptr[k + 1] - b0;
        for (int64_t j = threadIdx.x; j < len; j += kRowThreads) {
            const int64_t p = off + j;
            keys[p] = ((uint64_t)(uint32_t)b_col[b0 + j] << 32) | (uint64_t)(uint32_t)p;
            if (FILL) vals[p] = __fmul_rn(av, b_val[b0 + j]);
        }
        off += len;
    }
    for (int64_t p = n + threadIdx.x; p < m; p += kRowThreads) keys[p] = ~0ull;
    __syncthreads();

    // bitonic sort of the distinct keys: the stable order by column
    for (int64_t k = 2; k <= m; k <<= 1) {
        for (int64_t j = k >> 1; j > 0; j >>= 1) {
            for (int64_t p = threadIdx.x; p < m; p += kRowThreads) {
                const int64_t q = p ^ j;
                if (q > p) {
                    const uint64_t a = keys[p], b = keys[q];
                    if ((a > b) == ((p & k) == 0)) {
                        keys[p] = b;
                        keys[q] = a;
                    }
                }
            }
            __syncthreads();
        }
    }

    // compress: one output entry per run of equal columns, summed in production order
    const int64_t base = FILL ? c_rowptr[i] : 0;
    int64_t carry = 0;
    for (int64_t t0 = 0; t0 < n; t0 += kRowThreads) {
        const int64_t p = t0 + threadIdx.x;
        const uint32_t col = p < n ? (uint32_t)(keys[p] >> 32) : 0u;
        const bool head = p < n && (p == 0 || (uint32_t)(keys[p - 1] >> 32) != col);
        int total = 0;
        const int rank = block_exclusive_count(head, s_buf, total);
        if (FILL && head) {
            float acc = vals[(uint32_t)keys[p]];
            for (int64_t q = p + 1; q < n && (uint32_t)(keys[q] >> 32) == col; ++q)
                acc = __fadd_rn(acc, vals[(uint32_t)keys[q]]);
            c_col[base + carry + rank] = (int32_t)col;
            c_val[base + carry + rank] = acc;
        }
        carry += total;
    }
    if (!FILL && threadIdx.x == 0) c_count[i] = carry;
}

// ---- K12: the gradient of C = A B with respect to A's and B's values ----
//
// Both modes walk, for every CSR entry p of X, one row of Y and look the values of dC up in C:
//   left  (X = A, Y = B):   dA[p = (i, k)] = sum_{q in B.row(k)}  B.val[q]  * dC(i, B.col[q])
//   right (X = B, Y = A^T): dB[p = (k, j)] = sum_{q in At.row(k)} At.val[q] * dC(At.col[q], j)
// A Y row is cut into slices of kSlice entries; a slice sums its products (each rounded once) from +0 in Y's order, and
// the entry sums its slices from +0 in slice order.  Entries with one slice are computed by one thread in one pass; the
// slices of longer rows ("hub" entries, listed by the plan from row lengths alone) are spread over threads, write their
// partial sums to the caller's scratch, and the entry pass adds them in order.  Same bits either way; no atomics.

constexpr int kSlice = TFGK_SPGEMM_GRAD_SLICE;
constexpr int kLookups = 4;                              // binary searches of C in flight per thread

// largest r in [0, n) with ptr[r] <= v, given ptr[0] <= v < ptr[n] (the row, or the entry, that holds v)
__device__ __forceinline__ int64_t last_le(const int64_t *__restrict__ ptr, int64_t n, int64_t v) {
    int64_t lo = 0, len = n;
    while (len > 1) {
        const int64_t half = len >> 1;
        if (ptr[lo + half] <= v) {
            lo += half;
            len -= half;
        } else {
            len = half;
        }
    }
    return lo;
}

// sum of the products of Y's entries [q0, q1) with dC.  LEFT: C's row is [c0, c1) and the column is y_col[q]; right: C's
// row is y_col[q] and the column is j.  A column C's row does not hold contributes 0.
template <bool LEFT>
__device__ float grad_slice_sum(const int32_t *__restrict__ y_col, const float *__restrict__ y_val, int64_t q0, int64_t q1,
                                const int64_t *__restrict__ c_rowptr, const int32_t *__restrict__ c_col,
                                const float *__restrict__ dC, int64_t c0, int64_t c1, int32_t j) {
    float acc = 0.0f;
    for (int64_t q = q0; q < q1; q += kLookups) {
        int64_t lo[kLookups], len[kLookups];
        int32_t want[kLookups];
#pragma unroll
        for (int u = 0; u < kLookups; ++u) {
            lo[u] = 0;
            len[u] = 0;
            want[u] = 0;
            if (q + u < q1) {
                const int32_t yc = y_col[q + u];
                if (LEFT) {
                    lo[u] = c0;
                    len[u] = c1 - c0;
                    want[u] = yc;
                } else {
                    lo[u] = c_rowptr[yc];
                    len[u] = c_rowptr[yc + 1] - lo[u];
                    want[u] = j;
                }
            }
        }
        // the searches advance in lock step so that their loads overlap: last position with c_col <= want
        bool more = true;
        while (more) {
            more = false;
#pragma unroll
            for (int u = 0; u < kLookups; ++u) {
                if (len[u] > 1) {
                    const int64_t half = len[u] >> 1;
                    if (c_col[lo[u] + half] <= want[u]) lo[u] += half;
                    len[u] -= half;
                    more |= len[u] > 1;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kLookups; ++u)
            if (len[u] == 1 && c_col[lo[u]] == want[u]) acc = __fadd_rn(acc, __fmul_rn(y_val[q + u], dC[lo[u]]));
    }
    return acc;
}

// slices per X entry (0 when one thread takes the whole Y row) and the validation of X's column ids
template <bool LEFT>
__global__ void grad_plan_kernel(const int64_t *__restrict__ x_rowptr, const int32_t *__restrict__ x_col, int32_t n_x_rows,
                                 int64_t nnz_x, int32_t x_ncols, const int64_t *__restrict__ y_rowptr,
                                 int64_t *__restrict__ cnt, int32_t *__restrict__ flag) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < nnz_x; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t k = x_col[p];
        if (k < 0 || k >= x_ncols) {
            flag[0] = 1;
            cnt[p] = 0;
            continue;
        }
        const int64_t yr = LEFT ? (int64_t)k : last_le(x_rowptr, n_x_rows, p);
        const int64_t len = y_rowptr[yr + 1] - y_rowptr[yr];
        cnt[p] = len > kSlice ? (len + kSlice - 1) / kSlice : 0;
    }
}

template <bool LEFT>
__device__ __forceinline__ float grad_range(const int64_t *__restrict__ x_rowptr, const int32_t *__restrict__ x_col,
                                            int32_t n_x_rows, int64_t p, int64_t t, const int64_t *__restrict__ y_rowptr,
                                            const int32_t *__restrict__ y_col, const float *__restrict__ y_val,
                                            const int64_t *__restrict__ c_rowptr, const int32_t *__restrict__ c_col,
                                            const float *__restrict__ dC, bool whole) {
    const int64_t r = last_le(x_rowptr, n_x_rows, p);
    const int32_t k = x_col[p];
    const int64_t yr = LEFT ? (int64_t)k : r;
    const int64_t y_end = y_rowptr[yr + 1];
    const int64_t q0 = y_rowptr[yr] + (whole ? 0 : t * kSlice);
    const int64_t q1 = whole ? y_end : min(q0 + kSlice, y_end);
    if (LEFT) return grad_slice_sum<true>(y_col, y_val, q0, q1, c_rowptr, c_col, dC, c_rowptr[r], c_rowptr[r + 1], 0);
    return grad_slice_sum<false>(y_col, y_val, q0, q1, c_rowptr, c_col, dC, 0, 0, k);
}

// one thread per slice of the hub entries: partial[s]
template <bool LEFT>
__global__ void __launch_bounds__(256) grad_slices_kernel(
    const int64_t *__restrict__ x_rowptr, const int32_t *__restrict__ x_col, int32_t n_x_rows, int64_t nnz_x,
    const int64_t *__restrict__ y_rowptr, const int32_t *__restrict__ y_col, const float *__restrict__ y_val,
    const int64_t *__restrict__ c_rowptr, const int32_t *__restrict__ c_col, const float *__restrict__ dC,
    const int64_t *__restrict__ slice_ptr, int64_t n_slices, float *__restrict__ partial) {
    for (int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; s < n_slices; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = last_le(slice_ptr, nnz_x, s);
        partial[s] = grad_range<LEFT>(x_rowptr, x_col, n_x_rows, p, s - slice_ptr[p], y_rowptr, y_col, y_val, c_rowptr,
                                      c_col, dC, false);
    }
}

// one thread per X entry: the whole Y row, or the sum of the entry's slices in order
template <bool LEFT>
__global__ void __launch_bounds__(256) grad_entries_kernel(
    const int64_t *__restrict__ x_rowptr, const int32_t *__restrict__ x_col, const int32_t *__restrict__ x_perm,
    int32_t n_x_rows, int64_t nnz_x, const int64_t *__restrict__ y_rowptr, const int32_t *__restrict__ y_col,
    const float *__restrict__ y_val, const int64_t *__restrict__ c_rowptr, const int32_t *__restrict__ c_col,
    const float *__restrict__ dC, const int64_t *__restrict__ slice_ptr, const float *__restrict__ partial,
    float *__restrict__ out) {
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < nnz_x; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s0 = slice_ptr[p], s1 = slice_ptr[p + 1];
        float acc = 0.0f;
        if (s1 > s0) {
            for (int64_t s = s0; s < s1; ++s) acc = __fadd_rn(acc, partial[s]);
        } else {
            acc = grad_range<LEFT>(x_rowptr, x_col, n_x_rows, p, 0, y_rowptr, y_col, y_val, c_rowptr, c_col, dC, true);
        }
        out[x_perm ? (int64_t)x_perm[p] : p] = acc;
    }
}

struct GradWorkspace {
    size_t off_flag, off_cnt, off_sums, total;
    explicit GradWorkspace(int64_t nnz_x) {
        off_flag = 0;
        off_cnt = align_up(8);
        off_sums = off_cnt + align_up((size_t)nnz_x * 8 + 8);
        total = off_sums + scan_scratch_bytes(nnz_x + 1);
    }
};

// X's rows, X's column bound and Y's column bound of a mode (A is [M, K], B [K, N])
struct GradShape {
    int32_t x_rows, x_ncols, y_ncols;
    GradShape(int mode, int32_t M, int32_t K, int32_t N)
        : x_rows(mode == TFGK_SPGEMM_GRAD_LEFT ? M : K), x_ncols(mode == TFGK_SPGEMM_GRAD_LEFT ? K : N),
          y_ncols(mode == TFGK_SPGEMM_GRAD_LEFT ? N : M) {}
};

struct PlanWorkspace {
    size_t off_flag, off_prod, off_big, off_sums, total;
    explicit PlanWorkspace(int32_t M) {
        off_flag = 0;
        off_prod = align_up(8);
        off_big = off_prod + align_up((size_t)M * 8 + 8);
        off_sums = off_big + align_up((size_t)M * 8 + 8);
        total = off_sums + scan_scratch_bytes((int64_t)M + 1);
    }
};

int rows_common(const int64_t *a_rowptr, const int32_t *a_col, const int64_t *b_rowptr, const int32_t *b_col,
                int32_t row0, int32_t row1, const int64_t *prod_ptr, const int64_t *big_ptr, int64_t big_products,
                size_t workspace_bytes, void *workspace, const char *what) {
    TFGK_CHECK_ARG(row0 >= 0 && row1 >= row0, "%s: bad row range [%d, %d)", what, row0, row1);
    // a_col / b_col may be null when A / B have no entries: only the slots inside the row ranges are read
    TFGK_CHECK_ARG(a_rowptr && b_rowptr && prod_ptr && big_ptr, "%s: null pointer", what);
    size_t need = 0;
    tfgk_spgemm_rows_workspace_bytes(big_products, &need);
    if (need > 0 && (workspace == nullptr || workspace_bytes < need))
        return set_error(TFGK_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", what, workspace_bytes, need);
    return TFGK_OK;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_spgemm_plan_workspace_bytes(int32_t M, size_t *out_bytes) {
    TFGK_CHECK_ARG(M >= 0 && out_bytes, "spgemm_plan_workspace_bytes: bad M %d or null output", M);
    *out_bytes = PlanWorkspace(M).total;
    return TFGK_OK;
}

int tfgk_spgemm_rows_workspace_bytes(int64_t big_products, size_t *out_bytes) {
    TFGK_CHECK_ARG(big_products >= 0 && out_bytes, "spgemm_rows_workspace_bytes: bad size or null output");
    // keys (8 bytes) and values (4 bytes), twice the products: the sort pads every big row to a power of two
    *out_bytes = big_products ? align_up((size_t)big_products * 16) + align_up((size_t)big_products * 8) : 0;
    return TFGK_OK;
}

int tfgk_spgemm_plan(const int64_t *a_rowptr, const int32_t *a_col, int32_t M, int32_t K, const int64_t *b_rowptr,
                     const int32_t *b_col, int32_t Ncol, int64_t *prod_ptr, int64_t *big_ptr, int64_t *prod_ptr_host,
                     int64_t *big_ptr_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(M >= 0 && K >= 0 && Ncol >= 0, "spgemm_plan: negative M, K or Ncol");
    TFGK_CHECK_ARG(a_rowptr && b_rowptr && prod_ptr && big_ptr && prod_ptr_host && big_ptr_host,
                   "spgemm_plan: null pointer");
    const PlanWorkspace L(M);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "spgemm_plan: workspace too small (%zu < %zu bytes)", workspace_bytes, L.total);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int64_t *prod = reinterpret_cast<int64_t *>(ws + L.off_prod);
    int64_t *big = reinterpret_cast<int64_t *>(ws + L.off_big);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + L.off_sums);
    TFGK_CUDA(cudaMemsetAsync(flag, 0, 8, st));
    if (M > 0) {
        spgemm_rowprod_kernel<<<grid_for(M), 256, 0, st>>>(a_rowptr, a_col, M, K, b_rowptr, prod, big, flag);
        TFGK_LAUNCH_CHECK();
    }
    if (K > 0) {
        // nnz(B) is only known on the device: a grid of 4 CTAs per SM strides over it
        spgemm_check_cols_kernel<<<(unsigned)sm_count() * 4, 256, 0, st>>>(b_rowptr, K, b_col, Ncol, flag);
        TFGK_LAUNCH_CHECK();
    }
    int rc = exclusive_scan<int64_t, int64_t>(prod, M, (int64_t)M + 1, prod_ptr, sums, st);
    if (rc != TFGK_OK) return rc;
    rc = exclusive_scan<int64_t, int64_t>(big, M, (int64_t)M + 1, big_ptr, sums, st);
    if (rc != TFGK_OK) return rc;
    int32_t bad[2] = {0, 0};
    TFGK_CUDA(cudaMemcpyAsync(bad, flag, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(prod_ptr_host, prod_ptr, ((size_t)M + 1) * 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(big_ptr_host, big_ptr, ((size_t)M + 1) * 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (bad[0])
        return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "spgemm_plan: a column id of A is outside [0, %d) or of B outside [0, %d)",
                         K, Ncol);
    if (bad[1]) return set_error(TFGK_ERR_UNSUPPORTED, "spgemm_plan: a row of C has 2^31 or more products");
    return TFGK_OK;
}

int tfgk_spgemm_count(const int64_t *a_rowptr, const int32_t *a_col, const int64_t *b_rowptr, const int32_t *b_col,
                      int32_t row0, int32_t row1, const int64_t *prod_ptr, const int64_t *big_ptr, int64_t big_products,
                      int64_t *c_count, void *workspace, size_t workspace_bytes, void *stream) {
    int rc = rows_common(a_rowptr, a_col, b_rowptr, b_col, row0, row1, prod_ptr, big_ptr, big_products, workspace_bytes,
                         workspace, "spgemm_count");
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(c_count, "spgemm_count: null c_count");
    if (row1 == row0) return TFGK_OK;
    uint64_t *keys = static_cast<uint64_t *>(workspace);
    float *vals = big_products ? reinterpret_cast<float *>(static_cast<char *>(workspace) + align_up((size_t)big_products * 16))
                               : nullptr;
    spgemm_rows_kernel<false><<<(unsigned)(row1 - row0), kRowThreads, 0, as_stream(stream)>>>(
        a_rowptr, a_col, nullptr, b_rowptr, b_col, nullptr, row0, prod_ptr, big_ptr, c_count, nullptr, nullptr, nullptr,
        keys, vals);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_spgemm_rowptr(const int64_t *c_count, int32_t M, int64_t *c_rowptr, int64_t *nnz_host, void *workspace,
                       size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(M >= 0 && c_rowptr && nnz_host && (M == 0 || c_count), "spgemm_rowptr: bad M or null pointer");
    const size_t need = scan_scratch_bytes((int64_t)M + 1);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "spgemm_rowptr: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    const int rc = exclusive_scan<int64_t, int64_t>(c_count, M, (int64_t)M + 1, c_rowptr,
                                                    static_cast<int64_t *>(workspace), st);
    if (rc != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(nnz_host, c_rowptr + M, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

int tfgk_spgemm_fill_f32(const int64_t *a_rowptr, const int32_t *a_col, const float *a_val, const int64_t *b_rowptr,
                         const int32_t *b_col, const float *b_val, int32_t row0, int32_t row1, const int64_t *prod_ptr,
                         const int64_t *big_ptr, int64_t big_products, const int64_t *c_rowptr, int32_t *c_col,
                         float *c_val, void *workspace, size_t workspace_bytes, void *stream) {
    int rc = rows_common(a_rowptr, a_col, b_rowptr, b_col, row0, row1, prod_ptr, big_ptr, big_products, workspace_bytes,
                         workspace, "spgemm_fill");
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(a_val && b_val && c_rowptr && c_col && c_val, "spgemm_fill: null values or output");
    if (row1 == row0) return TFGK_OK;
    uint64_t *keys = static_cast<uint64_t *>(workspace);
    float *vals = big_products ? reinterpret_cast<float *>(static_cast<char *>(workspace) + align_up((size_t)big_products * 16))
                               : nullptr;
    spgemm_rows_kernel<true><<<(unsigned)(row1 - row0), kRowThreads, 0, as_stream(stream)>>>(
        a_rowptr, a_col, a_val, b_rowptr, b_col, b_val, row0, prod_ptr, big_ptr, nullptr, c_rowptr, c_col, c_val, keys,
        vals);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_spgemm_grad_workspace_bytes(int64_t nnz_x, size_t *out_bytes) {
    TFGK_CHECK_ARG(nnz_x >= 0 && out_bytes, "spgemm_grad_workspace_bytes: bad nnz_x or null output");
    *out_bytes = GradWorkspace(nnz_x).total;
    return TFGK_OK;
}

int tfgk_spgemm_grad_plan(int mode, const int64_t *x_rowptr, const int32_t *x_col, int64_t nnz_x, const int64_t *y_rowptr,
                          const int32_t *y_col, int32_t M, int32_t K, int32_t N, int64_t *slice_ptr,
                          int64_t *n_slices_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(mode == TFGK_SPGEMM_GRAD_LEFT || mode == TFGK_SPGEMM_GRAD_RIGHT, "spgemm_grad_plan: bad mode %d", mode);
    TFGK_CHECK_ARG(M >= 0 && K >= 0 && N >= 0 && nnz_x >= 0, "spgemm_grad_plan: negative M, K, N or nnz_x");
    TFGK_CHECK_ARG(x_rowptr && y_rowptr && slice_ptr && n_slices_host && (nnz_x == 0 || x_col),
                   "spgemm_grad_plan: null pointer");
    const GradWorkspace L(nnz_x);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "spgemm_grad_plan: workspace too small (%zu < %zu bytes)", workspace_bytes,
                         L.total);
    const GradShape S(mode, M, K, N);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int64_t *cnt = reinterpret_cast<int64_t *>(ws + L.off_cnt);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + L.off_sums);
    TFGK_CUDA(cudaMemsetAsync(flag, 0, 8, st));
    if (nnz_x > 0) {
        if (mode == TFGK_SPGEMM_GRAD_LEFT)
            grad_plan_kernel<true><<<grid_for(nnz_x), 256, 0, st>>>(x_rowptr, x_col, S.x_rows, nnz_x, S.x_ncols, y_rowptr,
                                                                     cnt, flag);
        else
            grad_plan_kernel<false><<<grid_for(nnz_x), 256, 0, st>>>(x_rowptr, x_col, S.x_rows, nnz_x, S.x_ncols, y_rowptr,
                                                                      cnt, flag);
        TFGK_LAUNCH_CHECK();
    }
    if (K > 0) {
        // Y has K rows in both modes; nnz(Y) is only known on the device
        spgemm_check_cols_kernel<<<(unsigned)sm_count() * 4, 256, 0, st>>>(y_rowptr, K, y_col, S.y_ncols, flag);
        TFGK_LAUNCH_CHECK();
    }
    const int rc = exclusive_scan<int64_t, int64_t>(cnt, nnz_x, nnz_x + 1, slice_ptr, sums, st);
    if (rc != TFGK_OK) return rc;
    int32_t bad[2] = {0, 0};
    TFGK_CUDA(cudaMemcpyAsync(bad, flag, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(n_slices_host, slice_ptr + nnz_x, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (bad[0])
        return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "spgemm_grad_plan: a column id of X is outside [0, %d) or of Y outside "
                         "[0, %d)", S.x_ncols, S.y_ncols);
    return TFGK_OK;
}

int tfgk_spgemm_grad_f32(int mode, const int64_t *x_rowptr, const int32_t *x_col, const int32_t *x_perm, int64_t nnz_x,
                         const int64_t *y_rowptr, const int32_t *y_col, const float *y_val, int32_t M, int32_t K, int32_t N,
                         const int64_t *c_rowptr, const int32_t *c_col, const float *dC, const int64_t *slice_ptr,
                         int64_t n_slices, float *partial, float *out, void *stream) {
    TFGK_CHECK_ARG(mode == TFGK_SPGEMM_GRAD_LEFT || mode == TFGK_SPGEMM_GRAD_RIGHT, "spgemm_grad: bad mode %d", mode);
    TFGK_CHECK_ARG(M >= 0 && K >= 0 && N >= 0 && nnz_x >= 0 && n_slices >= 0, "spgemm_grad: negative size");
    if (nnz_x == 0) return TFGK_OK;
    // y_col, y_val, c_col and dC may be null when Y or C have no entries: no slot outside the row ranges is read
    TFGK_CHECK_ARG(x_rowptr && x_col && y_rowptr && c_rowptr && slice_ptr && out && (n_slices == 0 || partial),
                   "spgemm_grad: null pointer");
    const GradShape S(mode, M, K, N);
    cudaStream_t st = as_stream(stream);
    const bool left = mode == TFGK_SPGEMM_GRAD_LEFT;
    if (n_slices > 0) {
        if (left)
            grad_slices_kernel<true><<<grid_for(n_slices), 256, 0, st>>>(x_rowptr, x_col, S.x_rows, nnz_x, y_rowptr, y_col,
                                                                          y_val, c_rowptr, c_col, dC, slice_ptr, n_slices,
                                                                          partial);
        else
            grad_slices_kernel<false><<<grid_for(n_slices), 256, 0, st>>>(x_rowptr, x_col, S.x_rows, nnz_x, y_rowptr, y_col,
                                                                           y_val, c_rowptr, c_col, dC, slice_ptr, n_slices,
                                                                           partial);
        TFGK_LAUNCH_CHECK();
    }
    if (left)
        grad_entries_kernel<true><<<grid_for(nnz_x), 256, 0, st>>>(x_rowptr, x_col, x_perm, S.x_rows, nnz_x, y_rowptr, y_col,
                                                                    y_val, c_rowptr, c_col, dC, slice_ptr, partial, out);
    else
        grad_entries_kernel<false><<<grid_for(nnz_x), 256, 0, st>>>(x_rowptr, x_col, x_perm, S.x_rows, nnz_x, y_rowptr,
                                                                     y_col, y_val, c_rowptr, c_col, dC, slice_ptr, partial,
                                                                     out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // extern "C"
