// Link prediction (SURVEY.md 8(f)5, demo/demo_gae.py): K6 edge scoring and exact negative sampling.
//
// K6 (tfgk_edge_dot_f32) replaces predict_edge of demo/demo_gae.py:53-60 (tf.gather of both endpoints, a product and
// reduce_sum): out[e] = sum_d h[row_e, d] * h[col_e, d].  Edge-parallel, no structure.  A group of G lanes owns one
// edge at a time and keeps U edges' rows in flight; each lane owns NC vectors of VEC columns per column chunk, sums
// them in a fixed order with fmaf, and the group finishes with an xor butterfly (fp addition is commutative, so every
// lane ends with the same bits).  G, NC, VEC and U depend only on D and the alignment of h, so an edge's result is a
// function of that edge and h alone: the same bits whatever E, the grid, or the edge's position in the list.
// Algorithmic bytes per launch: E * (8 D + 12)  (both rows counted once per use, two ids, one output).
//
// Negative sampling replaces utils/graph_utils.py:369-452.  The reference builds a dense N x N matrix and lists
// np.nonzero(np.triu(adj, 1)) with the positive pairs cleared; here that candidate list stays implicit.  With X_i the
// sorted distinct excluded columns of row i (a CSR built by the caller) and base_i the first column row i may use
// (i + 1 for the undirected list, 0 for the start-node list, whose X_a holds a itself), row i has
// (N - base_i) - |X_i| candidates in ascending column order, rows follow each other, and candidate k decodes as
//   i = the row whose int64 offset range holds k,  r = k - offset_i,
//   j = base_i + r + #{m : X_i[m] - base_i - m <= r}                       (both by binary search).
// Draws are counter-based (rng.cuh random_below64), so every output is a pure function of (seed, inputs).
#include "common.cuh"
#include "scan.cuh"
#include "rng.cuh"

namespace tfgk {
namespace {

constexpr int kDotThreads = 256;

// G lanes per edge, NC vectors of VEC floats per lane and column chunk, U edges in flight per group
template <int VEC, int G, int NC, int U>
__global__ void __launch_bounds__(kDotThreads) edge_dot_kernel(const float *__restrict__ h, int64_t ldh, int32_t N,
                                                               const int32_t *__restrict__ row,
                                                               const int32_t *__restrict__ col, int64_t E, int32_t D,
                                                               float *__restrict__ out) {
    constexpr int GPW = 32 / G;                 // groups per warp
    constexpr int CHUNK = G * NC * VEC;         // columns per pass of a group
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int grp = lane / G;
    const int64_t warp = ((int64_t)blockIdx.x * kDotThreads + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * kDotThreads) >> 5;
    // the loop bound is warp-uniform: the butterfly below needs every lane of the warp
    for (int64_t wb = warp * (GPW * U); wb < E; wb += n_warps * (GPW * U)) {
        const int64_t e0 = wb + (int64_t)grp * U;
        const float *pa[U];
        const float *pb[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int64_t e = e0 + u;
            int32_t r = 0, c = 0;
            ok[u] = e < E;
            if (ok[u]) {
                r = ld_stream_i32(row + e);
                c = ld_stream_i32(col + e);
                ok[u] = (uint32_t)r < (uint32_t)N && (uint32_t)c < (uint32_t)N;
            }
            pa[u] = h + (int64_t)(ok[u] ? r : 0) * ldh;
            pb[u] = h + (int64_t)(ok[u] ? c : 0) * ldh;
        }
        float s[U];
#pragma unroll
        for (int u = 0; u < U; ++u) s[u] = 0.0f;
        for (int c0 = 0; c0 < D; c0 += CHUNK) {
            float a[U][NC][VEC], b[U][NC][VEC];
#pragma unroll
            for (int u = 0; u < U; ++u) {
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    const int off = c0 + (gl + k * G) * VEC;
                    if (ok[u] && off < D) {
                        if constexpr (VEC == 4) {
                            const float4 x = __ldg(reinterpret_cast<const float4 *>(pa[u] + off));
                            const float4 y = __ldg(reinterpret_cast<const float4 *>(pb[u] + off));
                            a[u][k][0] = x.x; a[u][k][1] = x.y; a[u][k][2] = x.z; a[u][k][3] = x.w;
                            b[u][k][0] = y.x; b[u][k][1] = y.y; b[u][k][2] = y.z; b[u][k][3] = y.w;
                        } else {
                            a[u][k][0] = __ldg(pa[u] + off);
                            b[u][k][0] = __ldg(pb[u] + off);
                        }
                    } else {
#pragma unroll
                        for (int v = 0; v < VEC; ++v) a[u][k][v] = b[u][k][v] = 0.0f;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u)
#pragma unroll
                for (int k = 0; k < NC; ++k)
#pragma unroll
                    for (int v = 0; v < VEC; ++v) s[u] = fmaf(a[u][k][v], b[u][k][v], s[u]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
            for (int off = G / 2; off >= 1; off >>= 1) s[u] += __shfl_xor_sync(0xffffffffu, s[u], off, G);
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (gl == (u % G) && e0 + u < E) out[e0 + u] = ok[u] ? s[u] : __int_as_float(0x7fc00000);
    }
}

template <int VEC, int G, int NC, int U>
int launch_edge_dot(const float *h, int64_t ldh, int32_t N, const int32_t *row, const int32_t *col, int64_t E, int32_t D,
                    float *out, cudaStream_t st) {
    constexpr int per_cta = (kDotThreads / 32) * (32 / G) * U;       // edges per CTA per grid-stride step
    int64_t blocks = ceil_div64(E, per_cta);
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    edge_dot_kernel<VEC, G, NC, U><<<(unsigned)blocks, kDotThreads, 0, st>>>(h, ldh, N, row, col, E, D, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

// ---- negative sampling -------------------------------------------------------------------------------------------

__device__ __forceinline__ int64_t row_base(int mode, int64_t i) { return mode == TFGK_NEG_UPPER ? i + 1 : 0; }

// j = base + r + #{m : x[m] - base - m <= r}  (x ascending and distinct, all >= base)
__device__ __forceinline__ int32_t decode_in_row(const int32_t *__restrict__ x, int64_t len, int64_t base, int64_t r) {
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)x[mid] - base - mid <= r) lo = mid + 1;
        else hi = mid;
    }
    return (int32_t)(base + r + lo);
}

__global__ void neg_count_kernel(const int64_t *__restrict__ rowptr, int32_t N, int mode, int64_t *__restrict__ cnt) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = ((int64_t)N - row_base(mode, i)) - (rowptr[i + 1] - rowptr[i]);
        cnt[i] = c > 0 ? c : 0;
    }
}

__global__ void neg_draw_kernel(int64_t C, const int32_t *__restrict__ index, int64_t n, uint64_t seed, uint32_t stream,
                                uint32_t round, int64_t *__restrict__ k) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = index ? index[t] : t;
        k[s] = (int64_t)random_below64(seed, stream, ((uint64_t)round << 32) | (uint64_t)s, (uint64_t)C);
    }
}

__global__ void neg_dup_kernel(const int64_t *__restrict__ k, const int32_t *__restrict__ order, int64_t S,
                               int32_t *__restrict__ flag) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < S; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t s = order[p];
        flag[s] = (p > 0 && k[s] == k[order[p - 1]]) ? 1 : 0;
    }
}

__global__ void neg_decode_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col,
                                  const int64_t *__restrict__ offsets, int32_t N, int mode, const int64_t *__restrict__ k,
                                  int64_t S, int32_t *__restrict__ out_row, int32_t *__restrict__ out_col) {
    const int64_t C = offsets[N];
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (int64_t)gridDim.x * blockDim.x) {
        const int64_t kk = k[s];
        if (kk < 0 || kk >= C) {                  // not a candidate index: never decoded
            out_row[s] = -1;
            out_col[s] = -1;
            continue;
        }
        int64_t lo = 0, hi = N;                   // last row i with offsets[i] <= kk (rows without candidates are skipped)
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (offsets[mid] <= kk) lo = mid;
            else hi = mid;
        }
        const int64_t r0 = rowptr[lo];
        out_row[s] = (int32_t)lo;
        out_col[s] = decode_in_row(col + r0, rowptr[lo + 1] - r0, row_base(mode, lo), kk - offsets[lo]);
    }
}

__global__ void neg_start_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col, int32_t N,
                                 const int32_t *__restrict__ start, int64_t S, uint64_t seed, uint32_t stream,
                                 int32_t *__restrict__ out_col) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (int64_t)gridDim.x * blockDim.x) {
        const int32_t a = start[s];
        if ((uint32_t)a >= (uint32_t)N) { out_col[s] = -1; continue; }
        const int64_t r0 = rowptr[a], len = rowptr[a + 1] - r0;
        const int64_t cnt = (int64_t)N - len;
        if (cnt <= 0) { out_col[s] = -1; continue; }
        const int64_t r = (int64_t)random_below64(seed, stream, (uint64_t)s, (uint64_t)cnt);
        out_col[s] = decode_in_row(col + r0, len, 0, r);
    }
}

// both ends by 64-bit multiply-shift (draws 2 s and 2 s + 1: one Philox block per pair), uniform to within N / 2^64; a
// 32-bit multiply-shift over-weights 2^32 mod N of the ids by N / 2^32
__global__ void random_pairs_kernel(int32_t N, int64_t S, uint64_t seed, uint32_t stream, int32_t *__restrict__ out) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (int64_t)gridDim.x * blockDim.x) {
        out[s] = (int32_t)random_below64(seed, stream, 2 * (uint64_t)s, (uint64_t)N);
        out[S + s] = (int32_t)random_below64(seed, stream, 2 * (uint64_t)s + 1, (uint64_t)N);
    }
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_edge_dot_f32(const float *h, int64_t ldh, int32_t N, const int32_t *row, const int32_t *col, int64_t E, int32_t D,
                      float *out, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && E < (1ll << 31) - 1, "edge_dot: bad edge count %lld", (long long)E);
    TFGK_CHECK_ARG(N >= 0 && D >= 0, "edge_dot: negative N or D");
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(row && col && out, "edge_dot: null pointer");
    TFGK_CHECK_ARG(D == 0 || N == 0 || (h != nullptr && ldh >= D), "edge_dot: bad h (ldh %lld < D %d)", (long long)ldh, D);
    cudaStream_t st = as_stream(stream);
    if (D == 0 || N == 0) D = 0;              // empty rows: every in-range edge scores 0, the others NaN
    if (D > 0 && D % 4 == 0 && ldh % 4 == 0 && aligned16(h)) {
        if (D <= 16) return launch_edge_dot<4, 4, 1, 4>(h, ldh, N, row, col, E, D, out, st);
        if (D <= 32) return launch_edge_dot<4, 8, 1, 4>(h, ldh, N, row, col, E, D, out, st);
        if (D <= 64) return launch_edge_dot<4, 16, 1, 4>(h, ldh, N, row, col, E, D, out, st);
        if (D <= 128) return launch_edge_dot<4, 32, 1, 4>(h, ldh, N, row, col, E, D, out, st);
        return launch_edge_dot<4, 32, 2, 2>(h, ldh, N, row, col, E, D, out, st);
    }
    if (D <= 4) return launch_edge_dot<1, 4, 1, 4>(h, ldh, N, row, col, E, D, out, st);
    if (D <= 8) return launch_edge_dot<1, 8, 1, 4>(h, ldh, N, row, col, E, D, out, st);
    if (D <= 16) return launch_edge_dot<1, 16, 1, 4>(h, ldh, N, row, col, E, D, out, st);
    if (D <= 32) return launch_edge_dot<1, 32, 1, 4>(h, ldh, N, row, col, E, D, out, st);
    return launch_edge_dot<1, 32, 4, 2>(h, ldh, N, row, col, E, D, out, st);
}

int tfgk_neg_offsets_workspace_bytes(int32_t N, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && N >= 0, "neg_offsets_workspace_bytes: bad argument");
    *out_bytes = align_up(((size_t)N + 1) * 8) + scan_scratch_bytes((int64_t)N + 1) + 256;
    return TFGK_OK;
}

int tfgk_neg_offsets(const int64_t *rowptr, int32_t N, int mode, int64_t *offsets, int64_t *total_host, void *workspace,
                     size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(N >= 0, "neg_offsets: negative N");
    TFGK_CHECK_ARG(mode == TFGK_NEG_UPPER || mode == TFGK_NEG_START, "neg_offsets: unknown mode %d", mode);
    TFGK_CHECK_ARG(offsets && total_host, "neg_offsets: null pointer");
    *total_host = 0;
    cudaStream_t st = as_stream(stream);
    if (N == 0) {
        TFGK_CUDA(cudaMemsetAsync(offsets, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr != nullptr, "neg_offsets: null rowptr");
    size_t need = 0;
    tfgk_neg_offsets_workspace_bytes(N, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "neg_offsets: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    char *ws = static_cast<char *>(workspace);
    int64_t *cnt = reinterpret_cast<int64_t *>(ws);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + align_up(((size_t)N + 1) * 8));
    neg_count_kernel<<<grid_for(N), 256, 0, st>>>(rowptr, N, mode, cnt);
    TFGK_LAUNCH_CHECK();
    const int rc = exclusive_scan<int64_t, int64_t>(cnt, N, (int64_t)N + 1, offsets, sums, st);
    if (rc != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(total_host, offsets + N, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

int tfgk_neg_draw(int64_t C, const int32_t *index, int64_t n, uint64_t seed, uint32_t rng_stream, int32_t round, int64_t *k,
                  void *stream) {
    TFGK_CHECK_ARG(C > 0 && n >= 0 && n < (1ll << 31) - 1 && round >= 0, "neg_draw: bad argument");
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(k != nullptr, "neg_draw: null output");
    neg_draw_kernel<<<grid_for(n), 256, 0, as_stream(stream)>>>(C, index, n, seed, rng_stream, (uint32_t)round, k);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_neg_dup_flags(const int64_t *k, const int32_t *order, int64_t S, int32_t *flag, void *stream) {
    TFGK_CHECK_ARG(S >= 0 && S < (1ll << 31) - 1, "neg_dup_flags: bad size");
    if (S == 0) return TFGK_OK;
    TFGK_CHECK_ARG(k && order && flag, "neg_dup_flags: null pointer");
    neg_dup_kernel<<<grid_for(S), 256, 0, as_stream(stream)>>>(k, order, S, flag);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_neg_decode(const int64_t *rowptr, const int32_t *col, const int64_t *offsets, int32_t N, int mode, const int64_t *k,
                    int64_t S, int32_t *out_row, int32_t *out_col, void *stream) {
    TFGK_CHECK_ARG(N >= 0 && S >= 0 && S < (1ll << 31) - 1, "neg_decode: bad size");
    TFGK_CHECK_ARG(mode == TFGK_NEG_UPPER || mode == TFGK_NEG_START, "neg_decode: unknown mode %d", mode);
    if (S == 0) return TFGK_OK;
    TFGK_CHECK_ARG(N > 0, "neg_decode: no nodes to decode into");
    TFGK_CHECK_ARG(rowptr && col && offsets && k && out_row && out_col, "neg_decode: null pointer");
    neg_decode_kernel<<<grid_for(S), 256, 0, as_stream(stream)>>>(rowptr, col, offsets, N, mode, k, S, out_row, out_col);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_neg_sample_start(const int64_t *rowptr, const int32_t *col, int32_t N, const int32_t *start, int64_t S,
                          uint64_t seed, uint32_t rng_stream, int32_t *out_col, void *stream) {
    TFGK_CHECK_ARG(N >= 0 && S >= 0 && S < (1ll << 31) - 1, "neg_sample_start: bad size");
    if (S == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && col && start && out_col, "neg_sample_start: null pointer");
    neg_start_kernel<<<grid_for(S), 256, 0, as_stream(stream)>>>(rowptr, col, N, start, S, seed, rng_stream, out_col);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_random_pairs_i32(int32_t N, int64_t S, uint64_t seed, uint32_t rng_stream, int32_t *out, void *stream) {
    TFGK_CHECK_ARG(N > 0 && S >= 0 && S < (1ll << 30), "random_pairs: bad argument (N %d, S %lld)", N, (long long)S);
    if (S == 0) return TFGK_OK;
    TFGK_CHECK_ARG(out != nullptr, "random_pairs: null output");
    random_pairs_kernel<<<grid_for(S), 256, 0, as_stream(stream)>>>(N, S, seed, rng_stream, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // extern "C"
