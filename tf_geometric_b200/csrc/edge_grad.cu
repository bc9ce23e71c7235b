// Gradients with respect to edge weights: K7, a sampled dense-dense product (SDDMM) over a destination-sorted CSR.
//
// For y_r = sum_{p in row r} w_p X[col_p] (K1 with reduce = sum, or mean with the 1 / max(cnt, 1) scale), the gradient of
// a loss with respect to the weight of slot p is <G[r], X[col_p]> (times the mean scale), with G = dL/dy.  K7 computes
//     out[perm ? perm[p] : p] = (alpha * row_scale[r]) * sum_d G[r, d] * X[col_p, d]
// for every slot p of every row r.  Unlike K6 (one table, both endpoints gathered per edge) the kernel walks the CSR, so
// G[r] is loaded once per row (kept in registers for D up to a few hundred) and only the X[col] rows are streamed.
//
// Work split: the CSR's edge range is cut into tasks of a fixed number of consecutive slots, one warp per task.  A warp
// finds the row holding its first slot with a 32-way search of rowptr (one ballot per level) and walks the rows from there;
// a row longer than a task (a hub) is therefore spread over several warps, and a task may span many short rows.  Each
// output is one edge, so nothing is reduced across warps: no atomics, no scratch, every output written exactly once.
//
// Inside a warp, a group of G lanes owns one edge at a time and keeps U edges' rows in flight; each lane owns NC vectors of
// VEC columns per column chunk, sums them in a fixed order with fmaf, and the group finishes with an xor butterfly.  G, NC,
// VEC and U depend only on D and on the alignment of G, X and their leading dimensions, so an edge's bits are a function
// of G[r], X[col], row_scale[r] and alpha alone: the same whatever the task size, the grid, or whether perm is given.
// Algorithmic bytes per launch: E * (4 D + 12)  (X row, col, perm, out)  +  N * (4 D + 8)  (G row, rowptr).
#include <stdlib.h>

#include "common.cuh"

namespace tfgk {
namespace {

constexpr int kSddmmThreads = 256;
constexpr int64_t kTaskEdgesDefault = 512;

// last row r in [0, n) with rowptr[r] <= e (the row holding slot e, skipping empty rows); rowptr[n] > e.
// Every lane returns the same value; the 32-way search costs one ballot per level (log32 N levels).
__device__ __forceinline__ int32_t find_row(const int64_t *__restrict__ rowptr, int32_t n, int64_t e, int lane) {
    int64_t lo = 0, hi = n;                       // rowptr[lo] <= e (rowptr[0] is the first slot), answer in [lo, hi)
    while (hi - lo > 1) {
        const int64_t span = hi - lo;
        const int64_t probe = span > 32 ? lo + (span * lane) / 32 : lo + lane;
        const bool ok = probe < hi && rowptr[probe] <= e;
        const unsigned mask = __ballot_sync(0xffffffffu, ok);       // monotone in lane; lane 0 (probe = lo) is set
        const int k = 31 - __clz(mask);
        const int64_t new_lo = span > 32 ? lo + (span * k) / 32 : lo + k;
        const int64_t new_hi = span > 32 ? (k == 31 ? hi : lo + (span * (k + 1)) / 32) : new_lo + 1;
        lo = new_lo;
        hi = new_hi;
    }
    return (int32_t)lo;
}

template <int VEC>
__device__ __forceinline__ void load_vec(const float *p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 x = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
    } else {
        v[0] = __ldg(p);
    }
}

// VEC floats per load, G lanes per edge, NC vectors per lane and column chunk, U edges in flight per group.
// RESIDENT: one chunk covers D, and G[r] is loaded once per row into registers; otherwise the G chunk is re-read (an L1
// hit) for every chunk of every edge group.  Both variants sum in the same order.
template <int VEC, int G, int NC, int U, bool RESIDENT>
__global__ void __launch_bounds__(kSddmmThreads) sddmm_csr_kernel(
    const int64_t *__restrict__ rowptr, const int32_t *__restrict__ col, const int32_t *__restrict__ perm, int32_t n_rows,
    const float *__restrict__ Gm, int64_t ldg, const float *__restrict__ X, int64_t ldx, int32_t D,
    const float *__restrict__ row_scale, float alpha, float *__restrict__ out, int64_t task_edges) {
    constexpr int GPW = 32 / G;                   // groups per warp
    constexpr int CHUNK = G * NC * VEC;           // columns per pass of a group
    constexpr int STEP = GPW * U;                 // edges per warp per iteration
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int grp = lane / G;
    const int64_t warp = ((int64_t)blockIdx.x * kSddmmThreads + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * kSddmmThreads) >> 5;
    const int64_t base = rowptr[0], end = rowptr[n_rows];
    const int64_t n_tasks = (end - base + task_edges - 1) / task_edges;
    // every loop bound below is warp-uniform: the butterfly and the ballot need every lane of the warp
    for (int64_t t = warp; t < n_tasks; t += n_warps) {
        const int64_t e0 = base + t * task_edges;
        const int64_t e1 = min(e0 + task_edges, end);
        int32_t r = find_row(rowptr, n_rows, e0, lane);
        int64_t p0 = e0;
        while (p0 < e1) {
            int64_t r_end = rowptr[r + 1];
            while (r_end <= p0) r_end = rowptr[++r + 1];           // empty rows hold no slot
            const int64_t p1 = min(r_end, e1);
            const float *g_row = Gm + (int64_t)r * ldg;
            const float f = row_scale ? alpha * row_scale[r] : alpha;
            float gr[NC][VEC];
            if constexpr (RESIDENT) {
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    const int off = (gl + k * G) * VEC;
                    if (off < D) load_vec<VEC>(g_row + off, gr[k]);
                    else
#pragma unroll
                        for (int v = 0; v < VEC; ++v) gr[k][v] = 0.0f;
                }
            }
            for (int64_t pb = p0; pb < p1; pb += STEP) {
                const float *px[U];
                bool ok[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int64_t p = pb + u * GPW + grp;
                    ok[u] = p < p1;
                    px[u] = X + (int64_t)(ok[u] ? ld_stream_i32(col + p) : 0) * ldx;
                }
                float s[U];
#pragma unroll
                for (int u = 0; u < U; ++u) s[u] = 0.0f;
                for (int c0 = 0; c0 < D; c0 += CHUNK) {
                    if constexpr (!RESIDENT) {
#pragma unroll
                        for (int k = 0; k < NC; ++k) {
                            const int off = c0 + (gl + k * G) * VEC;
                            if (off < D) load_vec<VEC>(g_row + off, gr[k]);
                            else
#pragma unroll
                                for (int v = 0; v < VEC; ++v) gr[k][v] = 0.0f;
                        }
                    }
                    float x[U][NC][VEC];
#pragma unroll
                    for (int u = 0; u < U; ++u)
#pragma unroll
                        for (int k = 0; k < NC; ++k) {
                            const int off = c0 + (gl + k * G) * VEC;
                            if (ok[u] && off < D) load_vec<VEC>(px[u] + off, x[u][k]);
                            else
#pragma unroll
                                for (int v = 0; v < VEC; ++v) x[u][k][v] = 0.0f;
                        }
#pragma unroll
                    for (int u = 0; u < U; ++u)
#pragma unroll
                        for (int k = 0; k < NC; ++k)
#pragma unroll
                            for (int v = 0; v < VEC; ++v) s[u] = fmaf(gr[k][v], x[u][k][v], s[u]);
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
#pragma unroll
                    for (int off = G / 2; off >= 1; off >>= 1) s[u] += __shfl_xor_sync(0xffffffffu, s[u], off, G);
                    const int64_t p = pb + u * GPW + grp;
                    if (ok[u] && gl == (u % G)) out[perm ? (int64_t)ld_stream_i32(perm + p) : p] = s[u] * f;
                }
            }
            p0 = p1;
        }
    }
}

template <int VEC, int G, int NC, int U, bool RESIDENT>
int launch_sddmm(const int64_t *rowptr, const int32_t *col, const int32_t *perm, int32_t n_rows, const float *Gm,
                 int64_t ldg, const float *X, int64_t ldx, int32_t D, const float *row_scale, float alpha, float *out,
                 int64_t task_edges, cudaStream_t st) {
    // the edge count lives on the device (rowptr[N]); reading it here would cost a synchronisation per call, so the grid
    // is the grid-stride cap and warps without a task exit after reading two words
    const unsigned blocks = (unsigned)sm_count() * 16;
    sddmm_csr_kernel<VEC, G, NC, U, RESIDENT><<<blocks, kSddmmThreads, 0, st>>>(
        rowptr, col, perm, n_rows, Gm, ldg, X, ldx, D, row_scale, alpha, out, task_edges);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

// slots per warp task: TFGK_SDDMM_TASK_EDGES overrides the default (a power of two is not required); a value larger than
// the edge count gives one task, i.e. no row is split
int64_t task_edges_setting() {
    const char *s = getenv("TFGK_SDDMM_TASK_EDGES");
    if (s == nullptr || *s == '\0') return kTaskEdgesDefault;
    const long long v = atoll(s);
    if (v < 32) return 32;
    return v > (1ll << 40) ? (1ll << 40) : (int64_t)v;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_sddmm_csr_f32(const int64_t *rowptr, const int32_t *col, const int32_t *perm, int32_t N_rows, const float *G,
                       int64_t ldg, const float *X, int64_t ldx, int32_t D, const float *row_scale, float alpha, float *out,
                       void *stream) {
    TFGK_CHECK_ARG(N_rows >= 0 && D >= 0, "sddmm_csr: negative N_rows or D");
    if (N_rows == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && col && out, "sddmm_csr: null rowptr, col or out");
    TFGK_CHECK_ARG(D == 0 || (G && X && ldg >= D && ldx >= D), "sddmm_csr: bad G / X (ldg %lld, ldx %lld, D %d)",
                   (long long)ldg, (long long)ldx, D);
    cudaStream_t st = as_stream(stream);
    const int64_t te = task_edges_setting();
#define TFGK_SDDMM(VEC, GL, NC, U, RES) \
    return launch_sddmm<VEC, GL, NC, U, RES>(rowptr, col, perm, N_rows, G, ldg, X, ldx, D, row_scale, alpha, out, te, st)
    if (D == 0) TFGK_SDDMM(1, 4, 1, 4, true);            // every slot scores alpha * scale * 0
    if (D % 4 == 0 && ldg % 4 == 0 && ldx % 4 == 0 && aligned16(G) && aligned16(X)) {
        if (D <= 16) TFGK_SDDMM(4, 4, 1, 4, true);
        if (D <= 32) TFGK_SDDMM(4, 8, 1, 4, true);
        if (D <= 64) TFGK_SDDMM(4, 16, 1, 4, true);
        if (D <= 128) TFGK_SDDMM(4, 32, 1, 4, true);
        if (D <= 256) TFGK_SDDMM(4, 32, 2, 2, true);
        if (D <= 512) TFGK_SDDMM(4, 32, 4, 2, true);
        TFGK_SDDMM(4, 32, 4, 2, false);
    }
    if (D <= 4) TFGK_SDDMM(1, 4, 1, 4, true);
    if (D <= 8) TFGK_SDDMM(1, 8, 1, 4, true);
    if (D <= 16) TFGK_SDDMM(1, 16, 1, 4, true);
    if (D <= 32) TFGK_SDDMM(1, 32, 1, 4, true);
    if (D <= 64) TFGK_SDDMM(1, 32, 2, 2, true);
    if (D <= 128) TFGK_SDDMM(1, 32, 4, 2, true);
    TFGK_SDDMM(1, 32, 4, 2, false);
#undef TFGK_SDDMM
}

}  // extern "C"
