// DiffPool / MinCutPool on the device: K8, the per-graph dense algebra of a batch whose nodes are assigned to C clusters
// per graph (nn/pool/cluster_pool.py:32-44 of the reference, which densifies the [G*C, N] assignment and the N x N
// adjacency instead).
//
// K8a, per-graph transposed product:  out[g*C + c, :] = sum_{n in g} S[n, c] * Y[n, :]
//   One launch gives S^T X (Y = X), S^T (A S) (Y = T = A S, from K1) or S^T S (Y = S).
//   Work split: every graph is cut into chunks of kChunkNodes consecutive node-list positions (an empty graph still has
//   one chunk, which writes zeros).  A task is (chunk, tile of TC clusters x TD columns) and is computed by one CTA: the
//   chunk's rows are staged through shared memory NB at a time and each thread keeps CT x DT accumulators, summing the
//   rows in node-list order with fmaf.  A graph with one chunk writes its block directly; the chunks of a larger graph
//   write partial blocks to the workspace, and a fix-up kernel adds them in chunk order.  So a one-graph MinCut over a
//   million nodes still spreads over the whole GPU, and a graph's bits depend only on its own rows (chunking is a
//   function of N_g alone): not on G, the grid, the tile shape or the other graphs.  No atomics.
//   The chunk prefix sums (which task belongs to which graph, where a split graph's partials go) are computed on the
//   device by a one-CTA scan, so the host never synchronises.
//
// K8b, row times its graph's block:  out[n, :] = beta * out[n, :] + Y[n, :] . B_g   (or . B_g^T)
//   with B_g the [C, K] block of rows g(n)*C .. g(n)*C + C - 1 of a block-layout matrix.  It gives dX = S dP,
//   dS = X dP^T + T dQ^T + U dQ and S dQ (for the edge-weight gradient through K7).  One thread per output element sums
//   over k in ascending order with fmaf, so rows are independent and the bits do not depend on the grid either.
#include "common.cuh"

namespace tfgk {
namespace {

constexpr int kTmmThreads = 256;           // 8 cluster rows x 32 column lanes
constexpr int kChunkNodes = 1024;          // node-list positions per K8a task
constexpr int kStageRows = 32;             // rows staged in shared memory at a time
constexpr int kPlanThreads = 1024;

// exclusive prefix sum over the 1024 threads of the block; `total` receives the block sum.  `buf` holds 32 int64.
__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t *buf, int64_t &total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int64_t x = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, off);
        if (lane >= off) x += y;
    }
    if (lane == 31) buf[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int64_t w = buf[lane];
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, w, off);
            if (lane >= off) w += y;
        }
        buf[lane] = w;
    }
    __syncthreads();
    const int64_t before = wid > 0 ? buf[wid - 1] : 0;
    total = buf[31];
    __syncthreads();                         // buf is reused by the next call
    return before + x - v;
}

// chunk_ptr[g] = chunks before graph g (chunk_ptr[G] = all), split_ptr[g] = workspace slots before g (only graphs with more
// than one chunk own slots), split_list = the graphs with more than one chunk in ascending order, meta[0] = how many.
__global__ void __launch_bounds__(kPlanThreads, 1) tmm_plan_kernel(const int64_t *__restrict__ gptr, int32_t G,
                                                                 int64_t *__restrict__ chunk_ptr,
                                                                 int64_t *__restrict__ split_ptr,
                                                                 int32_t *__restrict__ split_list,
                                                                 int64_t *__restrict__ meta) {
    __shared__ int64_t buf[32];
    int64_t carry_c = 0, carry_s = 0, carry_f = 0;
    for (int64_t base = 0; base < G; base += kPlanThreads) {
        const int64_t g = base + threadIdx.x;
        int64_t nc = 0, ns = 0, f = 0;
        if (g < G) {
            const int64_t n = max(gptr[g + 1] - gptr[g], (int64_t)0);
            nc = n <= kChunkNodes ? 1 : (n + kChunkNodes - 1) / kChunkNodes;
            if (nc > 1) { ns = nc; f = 1; }
        }
        int64_t tc, ts, tf;
        const int64_t ec = block_exclusive_scan(nc, buf, tc);
        const int64_t es = block_exclusive_scan(ns, buf, ts);
        const int64_t ef = block_exclusive_scan(f, buf, tf);
        if (g < G) {
            chunk_ptr[g] = carry_c + ec;
            split_ptr[g] = carry_s + es;
            if (f) split_list[carry_f + ef] = (int32_t)g;
        }
        carry_c += tc;
        carry_s += ts;
        carry_f += tf;
    }
    if (threadIdx.x == 0) {
        chunk_ptr[G] = carry_c;
        split_ptr[G] = carry_s;
        meta[0] = carry_f;
    }
}

// TC = 8 * CT clusters and TD = 32 * DT columns per task; thread (ty, tx) owns clusters ty + 8 i and columns tx + 32 j.
template <int CT, int DT>
__global__ void __launch_bounds__(kTmmThreads, 2) tmm_tile_kernel(
    const float *__restrict__ S, int64_t lds, const float *__restrict__ Y, int64_t ldy, int32_t N, int32_t C, int32_t D,
    const int64_t *__restrict__ gptr, const int32_t *__restrict__ gnodes, int32_t G, float *__restrict__ out, int64_t ldo,
    const int64_t *__restrict__ chunk_ptr, const int64_t *__restrict__ split_ptr, float *__restrict__ partial,
    int64_t max_slots) {
    constexpr int TC = 8 * CT, TD = 32 * DT;
    __shared__ float Ss[kStageRows][TC];
    __shared__ float Ys[kStageRows][TD];
    __shared__ int64_t node[kStageRows];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int n_ct = (C + TC - 1) / TC, n_dt = (D + TD - 1) / TD;
    const int64_t tiles = (int64_t)n_ct * n_dt;
    const int64_t n_tasks = chunk_ptr[G] * tiles;
    for (int64_t t = blockIdx.x; t < n_tasks; t += gridDim.x) {
        const int64_t k = t / tiles;
        const int tile = (int)(t - k * tiles);
        const int c0 = (tile / n_dt) * TC, d0 = (tile % n_dt) * TD;
        int32_t lo = 0, hi = G;                                   // graph g with chunk_ptr[g] <= k < chunk_ptr[g + 1]
        while (hi - lo > 1) {
            const int32_t mid = lo + (hi - lo) / 2;
            if (chunk_ptr[mid] <= k) lo = mid; else hi = mid;
        }
        const int32_t g = lo;
        const int64_t kl = k - chunk_ptr[g];
        const int64_t p_end = gptr[g + 1];
        const int64_t p0 = gptr[g] + kl * kChunkNodes;
        const int64_t p1 = min(p0 + kChunkNodes, p_end);
        float acc[CT][DT];
#pragma unroll
        for (int i = 0; i < CT; ++i)
#pragma unroll
            for (int j = 0; j < DT; ++j) acc[i][j] = 0.0f;
        for (int64_t pb = p0; pb < p1; pb += kStageRows) {
            const int nb = (int)min((int64_t)kStageRows, p1 - pb);
            __syncthreads();                                      // the previous rows have been consumed
            if (threadIdx.x < kStageRows) {
                int64_t n = -1;
                if (threadIdx.x < nb) {
                    const int64_t p = pb + threadIdx.x;
                    n = p < 0 || p >= N ? -1 : (gnodes ? (int64_t)gnodes[p] : p);   // gnodes has N entries
                    if (n < 0 || n >= N) n = -1;                  // an id outside [0, N) poisons its graph with NaN
                }
                node[threadIdx.x] = n;
            }
            __syncthreads();
            for (int i = threadIdx.x; i < kStageRows * TC; i += kTmmThreads) {
                const int r = i / TC, c = i % TC;
                float v = 0.0f;
                if (r < nb) {
                    const int64_t n = node[r];
                    v = n < 0 ? __int_as_float(0x7fc00000) : (c0 + c < C ? S[n * lds + c0 + c] : 0.0f);
                }
                Ss[r][c] = v;
            }
            for (int i = threadIdx.x; i < kStageRows * TD; i += kTmmThreads) {
                const int r = i / TD, d = i % TD;
                float v = 0.0f;
                if (r < nb) {
                    const int64_t n = node[r];
                    v = n < 0 ? __int_as_float(0x7fc00000) : (d0 + d < D ? Y[n * ldy + d0 + d] : 0.0f);
                }
                Ys[r][d] = v;
            }
            __syncthreads();
            for (int r = 0; r < nb; ++r) {
                float y[DT];
#pragma unroll
                for (int j = 0; j < DT; ++j) y[j] = Ys[r][tx + 32 * j];
#pragma unroll
                for (int i = 0; i < CT; ++i) {
                    const float s = Ss[r][ty + 8 * i];
#pragma unroll
                    for (int j = 0; j < DT; ++j) acc[i][j] = fmaf(s, y[j], acc[i][j]);
                }
            }
        }
        const bool direct = chunk_ptr[g + 1] - chunk_ptr[g] == 1;
        const int64_t slot = direct ? 0 : split_ptr[g] + kl;
        if (direct || slot < max_slots) {
#pragma unroll
            for (int i = 0; i < CT; ++i) {
                const int c = c0 + ty + 8 * i;
#pragma unroll
                for (int j = 0; j < DT; ++j) {
                    const int d = d0 + tx + 32 * j;
                    if (c < C && d < D) {
                        float *dst = direct ? out + ((int64_t)g * C + c) * ldo + d : partial + (slot * C + c) * (int64_t)D + d;
                        *dst = acc[i][j];
                    }
                }
            }
        }
        __syncthreads();                                          // node[] and the tiles are rewritten by the next task
    }
}

// out block of every split graph = its chunks' partial blocks added in chunk order
__global__ void tmm_fixup_kernel(const float *__restrict__ partial, int32_t C, int32_t D,
                                 const int64_t *__restrict__ chunk_ptr, const int64_t *__restrict__ split_ptr,
                                 const int32_t *__restrict__ split_list, const int64_t *__restrict__ meta,
                                 int64_t max_slots, float *__restrict__ out, int64_t ldo) {
    const int64_t cd = (int64_t)C * D;
    const int64_t total = meta[0] * cd;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = e / cd, i = e - j * cd;
        const int32_t g = split_list[j];
        const int64_t s0 = split_ptr[g], nch = chunk_ptr[g + 1] - chunk_ptr[g];
        float v;
        if (s0 + nch > max_slots) {
            v = __int_as_float(0x7fc00000);                      // gptr spans more than N positions: no partials were kept
        } else {
            v = partial[s0 * cd + i];
            for (int64_t q = 1; q < nch; ++q) v += partial[(s0 + q) * cd + i];
        }
        const int64_t c = i / D, d = i - c * D;
        out[((int64_t)g * C + c) * ldo + d] = v;
    }
}

template <bool TRANS>
__global__ void rmm_kernel(const float *__restrict__ Y, int64_t ldy, const int32_t *__restrict__ node_graph, int32_t N,
                           const float *__restrict__ B, int64_t ldb, int32_t G, int32_t C, int32_t K, float beta,
                           float *__restrict__ out, int64_t ldo) {
    const int32_t M = TRANS ? C : K;            // output columns
    const int32_t R = TRANS ? K : C;            // reduction length
    const int64_t total = (int64_t)N * M;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = e / M;
        const int32_t m = (int32_t)(e - n * M);
        const int32_t g = node_graph[n];
        float v;
        if (g < 0 || g >= G) {
            v = __int_as_float(0x7fc00000);
        } else {
            const float *y = Y + n * ldy;
            const float *b = TRANS ? B + ((int64_t)g * C + m) * ldb : B + (int64_t)g * C * ldb + m;
            const int64_t step = TRANS ? 1 : ldb;
            v = 0.0f;
            for (int32_t k = 0; k < R; ++k) v = fmaf(y[k], b[k * step], v);
        }
        float *o = out + n * ldo + m;
        *o = beta == 0.0f ? v : fmaf(beta, *o, v);
    }
}

struct TmmWorkspace {
    size_t chunk_ptr, split_ptr, split_list, meta, partial, total;
    int64_t max_slots;
};

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

TmmWorkspace tmm_workspace(int32_t G, int32_t N, int32_t C, int32_t D) {
    TmmWorkspace w;
    // a graph split into q > 1 chunks has more than (q - 1) * kChunkNodes nodes, so q <= 2 N_g / kChunkNodes and all split
    // graphs together own at most 2 N / kChunkNodes slots
    w.max_slots = 2 * (int64_t)N / kChunkNodes;
    w.chunk_ptr = 0;
    w.split_ptr = align256(w.chunk_ptr + (size_t)(G + 1) * 8);
    w.split_list = align256(w.split_ptr + (size_t)(G + 1) * 8);
    w.meta = align256(w.split_list + (size_t)(G + 1) * 4);
    w.partial = align256(w.meta + 8);
    w.total = align256(w.partial + (size_t)w.max_slots * C * D * 4);
    return w;
}

template <int CT, int DT>
int launch_tmm(const float *S, int64_t lds, const float *Y, int64_t ldy, int32_t N, int32_t C, int32_t D,
               const int64_t *gptr, const int32_t *gnodes, int32_t G, float *out, int64_t ldo, char *ws,
               const TmmWorkspace &w, cudaStream_t st) {
    int64_t *chunk_ptr = reinterpret_cast<int64_t *>(ws + w.chunk_ptr);
    int64_t *split_ptr = reinterpret_cast<int64_t *>(ws + w.split_ptr);
    int32_t *split_list = reinterpret_cast<int32_t *>(ws + w.split_list);
    int64_t *meta = reinterpret_cast<int64_t *>(ws + w.meta);
    float *partial = reinterpret_cast<float *>(ws + w.partial);
    tmm_plan_kernel<<<1, kPlanThreads, 0, st>>>(gptr, G, chunk_ptr, split_ptr, split_list, meta);
    TFGK_LAUNCH_CHECK();
    // the task count lives on the device: the grid is the grid-stride cap and CTAs without a task exit at once
    tmm_tile_kernel<CT, DT><<<(unsigned)sm_count() * 8, kTmmThreads, 0, st>>>(
        S, lds, Y, ldy, N, C, D, gptr, gnodes, G, out, ldo, chunk_ptr, split_ptr, partial, w.max_slots);
    TFGK_LAUNCH_CHECK();
    // also without workspace slots: a gptr that spans more than N positions still gets its split graphs' blocks (NaN)
    tmm_fixup_kernel<<<(unsigned)sm_count() * 4, 256, 0, st>>>(partial, C, D, chunk_ptr, split_ptr, split_list, meta,
                                                               w.max_slots, out, ldo);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_graph_tmm_workspace_bytes(int32_t G, int32_t N, int32_t C, int32_t D, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes, "graph_tmm_workspace_bytes: null out_bytes");
    TFGK_CHECK_ARG(G >= 0 && N >= 0 && C >= 1 && D >= 0, "graph_tmm_workspace_bytes: bad G %d, N %d, C %d or D %d", G, N,
                   C, D);
    *out_bytes = tmm_workspace(G, N, C, D).total;
    return TFGK_OK;
}

int tfgk_graph_tmm_f32(const float *S, int64_t lds, const float *Y, int64_t ldy, int32_t N, int32_t C, int32_t D,
                       const int64_t *gptr, const int32_t *gnodes, int32_t G, float *out, int64_t ldo, void *workspace,
                       size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(G >= 0 && N >= 0 && C >= 1 && D >= 0, "graph_tmm: bad G %d, N %d, C %d or D %d", G, N, C, D);
    if (G == 0 || D == 0) return TFGK_OK;
    TFGK_CHECK_ARG(gptr && out, "graph_tmm: null gptr or out");
    TFGK_CHECK_ARG(N == 0 || (S && Y), "graph_tmm: null S or Y");
    TFGK_CHECK_ARG(lds >= C && ldy >= D && ldo >= D, "graph_tmm: leading dimensions (lds %lld, ldy %lld, ldo %lld) below C %d / D %d",
                   (long long)lds, (long long)ldy, (long long)ldo, C, D);
    const TmmWorkspace w = tmm_workspace(G, N, C, D);
    TFGK_CHECK_ARG(workspace && workspace_bytes >= w.total, "graph_tmm: workspace of %zu bytes, %zu needed", workspace_bytes,
                   w.total);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
#define TFGK_TMM(CT, DT) return launch_tmm<CT, DT>(S, lds, Y, ldy, N, C, D, gptr, gnodes, G, out, ldo, ws, w, st)
    const int ct = C <= 8 ? 1 : (C <= 16 ? 2 : 4);
    const int dt = D <= 32 ? 1 : (D <= 64 ? 2 : 4);
    if (ct == 1) { if (dt == 1) TFGK_TMM(1, 1); if (dt == 2) TFGK_TMM(1, 2); TFGK_TMM(1, 4); }
    if (ct == 2) { if (dt == 1) TFGK_TMM(2, 1); if (dt == 2) TFGK_TMM(2, 2); TFGK_TMM(2, 4); }
    if (dt == 1) TFGK_TMM(4, 1);
    if (dt == 2) TFGK_TMM(4, 2);
    TFGK_TMM(4, 4);
#undef TFGK_TMM
}

int tfgk_graph_rmm_f32(const float *Y, int64_t ldy, const int32_t *node_graph, int32_t N, const float *B, int64_t ldb,
                       int32_t G, int32_t C, int32_t K, int trans, float beta, float *out, int64_t ldo, void *stream) {
    TFGK_CHECK_ARG(N >= 0 && G >= 0 && C >= 1 && K >= 0, "graph_rmm: bad N %d, G %d, C %d or K %d", N, G, C, K);
    TFGK_CHECK_ARG(trans == 0 || trans == 1, "graph_rmm: trans must be 0 or 1 (got %d)", trans);
    const int32_t y_cols = trans ? K : C, out_cols = trans ? C : K;
    if (N == 0 || out_cols == 0) return TFGK_OK;
    TFGK_CHECK_ARG(node_graph && out, "graph_rmm: null node_graph or out");
    TFGK_CHECK_ARG(y_cols == 0 || (Y && B), "graph_rmm: null Y or B");
    TFGK_CHECK_ARG(ldy >= y_cols && ldb >= K && ldo >= out_cols,
                   "graph_rmm: leading dimensions (ldy %lld, ldb %lld, ldo %lld) too small", (long long)ldy, (long long)ldb,
                   (long long)ldo);
    cudaStream_t st = as_stream(stream);
    const int64_t total = (int64_t)N * out_cols;
    const unsigned blocks = (unsigned)min(ceil_div64(total, 256), (int64_t)sm_count() * 16);
    if (trans) rmm_kernel<true><<<blocks, 256, 0, st>>>(Y, ldy, node_graph, N, B, ldb, G, C, K, beta, out, ldo);
    else rmm_kernel<false><<<blocks, 256, 0, st>>>(Y, ldy, node_graph, N, B, ldb, G, C, K, beta, out, ldo);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // extern "C"
