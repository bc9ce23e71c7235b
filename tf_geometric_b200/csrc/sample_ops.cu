// Device-side edge sampling (SURVEY.md 8(f)3-4): structural / Bernoulli edge flags, stable stream compaction and a
// CSR fan-out neighbour sampler.  They replace nn/sampling/drop_edge.py:6-52 (tf.nn.dropout + boolean_mask),
// utils/graph_utils.py:775-846 (UniformNeighborSampler) and the per-node Python loop of RandomNeighborSampler.sample
// (utils/graph_utils.py:669-776).  Integer work, HBM-bound; randomness is counter-based (rng.cuh) so every draw is a
// pure function of (seed, element) and the CPU restatement used by the tests reproduces the output bit for bit.
#include "common.cuh"
#include "scan.cuh"
#include "rng.cuh"

namespace tfgk {
namespace {

__global__ void edge_flags_kernel(const int32_t *__restrict__ row, const int32_t *__restrict__ col, int64_t E, int mode,
                                  const int32_t *__restrict__ row_map, const int32_t *__restrict__ col_map,
                                  int bernoulli, float prob, uint64_t seed, uint32_t stream, int32_t *__restrict__ flag) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
        bool keep = true;
        if (mode == TFGK_FLAG_UPPER) keep = row[e] < col[e];
        else if (mode == TFGK_FLAG_MAPPED) keep = row_map[row[e]] >= 0 && col_map[col[e]] >= 0;
        if (keep && bernoulli != TFGK_BERNOULLI_NONE) {
            const float u = random_uniform(seed, stream, (uint64_t)e);
            keep = bernoulli == TFGK_BERNOULLI_DROPOUT ? (u >= prob) : (u <= prob);
        }
        flag[e] = keep ? 1 : 0;
    }
}

__global__ void select_emit_kernel(const int32_t *__restrict__ flag, const int32_t *__restrict__ off, int64_t n,
                                   int32_t *__restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (flag[i]) out[off[i]] = (int32_t)i;
}

enum { kSampleAll = 0, kSampleReplace = 1, kSampleReservoir = 2 };

// how many neighbours row r contributes and by which rule (graph_utils.py:741-756)
__device__ __forceinline__ int sample_rule(int deg, int k, double ratio, int padding, int &num) {
    if (deg == 0) { num = 0; return kSampleAll; }
    if (padding == TFGK_SAMPLE_HEAD) {              // topk_pool.py:59-67: the first node_k entries of the row, in order
        num = ratio < 0.0 ? (k < deg ? k : deg) : (int)ceilf((float)deg * (float)ratio);
        if (num > deg) num = deg;
        if (num < 0) num = 0;
        return kSampleAll;
    }
    if ((k < 0 && ratio < 0.0) || (ratio < 0.0 && !padding && k >= deg)) { num = deg; return kSampleAll; }
    if (ratio < 0.0) { num = k; return (padding && k >= deg) ? kSampleReplace : kSampleReservoir; }
    num = (int)ceil((double)deg * ratio);
    return kSampleReservoir;
}

__global__ void sample_count_kernel(const int64_t *__restrict__ rowptr, int32_t N, int k, double ratio, int padding,
                                    int32_t *__restrict__ cnt) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    int num;
    sample_rule((int)(rowptr[r + 1] - rowptr[r]), k, ratio, padding, num);
    cnt[r] = num;
}

// one thread per row; rows are independent and write disjoint output ranges.  Without replacement: reservoir sampling
// (algorithm R) held directly in the row's output slots.
__global__ void sample_fill_kernel(const int64_t *__restrict__ rowptr, int32_t N, int k, double ratio, int padding,
                                   uint64_t seed, uint32_t stream, const int64_t *__restrict__ out_rowptr,
                                   int32_t *__restrict__ out_row, int32_t *__restrict__ out_pos) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const int64_t start = rowptr[r];
    const int deg = (int)(rowptr[r + 1] - start);
    int num;
    const int rule = sample_rule(deg, k, ratio, padding, num);
    const int64_t o = out_rowptr[r];
    const uint64_t base = (uint64_t)r << 32;
    for (int i = 0; i < num; ++i) out_row[o + i] = (int32_t)r;
    if (rule == kSampleReplace) {
        for (int i = 0; i < num; ++i)
            out_pos[o + i] = (int32_t)(start + random_below(seed, stream, base + (uint64_t)i, (uint32_t)deg));
        return;
    }
    for (int i = 0; i < num; ++i) out_pos[o + i] = (int32_t)(start + i);
    if (rule == kSampleReservoir) {
        for (int i = num; i < deg; ++i) {
            const uint32_t j = random_below(seed, stream, base + (uint64_t)i, (uint32_t)(i + 1));
            if (j < (uint32_t)num) out_pos[o + j] = (int32_t)(start + i);
        }
    }
}

// ---- K13: fan-out sampling from a list of rows ------------------------------------------------------------------
// Row t of the list is global row rows[t]; its draws use the keys of that global row, so every listed row gets exactly
// the positions sample_fill_kernel writes for it.  Algorithm R parallelises: with slot j initialised to start + j, the
// sequential loop leaves slot j at start + max{i >= num : draw_i = j} (later draws overwrite earlier ones, and every
// i >= num exceeds j), so an atomicMax per draw gives the same bits in any order.
constexpr int kRowsPerCta = 256;
constexpr int kThreadRowMax = 128;     // rows up to this degree are sampled by one thread, longer ones by the whole CTA

__global__ void sample_rows_count_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows,
                                         const int32_t *__restrict__ rows, int32_t n_list, int k, double ratio,
                                         int padding, int32_t *__restrict__ cnt, int32_t *__restrict__ n_bad) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_list) return;
    const int32_t r = rows[t];
    int num = 0;
    if (r < 0 || r >= n_rows) atomicAdd(n_bad, 1);
    else sample_rule((int)(rowptr[r + 1] - rowptr[r]), k, ratio, padding, num);
    cnt[t] = num;
}

// The fill of K13.  kBlock (the block sampler) also writes every sampled edge's global column col[pos] and weight
// w_csr[pos], once its position is final; the plain instantiation leaves that to the caller's gathers.
template <bool kBlock>
__device__ __forceinline__ void sample_rows_fill_body(const int64_t *__restrict__ rowptr, int32_t n_rows,
                                                      const int32_t *__restrict__ rows, int32_t n_list, int k,
                                                      double ratio, int padding, uint64_t seed, uint32_t stream,
                                                      const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                                                      int32_t *__restrict__ out_pos, const int32_t *__restrict__ csr_col,
                                                      const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol,
                                                      float *__restrict__ out_w) {
    __shared__ int32_t long_rows[kRowsPerCta];
    __shared__ int n_long;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    const int64_t t = (int64_t)blockIdx.x * kRowsPerCta + threadIdx.x;
    if (t < n_list) {
        const int32_t r = rows[t];
        if (r >= 0 && r < n_rows) {
            const int64_t start = rowptr[r];
            const int deg = (int)(rowptr[r + 1] - start);
            if (deg > kThreadRowMax) {
                long_rows[atomicAdd(&n_long, 1)] = threadIdx.x;      // slot order is irrelevant: rows write disjoint ranges
            } else {
                int num;
                const int rule = sample_rule(deg, k, ratio, padding, num);
                const int64_t o = out_rowptr[t];
                const uint64_t base = (uint64_t)r << 32;
                if (out_row)
                    for (int i = 0; i < num; ++i) out_row[o + i] = (int32_t)t;
                if (rule == kSampleReplace) {
                    for (int i = 0; i < num; ++i)
                        out_pos[o + i] = (int32_t)(start + random_below(seed, stream, base + (uint64_t)i, (uint32_t)deg));
                } else {
                    for (int i = 0; i < num; ++i) out_pos[o + i] = (int32_t)(start + i);
                    if (rule == kSampleReservoir)
                        for (int i = num; i < deg; ++i) {
                            const uint32_t j = random_below(seed, stream, base + (uint64_t)i, (uint32_t)(i + 1));
                            if (j < (uint32_t)num) out_pos[o + j] = (int32_t)(start + i);
                        }
                }
                if constexpr (kBlock)
                    for (int i = 0; i < num; ++i) {
                        const int32_t p = out_pos[o + i];
                        out_gcol[o + i] = csr_col[p];
                        out_w[o + i] = w_csr[p];
                    }
            }
        }
    }
    __syncthreads();
    const int nl = n_long;
    // pass 1: row ids, kept and drawn-with-replacement positions, and the initial reservoir slots
    for (int q = 0; q < nl; ++q) {
        const int64_t tl = (int64_t)blockIdx.x * kRowsPerCta + long_rows[q];
        const int32_t r = rows[tl];
        const int64_t start = rowptr[r];
        const int deg = (int)(rowptr[r + 1] - start);
        int num;
        const int rule = sample_rule(deg, k, ratio, padding, num);
        const int64_t o = out_rowptr[tl];
        const uint64_t base = (uint64_t)r << 32;
        for (int i = threadIdx.x; i < num; i += kRowsPerCta) {
            if (out_row) out_row[o + i] = (int32_t)tl;
            out_pos[o + i] = (int32_t)(start + (rule == kSampleReplace
                                                    ? random_below(seed, stream, base + (uint64_t)i, (uint32_t)deg) : i));
        }
    }
    __syncthreads();                   // every slot holds start + j before any draw competes for it
    // pass 2: the reservoir draws
    for (int q = 0; q < nl; ++q) {
        const int64_t tl = (int64_t)blockIdx.x * kRowsPerCta + long_rows[q];
        const int32_t r = rows[tl];
        const int64_t start = rowptr[r];
        const int deg = (int)(rowptr[r + 1] - start);
        int num;
        if (sample_rule(deg, k, ratio, padding, num) != kSampleReservoir) continue;
        const int64_t o = out_rowptr[tl];
        const uint64_t base = (uint64_t)r << 32;
        for (int i = num + threadIdx.x; i < deg; i += kRowsPerCta) {
            const uint32_t j = random_below(seed, stream, base + (uint64_t)i, (uint32_t)(i + 1));
            if (j < (uint32_t)num) atomicMax(out_pos + o + j, (int32_t)(start + i));
        }
    }
    if constexpr (kBlock) {
        __syncthreads();               // the reservoir's atomics are final
        for (int q = 0; q < nl; ++q) {
            const int64_t tl = (int64_t)blockIdx.x * kRowsPerCta + long_rows[q];
            const int32_t r = rows[tl];
            int num;
            sample_rule((int)(rowptr[r + 1] - rowptr[r]), k, ratio, padding, num);
            const int64_t o = out_rowptr[tl];
            for (int i = threadIdx.x; i < num; i += kRowsPerCta) {
                const int32_t p = out_pos[o + i];
                out_gcol[o + i] = csr_col[p];
                out_w[o + i] = w_csr[p];
            }
        }
    }
}

__global__ void __launch_bounds__(kRowsPerCta)
sample_rows_fill_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                        int32_t n_list, int k, double ratio, int padding, uint64_t seed, uint32_t stream,
                        const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                        int32_t *__restrict__ out_pos) {
    sample_rows_fill_body<false>(rowptr, n_rows, rows, n_list, k, ratio, padding, seed, stream, out_rowptr, out_row,
                                 out_pos, nullptr, nullptr, nullptr, nullptr);
}

// ---- relabelling: an [N] id -> position map that is -1 everywhere outside a call --------------------------------
enum { kBadIds = 0, kDupIds = 1, kNewIds = 2 };

__device__ __forceinline__ void scatter_one(int32_t id, int64_t p, int32_t N, int32_t *__restrict__ map,
                                            int32_t *__restrict__ counters) {
    if (id < 0 || id >= N) atomicAdd(counters + kBadIds, 1);
    else if (atomicCAS(map + id, -1, (int32_t)p) != -1) atomicAdd(counters + kDupIds, 1);
}

__global__ void node_scatter_kernel(const int32_t *__restrict__ nodes, int32_t n, int32_t N, int32_t *__restrict__ map,
                                    int32_t *__restrict__ counters) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
        scatter_one(nodes[p], p, N, map, counters);
}

// reset the map entries of nodes[0, n + *extra)
__global__ void node_reset_kernel(const int32_t *__restrict__ nodes, int64_t n, const int32_t *__restrict__ extra,
                                  int32_t N, int32_t *__restrict__ map) {
    const int64_t total = n + (extra ? *extra : 0);
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t id = nodes[p];
        if (id >= 0 && id < N) map[id] = -1;
    }
}

__device__ __forceinline__ void gather_one(const int32_t *__restrict__ ids, int64_t e, int32_t N,
                                           const int32_t *__restrict__ map, int32_t *__restrict__ out) {
    const int32_t id = ids[e];
    out[e] = (id >= 0 && id < N) ? map[id] : -1;
}

__global__ void reindex_gather_kernel(const int32_t *__restrict__ ids, int64_t n, int32_t N,
                                      const int32_t *__restrict__ map, int32_t *__restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        gather_one(ids, e, N, map, out);
}

// ids not yet in the map: map[id] = INT32_MIN + (first e holding id).  atomicMin keeps the smallest e whatever the
// order, and INT32_MIN + e <= -2 stays below the -1 of an absent id and below every position.
__device__ __forceinline__ void first_one(const int32_t *__restrict__ cols, int64_t e, int32_t N,
                                          int32_t *__restrict__ map, int32_t *__restrict__ counters) {
    const int32_t c = cols[e];
    if (c < 0 || c >= N) atomicAdd(counters + kBadIds, 1);
    else if (map[c] < 0) atomicMin(map + c, INT32_MIN + (int32_t)e);
}

__global__ void frontier_first_kernel(const int32_t *__restrict__ cols, int64_t S, int32_t N, int32_t *__restrict__ map,
                                      int32_t *__restrict__ counters) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < S; e += (int64_t)gridDim.x * blockDim.x)
        first_one(cols, e, N, map, counters);
}

__device__ __forceinline__ int32_t flag_one(const int32_t *__restrict__ cols, int64_t e, int32_t N,
                                            const int32_t *__restrict__ map) {
    const int32_t c = cols[e];
    return (c >= 0 && c < N && map[c] == INT32_MIN + (int32_t)e) ? 1 : 0;
}

__global__ void frontier_flag_kernel(const int32_t *__restrict__ cols, int64_t S, int32_t N,
                                     const int32_t *__restrict__ map, int32_t *__restrict__ flag) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < S; e += (int64_t)gridDim.x * blockDim.x)
        flag[e] = flag_one(cols, e, N, map);
}

__device__ __forceinline__ void emit_one(const int32_t *__restrict__ cols, int64_t e, const int32_t *__restrict__ off,
                                         int32_t n_nodes, int32_t *__restrict__ nodes, int32_t *__restrict__ map) {
    const int32_t pos = n_nodes + off[e];
    nodes[pos] = cols[e];
    map[cols[e]] = pos;
}

__global__ void frontier_emit_kernel(const int32_t *__restrict__ cols, int64_t S, const int32_t *__restrict__ flag,
                                     const int32_t *__restrict__ off, int32_t n_nodes, int32_t *__restrict__ nodes,
                                     int32_t *__restrict__ map) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < S; e += (int64_t)gridDim.x * blockDim.x)
        if (flag[e]) emit_one(cols, e, off, n_nodes, nodes, map);
}

// ---- the block sampler: the same steps with every size kept on the device --------------------------------------
// state (include/tfgk.h): [bad seeds, duplicate seeds, -, list length after hop 0..L, edges of hop 0..L-1].  Grids are
// sized by host-known capacities and threads past the device count exit, so a batch reads nothing back until its end.
constexpr int kStateSizes = 3;

__global__ void block_begin_kernel(const int32_t *__restrict__ seeds, int32_t n, int32_t N, int32_t *__restrict__ nodes,
                                   int32_t *__restrict__ map, int32_t *__restrict__ state) {
    if (blockIdx.x == 0 && threadIdx.x == 0) state[kStateSizes] = n;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
        const int32_t id = seeds[p];
        nodes[p] = id;
        scatter_one(id, p, N, map, state);
    }
}

// listed rows past the device count contribute 0, so the scan over the capacity ends in the hop's edge total
__global__ void block_count_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                                   const int32_t *__restrict__ n_list, int32_t cap, int k, int padding,
                                   int32_t *__restrict__ cnt) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cap) return;
    int num = 0;
    if (t < *n_list) {
        const int32_t r = rows[t];
        if (r >= 0 && r < n_rows) sample_rule((int)(rowptr[r + 1] - rowptr[r]), k, -1.0, padding, num);
    }
    cnt[t] = num;
}

__global__ void __launch_bounds__(kRowsPerCta)
block_fill_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                  const int32_t *__restrict__ n_list, int k, int padding, uint64_t seed, uint32_t stream,
                  const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row, int32_t *__restrict__ out_pos,
                  const int32_t *__restrict__ csr_col, const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol,
                  float *__restrict__ out_w) {
    sample_rows_fill_body<true>(rowptr, n_rows, rows, *n_list, k, -1.0, padding, seed, stream, out_rowptr, out_row,
                                out_pos, csr_col, w_csr, out_gcol, out_w);
}

__global__ void block_first_kernel(const int32_t *__restrict__ cols, const int64_t *__restrict__ S, int32_t N,
                                   int32_t *__restrict__ map, int32_t *__restrict__ counters) {
    const int64_t n = *S;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        first_one(cols, e, N, map, counters);
}

__global__ void block_flag_kernel(const int32_t *__restrict__ cols, const int64_t *__restrict__ S, int64_t cap,
                                  int32_t N, const int32_t *__restrict__ map, int32_t *__restrict__ flag) {
    const int64_t n = *S;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < cap; e += (int64_t)gridDim.x * blockDim.x)
        flag[e] = e < n ? flag_one(cols, e, N, map) : 0;
}

__global__ void block_emit_kernel(const int32_t *__restrict__ cols, const int64_t *__restrict__ S,
                                  const int32_t *__restrict__ flag, const int32_t *__restrict__ off,
                                  const int32_t *__restrict__ n_nodes, int32_t *__restrict__ nodes,
                                  int32_t *__restrict__ map) {
    const int64_t n = *S;
    const int32_t base = *n_nodes;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        if (flag[e]) emit_one(cols, e, off, base, nodes, map);
}

__global__ void block_gather_kernel(const int32_t *__restrict__ ids, const int64_t *__restrict__ S, int32_t N,
                                    const int32_t *__restrict__ map, int32_t *__restrict__ out) {
    const int64_t n = *S;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        gather_one(ids, e, N, map, out);
}

// list length after hop h + 1 and the edges of hop h
__global__ void block_sizes_kernel(const int64_t *__restrict__ S, const int32_t *__restrict__ n_new, int32_t hop,
                                   int32_t n_hops, int32_t *__restrict__ state) {
    state[kStateSizes + hop + 1] = state[kStateSizes + hop] + *n_new;
    state[kStateSizes + n_hops + 1 + hop] = (int32_t)*S;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_edge_flags_i32(const int32_t *row, const int32_t *col, int64_t E, int mode,
                        const int32_t *row_map, const int32_t *col_map,
                        int bernoulli, float prob, uint64_t seed, uint32_t rng_stream, int32_t *flag, void *stream) {
    TFGK_CHECK_ARG(E >= 0, "edge_flags: negative E");
    TFGK_CHECK_ARG(mode == TFGK_FLAG_ALL || mode == TFGK_FLAG_UPPER || mode == TFGK_FLAG_MAPPED, "edge_flags: unknown mode %d", mode);
    TFGK_CHECK_ARG(bernoulli == TFGK_BERNOULLI_NONE || bernoulli == TFGK_BERNOULLI_DROPOUT || bernoulli == TFGK_BERNOULLI_KEEP,
                   "edge_flags: unknown bernoulli rule %d", bernoulli);
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(flag != nullptr, "edge_flags: null output");
    TFGK_CHECK_ARG(mode == TFGK_FLAG_ALL || (row && col), "edge_flags: null edge list");
    TFGK_CHECK_ARG(mode != TFGK_FLAG_MAPPED || (row_map && col_map), "edge_flags: null node map");
    edge_flags_kernel<<<grid_for(E), 256, 0, as_stream(stream)>>>(row, col, E, mode, row_map, col_map, bernoulli, prob, seed,
                                                                  rng_stream, flag);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_select_workspace_bytes(int64_t n, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n >= 0 && n < (1ll << 31) - 1, "select_workspace_bytes: bad argument");
    *out_bytes = align_up((size_t)(n + 1) * 4) + scan_scratch_bytes(n + 1) + 256;
    return TFGK_OK;
}

int tfgk_select_flagged_i32(const int32_t *flag, int64_t n, int32_t *out_index, int64_t *n_out_host,
                            void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n >= 0 && n < (1ll << 31) - 1, "select_flagged: bad size");
    TFGK_CHECK_ARG(n_out_host != nullptr, "select_flagged: null count");
    *n_out_host = 0;
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(flag && out_index, "select_flagged: null pointer");
    size_t need = 0;
    tfgk_select_workspace_bytes(n, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "select_flagged: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int32_t *off = reinterpret_cast<int32_t *>(ws);
    int32_t *sums = reinterpret_cast<int32_t *>(ws + align_up((size_t)(n + 1) * 4));
    // offsets count the non-zero flags, not their values: a flag of 2 or -1 selects its position once, like a 1
    const int rc = exclusive_scan<int32_t, int32_t, true>(flag, n, n + 1, off, sums, st);
    if (rc != TFGK_OK) return rc;
    int32_t total = 0;
    TFGK_CUDA(cudaMemcpyAsync(&total, off + n, 4, cudaMemcpyDeviceToHost, st));
    select_emit_kernel<<<grid_for(n), 256, 0, st>>>(flag, off, n, out_index);
    TFGK_LAUNCH_CHECK();
    TFGK_CUDA(cudaStreamSynchronize(st));
    *n_out_host = total;
    return TFGK_OK;
}

int tfgk_neighbor_sample_workspace_bytes(int32_t n_rows, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n_rows >= 0, "neighbor_sample_workspace_bytes: bad argument");
    *out_bytes = align_up(((size_t)n_rows + 1) * 4) + scan_scratch_bytes((int64_t)n_rows + 1) + 256;
    return TFGK_OK;
}

static int check_sample_args(const char *fn, int32_t n_rows, int32_t k, double ratio) {
    TFGK_CHECK_ARG(n_rows >= 0, "%s: negative row count", fn);
    TFGK_CHECK_ARG(!(k >= 0 && ratio >= 0.0), "%s: k and ratio cannot be provided simultaneously", fn);
    TFGK_CHECK_ARG(ratio <= 1.0, "%s: ratio %g > 1 cannot be sampled without replacement", fn, ratio);
    return TFGK_OK;
}

static int check_sample_mode(const char *fn, int32_t k, double ratio, int padding) {
    TFGK_CHECK_ARG(padding == 0 || padding == 1 || padding == TFGK_SAMPLE_HEAD, "%s: unknown padding mode %d", fn, padding);
    TFGK_CHECK_ARG(padding != TFGK_SAMPLE_HEAD || k >= 0 || ratio >= 0.0, "%s: the head rule needs k or ratio", fn);
    return TFGK_OK;
}

int tfgk_neighbor_sample_count(const int64_t *rowptr, int32_t n_rows, int32_t k, double ratio, int padding,
                               int64_t *out_rowptr, int64_t *total_host, void *workspace, size_t workspace_bytes,
                               void *stream) {
    int rc = check_sample_args("neighbor_sample_count", n_rows, k, ratio);
    if (rc != TFGK_OK) return rc;
    if ((rc = check_sample_mode("neighbor_sample_count", k, ratio, padding)) != TFGK_OK) return rc;
    TFGK_CHECK_ARG(total_host != nullptr && out_rowptr != nullptr, "neighbor_sample_count: null pointer");
    *total_host = 0;
    cudaStream_t st = as_stream(stream);
    if (n_rows == 0) {
        TFGK_CUDA(cudaMemsetAsync(out_rowptr, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr != nullptr, "neighbor_sample_count: null rowptr");
    size_t need = 0;
    tfgk_neighbor_sample_workspace_bytes(n_rows, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "neighbor_sample_count: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    char *ws = static_cast<char *>(workspace);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + align_up(((size_t)n_rows + 1) * 4));
    sample_count_kernel<<<(unsigned)ceil_div64(n_rows, 256), 256, 0, st>>>(rowptr, n_rows, k, ratio, padding, cnt);
    TFGK_LAUNCH_CHECK();
    rc = exclusive_scan<int32_t, int64_t>(cnt, n_rows, (int64_t)n_rows + 1, out_rowptr, sums, st);
    if (rc != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(total_host, out_rowptr + n_rows, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    TFGK_CHECK_ARG(*total_host < (1ll << 31) - 1, "neighbor_sample_count: %lld sampled edges exceed int32 positions", (long long)*total_host);
    return TFGK_OK;
}

int tfgk_neighbor_sample_fill(const int64_t *rowptr, int32_t n_rows, int32_t k, double ratio, int padding,
                              uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                              int32_t *out_row, int32_t *out_pos, void *stream) {
    int rc = check_sample_args("neighbor_sample_fill", n_rows, k, ratio);
    if (rc != TFGK_OK) return rc;
    if ((rc = check_sample_mode("neighbor_sample_fill", k, ratio, padding)) != TFGK_OK) return rc;
    if (n_rows == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && out_rowptr, "neighbor_sample_fill: null pointer");
    sample_fill_kernel<<<(unsigned)ceil_div64(n_rows, 128), 128, 0, as_stream(stream)>>>(rowptr, n_rows, k, ratio, padding, seed,
                                                                                       rng_stream, out_rowptr, out_row, out_pos);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_neighbor_sample_rows_count(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list, int32_t k,
                                    double ratio, int padding, int64_t *out_rowptr, int64_t *total_host, void *workspace,
                                    size_t workspace_bytes, void *stream) {
    int rc = check_sample_args("neighbor_sample_rows_count", n_list, k, ratio);
    if (rc != TFGK_OK) return rc;
    if ((rc = check_sample_mode("neighbor_sample_rows_count", k, ratio, padding)) != TFGK_OK) return rc;
    TFGK_CHECK_ARG(n_rows >= 0, "neighbor_sample_rows_count: negative CSR row count");
    TFGK_CHECK_ARG(total_host != nullptr && out_rowptr != nullptr, "neighbor_sample_rows_count: null pointer");
    *total_host = 0;
    cudaStream_t st = as_stream(stream);
    if (n_list == 0) {
        TFGK_CUDA(cudaMemsetAsync(out_rowptr, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr != nullptr && rows != nullptr, "neighbor_sample_rows_count: null rowptr or row list");
    size_t need = 0;
    tfgk_neighbor_sample_workspace_bytes(n_list, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "neighbor_sample_rows_count: workspace too small (%zu < %zu bytes)",
                         workspace_bytes, need);
    char *ws = static_cast<char *>(workspace);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + align_up(((size_t)n_list + 1) * 4));
    int32_t *n_bad = reinterpret_cast<int32_t *>(ws + need - 256);      // the workspace's last 256 bytes
    TFGK_CUDA(cudaMemsetAsync(n_bad, 0, 4, st));
    sample_rows_count_kernel<<<(unsigned)ceil_div64(n_list, 256), 256, 0, st>>>(rowptr, n_rows, rows, n_list, k, ratio,
                                                                                padding, cnt, n_bad);
    TFGK_LAUNCH_CHECK();
    rc = exclusive_scan<int32_t, int64_t>(cnt, n_list, (int64_t)n_list + 1, out_rowptr, sums, st);
    if (rc != TFGK_OK) return rc;
    int32_t bad = 0;
    TFGK_CUDA(cudaMemcpyAsync(total_host, out_rowptr + n_list, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(&bad, n_bad, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (bad) {
        *total_host = 0;
        return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "neighbor_sample_rows_count: %d listed rows outside [0, %d)", bad,
                         n_rows);
    }
    TFGK_CHECK_ARG(*total_host < (1ll << 31) - 1, "neighbor_sample_rows_count: %lld sampled edges exceed int32 positions",
                   (long long)*total_host);
    return TFGK_OK;
}

int tfgk_neighbor_sample_rows_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list, int32_t k,
                                   double ratio, int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                   int32_t *out_row, int32_t *out_pos, void *stream) {
    int rc = check_sample_args("neighbor_sample_rows_fill", n_list, k, ratio);
    if (rc != TFGK_OK) return rc;
    if ((rc = check_sample_mode("neighbor_sample_rows_fill", k, ratio, padding)) != TFGK_OK) return rc;
    if (n_list == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && rows && out_rowptr && out_pos, "neighbor_sample_rows_fill: null pointer");
    sample_rows_fill_kernel<<<(unsigned)ceil_div64(n_list, kRowsPerCta), kRowsPerCta, 0, as_stream(stream)>>>(
        rowptr, n_rows, rows, n_list, k, ratio, padding, seed, rng_stream, out_rowptr, out_row, out_pos);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_relabel_workspace_bytes(int64_t n_ids, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n_ids >= 0 && n_ids < (1ll << 31) - 1, "relabel_workspace_bytes: bad argument");
    *out_bytes = 2 * align_up((size_t)(n_ids + 1) * 4) + scan_scratch_bytes(n_ids + 1) + 256;
    return TFGK_OK;
}

// the three counters live in the workspace's last 256 bytes
static int read_counters(const int32_t *counters, int32_t *host, cudaStream_t st) {
    TFGK_CUDA(cudaMemcpyAsync(host, counters, 3 * 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

int tfgk_reindex_i32(const int32_t *nodes, int32_t n_nodes, const int32_t *ids, int64_t n_ids, int32_t N, int32_t *map,
                     int32_t *out, int32_t *n_dup_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n_nodes >= 0 && n_ids >= 0 && N >= 0 && n_dup_host != nullptr, "reindex: bad argument");
    *n_dup_host = 0;
    if (n_nodes == 0 && n_ids == 0) return TFGK_OK;
    TFGK_CHECK_ARG(map != nullptr && (n_nodes == 0 || nodes) && (n_ids == 0 || (ids && out)), "reindex: null pointer");
    size_t need = 0;
    tfgk_relabel_workspace_bytes(0, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "reindex: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    int32_t *counters = reinterpret_cast<int32_t *>(static_cast<char *>(workspace) + need - 256);
    TFGK_CUDA(cudaMemsetAsync(counters, 0, 3 * 4, st));
    if (n_nodes) {
        node_scatter_kernel<<<grid_for(n_nodes), 256, 0, st>>>(nodes, n_nodes, N, map, counters);
        TFGK_LAUNCH_CHECK();
    }
    if (n_ids) {
        reindex_gather_kernel<<<grid_for(n_ids), 256, 0, st>>>(ids, n_ids, N, map, out);
        TFGK_LAUNCH_CHECK();
    }
    if (n_nodes) {
        node_reset_kernel<<<grid_for(n_nodes), 256, 0, st>>>(nodes, n_nodes, nullptr, N, map);
        TFGK_LAUNCH_CHECK();
    }
    int32_t c[3];
    int rc = read_counters(counters, c, st);
    if (rc != TFGK_OK) return rc;
    if (c[kBadIds]) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "reindex: %d node ids outside [0, %d)", c[kBadIds], N);
    *n_dup_host = c[kDupIds];
    return TFGK_OK;
}

int tfgk_frontier_i32(const int32_t *cols, int64_t S, int32_t N, int32_t *nodes, int32_t n_nodes, int32_t *map,
                      int32_t *local_col, int32_t *n_new_host, int32_t *n_dup_host, void *workspace, size_t workspace_bytes,
                      void *stream) {
    TFGK_CHECK_ARG(S >= 0 && S < (1ll << 31) - 1 && n_nodes >= 0 && N >= 0 && (int64_t)n_nodes + S < (1ll << 31) - 1,
                   "frontier: bad size");
    TFGK_CHECK_ARG(n_new_host != nullptr && n_dup_host != nullptr, "frontier: null count");
    *n_new_host = 0;
    *n_dup_host = 0;
    if (n_nodes == 0 && S == 0) return TFGK_OK;
    TFGK_CHECK_ARG(map && nodes && (S == 0 || (cols && local_col)), "frontier: null pointer");
    size_t need = 0;
    tfgk_relabel_workspace_bytes(S, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "frontier: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int32_t *flag = reinterpret_cast<int32_t *>(ws);
    int32_t *off = reinterpret_cast<int32_t *>(ws + align_up((size_t)(S + 1) * 4));
    int32_t *sums = reinterpret_cast<int32_t *>(ws + 2 * align_up((size_t)(S + 1) * 4));
    int32_t *counters = reinterpret_cast<int32_t *>(ws + need - 256);
    TFGK_CUDA(cudaMemsetAsync(counters, 0, 3 * 4, st));
    if (n_nodes) {
        node_scatter_kernel<<<grid_for(n_nodes), 256, 0, st>>>(nodes, n_nodes, N, map, counters);
        TFGK_LAUNCH_CHECK();
    }
    if (S) {
        frontier_first_kernel<<<grid_for(S), 256, 0, st>>>(cols, S, N, map, counters);
        TFGK_LAUNCH_CHECK();
        frontier_flag_kernel<<<grid_for(S), 256, 0, st>>>(cols, S, N, map, flag);
        TFGK_LAUNCH_CHECK();
        int rc = exclusive_scan<int32_t, int32_t>(flag, S, S + 1, off, sums, st);
        if (rc != TFGK_OK) return rc;
        frontier_emit_kernel<<<grid_for(S), 256, 0, st>>>(cols, S, flag, off, n_nodes, nodes, map);
        TFGK_LAUNCH_CHECK();
        reindex_gather_kernel<<<grid_for(S), 256, 0, st>>>(cols, S, N, map, local_col);
        TFGK_LAUNCH_CHECK();
        TFGK_CUDA(cudaMemcpyAsync(counters + kNewIds, off + S, 4, cudaMemcpyDeviceToDevice, st));
    }
    node_reset_kernel<<<grid_for((int64_t)n_nodes + S), 256, 0, st>>>(nodes, n_nodes, S ? off + S : nullptr, N, map);
    TFGK_LAUNCH_CHECK();
    int32_t c[3];
    int rc = read_counters(counters, c, st);
    if (rc != TFGK_OK) return rc;
    if (c[kBadIds]) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "frontier: %d node ids outside [0, %d)", c[kBadIds], N);
    *n_dup_host = c[kDupIds];
    *n_new_host = c[kNewIds];
    return TFGK_OK;
}

// ---- block sampler (include/tfgk.h) -----------------------------------------------------------------------------
namespace {
struct BlockWorkspace {
    size_t off_sums, off_pos, off_flag, off_off, total;
    BlockWorkspace(int32_t cap_list, int64_t cap_edges) {
        size_t sums = scan_scratch_bytes((int64_t)cap_list + 1);
        if (scan_scratch_bytes(cap_edges + 1) > sums) sums = scan_scratch_bytes(cap_edges + 1);
        off_sums = align_up(((size_t)cap_list + 1) * 4);                   // per-row counts first
        off_pos = off_sums + sums;
        off_flag = off_pos + align_up((size_t)(cap_edges > 0 ? cap_edges : 1) * 4);
        off_off = off_flag + align_up((size_t)(cap_edges + 1) * 4);
        total = off_off + align_up((size_t)(cap_edges + 1) * 4);
    }
};
}  // namespace

static int block_workspace_check(const char *fn, int32_t cap_list, int64_t cap_edges, void *workspace,
                                 size_t workspace_bytes) {
    const size_t need = BlockWorkspace(cap_list, cap_edges).total;
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", fn, workspace_bytes, need);
    return TFGK_OK;
}

int tfgk_block_sample_workspace_bytes(int32_t cap_list, int64_t cap_edges, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && cap_list >= 0 && cap_edges >= 0 && cap_edges < (1ll << 31) - 1,
                   "block_sample_workspace_bytes: bad argument");
    *out_bytes = BlockWorkspace(cap_list, cap_edges).total;
    return TFGK_OK;
}

int tfgk_block_sample_begin(const int32_t *seeds, int32_t n_seeds, int32_t N, int32_t *nodes, int32_t *map,
                            int32_t *state, int32_t n_hops, void *stream) {
    TFGK_CHECK_ARG(n_seeds >= 0 && N >= 0 && n_hops >= 0, "block_sample_begin: bad size");
    TFGK_CHECK_ARG(state != nullptr && (n_seeds == 0 || (seeds && nodes && map)), "block_sample_begin: null pointer");
    cudaStream_t st = as_stream(stream);
    TFGK_CUDA(cudaMemsetAsync(state, 0, (size_t)(4 + 2 * n_hops) * 4, st));
    block_begin_kernel<<<grid_for(n_seeds), 256, 0, st>>>(seeds, n_seeds, N, nodes, map, state);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_block_sample_count(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                            int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding, int64_t *out_rowptr,
                            void *workspace, size_t workspace_bytes, void *stream) {
    int rc = check_sample_mode("block_sample_count", k, -1.0, padding);
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(n_rows >= 0 && hop >= 0 && hop < n_hops && cap_list >= 0, "block_sample_count: bad size");
    TFGK_CHECK_ARG(state != nullptr && out_rowptr != nullptr, "block_sample_count: null pointer");
    cudaStream_t st = as_stream(stream);
    if (cap_list == 0) {
        TFGK_CUDA(cudaMemsetAsync(out_rowptr, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr != nullptr && nodes != nullptr, "block_sample_count: null rowptr or node list");
    if ((rc = block_workspace_check("block_sample_count", cap_list, 0, workspace, workspace_bytes)) != TFGK_OK) return rc;
    char *ws = static_cast<char *>(workspace);
    const BlockWorkspace L(cap_list, 0);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws);
    block_count_kernel<<<(unsigned)ceil_div64(cap_list, 256), 256, 0, st>>>(rowptr, n_rows, nodes,
                                                                            state + kStateSizes + hop, cap_list, k,
                                                                            padding, cnt);
    TFGK_LAUNCH_CHECK();
    return exclusive_scan<int32_t, int64_t>(cnt, cap_list, (int64_t)cap_list + 1, out_rowptr,
                                            reinterpret_cast<int64_t *>(ws + L.off_sums), st);
}

int tfgk_block_sample_read_total(const int32_t *state, int32_t hop, const int64_t *out_rowptr, int32_t cap_list,
                                 int32_t *n_list_host, int64_t *total_host, void *stream) {
    TFGK_CHECK_ARG(state && out_rowptr && n_list_host && total_host && hop >= 0 && cap_list >= 0,
                   "block_sample_read_total: bad argument");
    cudaStream_t st = as_stream(stream);
    TFGK_CUDA(cudaMemcpyAsync(n_list_host, state + kStateSizes + hop, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(total_host, out_rowptr + cap_list, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    TFGK_CHECK_ARG(*total_host < (1ll << 31) - 1, "block_sample_read_total: %lld sampled edges exceed int32 positions",
                   (long long)*total_host);
    return TFGK_OK;
}

int tfgk_block_sample_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr, int32_t N,
                           int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                           int64_t cap_edges, int32_t k, int padding, uint64_t seed, uint32_t rng_stream,
                           const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local, int32_t *out_gcol,
                           float *out_w, void *workspace, size_t workspace_bytes, void *stream) {
    int rc = check_sample_mode("block_sample_fill", k, -1.0, padding);
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(n_rows >= 0 && N >= 0 && hop >= 0 && hop < n_hops && cap_list >= 0 && cap_edges >= 0 &&
                   cap_edges < (1ll << 31) - 1, "block_sample_fill: bad size");
    TFGK_CHECK_ARG(state && out_rowptr, "block_sample_fill: null pointer");
    if ((rc = block_workspace_check("block_sample_fill", cap_list, cap_edges, workspace, workspace_bytes)) != TFGK_OK)
        return rc;
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    const BlockWorkspace L(cap_list, cap_edges);
    int32_t *pos = reinterpret_cast<int32_t *>(ws + L.off_pos);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int32_t *off = reinterpret_cast<int32_t *>(ws + L.off_off);
    const int32_t *n_list = state + kStateSizes + hop;
    const int64_t *S = out_rowptr + cap_list;               // listed rows past the count add no edges
    if (cap_list > 0 && cap_edges > 0) {
        TFGK_CHECK_ARG(rowptr && col && w_csr && nodes && map && out_row && out_local && out_gcol && out_w,
                       "block_sample_fill: null pointer");
        block_fill_kernel<<<(unsigned)ceil_div64(cap_list, kRowsPerCta), kRowsPerCta, 0, st>>>(
            rowptr, n_rows, nodes, n_list, k, padding, seed, rng_stream, out_rowptr, out_row, pos, col, w_csr, out_gcol,
            out_w);
        TFGK_LAUNCH_CHECK();
        block_first_kernel<<<grid_for(cap_edges), 256, 0, st>>>(out_gcol, S, N, map, state);
        TFGK_LAUNCH_CHECK();
        block_flag_kernel<<<grid_for(cap_edges), 256, 0, st>>>(out_gcol, S, cap_edges, N, map, flag);
        TFGK_LAUNCH_CHECK();
        rc = exclusive_scan<int32_t, int32_t>(flag, cap_edges, cap_edges + 1, off, reinterpret_cast<int32_t *>(ws + L.off_sums),
                                              st);
        if (rc != TFGK_OK) return rc;
        block_emit_kernel<<<grid_for(cap_edges), 256, 0, st>>>(out_gcol, S, flag, off, n_list, nodes, map);
        TFGK_LAUNCH_CHECK();
        block_gather_kernel<<<grid_for(cap_edges), 256, 0, st>>>(out_gcol, S, N, map, out_local);
        TFGK_LAUNCH_CHECK();
    } else {
        TFGK_CUDA(cudaMemsetAsync(off, 0, 4, st));          // no edges, no new nodes
    }
    block_sizes_kernel<<<1, 1, 0, st>>>(S, off + cap_edges, hop, n_hops, state);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_block_sample_end(const int32_t *nodes, int32_t cap_nodes, int32_t N, int32_t *map, const int32_t *state,
                          int32_t n_hops, int32_t *state_host, void *stream) {
    TFGK_CHECK_ARG(cap_nodes >= 0 && N >= 0 && n_hops >= 0, "block_sample_end: bad size");
    TFGK_CHECK_ARG(state && state_host && (cap_nodes == 0 || (nodes && map)), "block_sample_end: null pointer");
    cudaStream_t st = as_stream(stream);
    if (cap_nodes > 0) {
        node_reset_kernel<<<grid_for(cap_nodes), 256, 0, st>>>(nodes, 0, state + kStateSizes + n_hops, N, map);
        TFGK_LAUNCH_CHECK();
    }
    TFGK_CUDA(cudaMemcpyAsync(state_host, state, (size_t)(4 + 2 * n_hops) * 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

}  // extern "C"
