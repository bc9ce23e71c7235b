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

// the reservoir's order-free maximum on a CSR position (positions are >= 0, so the unsigned 64-bit order is theirs)
__device__ __forceinline__ void atomic_max_pos(int32_t *p, int32_t v) { atomicMax(p, v); }
__device__ __forceinline__ void atomic_max_pos(int64_t *p, int64_t v) {
    atomicMax(reinterpret_cast<unsigned long long *>(p), (unsigned long long)v);
}

// Excluded CSR entries (the link sampler's target edges): list row t < n_excl skips the x_t ascending CSR positions
// excl_pos[excl_off[t], excl_off[t + 1]).  Its rule and draws run over the deg - x_t kept entries, so a draw's position is
// virtual (the v-th kept entry); excl_real maps it to the real one.  The j-th excluded entry has e_j - j kept entries
// before it, a nondecreasing count, so the v-th kept entry lies past exactly the j with e_j - j <= v.
__device__ __forceinline__ int excl_count(const int64_t *__restrict__ excl_off, int32_t n_excl, int64_t t) {
    return t < n_excl ? (int)(excl_off[t + 1] - excl_off[t]) : 0;
}

template <typename TPos>
__device__ __forceinline__ TPos excl_real(const TPos *__restrict__ ex, int x, int64_t start, TPos p) {
    const int64_t v = (int64_t)p - start;
    int lo = 0, hi = x;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((int64_t)ex[mid] - start - mid <= v) lo = mid + 1;
        else hi = mid;
    }
    return (TPos)(p + lo);
}

// The fill of K13.  kBlock (the block sampler) also writes every sampled edge's global column col[pos] and weight
// w_csr[pos] (1.0f when w_csr is null), once its position is final; the plain instantiation leaves that to the caller's
// gathers.  TPos is the type of the CSR positions: int32_t for a CSR on the device, int64_t for one in host memory, which
// may hold 2^31 edges or more.  kExcl (with kBlock) skips the excluded entries above: positions stay virtual until the
// final pass maps them, so the reservoir's atomicMax compares virtual positions, in the same order as the real ones.
template <bool kBlock, typename TPos, bool kExcl = false>
__device__ __forceinline__ void sample_rows_fill_body(const int64_t *__restrict__ rowptr, int32_t n_rows,
                                                      const int32_t *__restrict__ rows, int32_t n_list, int k,
                                                      double ratio, int padding, uint64_t seed, uint32_t stream,
                                                      const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                                                      TPos *__restrict__ out_pos, const int32_t *__restrict__ csr_col,
                                                      const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol,
                                                      float *__restrict__ out_w,
                                                      const int64_t *__restrict__ excl_off = nullptr,
                                                      const TPos *__restrict__ excl_pos = nullptr, int32_t n_excl = 0) {
    __shared__ int32_t long_rows[kRowsPerCta];
    __shared__ int n_long;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    const int64_t t = (int64_t)blockIdx.x * kRowsPerCta + threadIdx.x;
    if (t < n_list) {
        const int32_t r = rows[t];
        if (r >= 0 && r < n_rows) {
            const int64_t start = rowptr[r];
            const int x = kExcl ? excl_count(excl_off, n_excl, t) : 0;
            const int deg = (int)(rowptr[r + 1] - start) - x;
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
                        out_pos[o + i] = (TPos)(start + random_below(seed, stream, base + (uint64_t)i, (uint32_t)deg));
                } else {
                    for (int i = 0; i < num; ++i) out_pos[o + i] = (TPos)(start + i);
                    if (rule == kSampleReservoir)
                        for (int i = num; i < deg; ++i) {
                            const uint32_t j = random_below(seed, stream, base + (uint64_t)i, (uint32_t)(i + 1));
                            if (j < (uint32_t)num) out_pos[o + j] = (TPos)(start + i);
                        }
                }
                if constexpr (kBlock)
                    for (int i = 0; i < num; ++i) {
                        TPos p = out_pos[o + i];
                        if constexpr (kExcl)
                            if (x) p = excl_real(excl_pos + excl_off[t], x, start, p);
                        out_gcol[o + i] = csr_col[p];
                        out_w[o + i] = w_csr ? w_csr[p] : 1.0f;
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
        const int deg = (int)(rowptr[r + 1] - start) - (kExcl ? excl_count(excl_off, n_excl, tl) : 0);
        int num;
        const int rule = sample_rule(deg, k, ratio, padding, num);
        const int64_t o = out_rowptr[tl];
        const uint64_t base = (uint64_t)r << 32;
        for (int i = threadIdx.x; i < num; i += kRowsPerCta) {
            if (out_row) out_row[o + i] = (int32_t)tl;
            out_pos[o + i] = (TPos)(start + (rule == kSampleReplace
                                                    ? random_below(seed, stream, base + (uint64_t)i, (uint32_t)deg) : i));
        }
    }
    __syncthreads();                   // every slot holds start + j before any draw competes for it
    // pass 2: the reservoir draws
    for (int q = 0; q < nl; ++q) {
        const int64_t tl = (int64_t)blockIdx.x * kRowsPerCta + long_rows[q];
        const int32_t r = rows[tl];
        const int64_t start = rowptr[r];
        const int deg = (int)(rowptr[r + 1] - start) - (kExcl ? excl_count(excl_off, n_excl, tl) : 0);
        int num;
        if (sample_rule(deg, k, ratio, padding, num) != kSampleReservoir) continue;
        const int64_t o = out_rowptr[tl];
        const uint64_t base = (uint64_t)r << 32;
        for (int i = num + threadIdx.x; i < deg; i += kRowsPerCta) {
            const uint32_t j = random_below(seed, stream, base + (uint64_t)i, (uint32_t)(i + 1));
            if (j < (uint32_t)num) atomic_max_pos(out_pos + o + j, (TPos)(start + i));
        }
    }
    if constexpr (kBlock) {
        __syncthreads();               // the reservoir's atomics are final
        for (int q = 0; q < nl; ++q) {
            const int64_t tl = (int64_t)blockIdx.x * kRowsPerCta + long_rows[q];
            const int32_t r = rows[tl];
            const int x = kExcl ? excl_count(excl_off, n_excl, tl) : 0;
            int num;
            sample_rule((int)(rowptr[r + 1] - rowptr[r]) - x, k, ratio, padding, num);
            const int64_t o = out_rowptr[tl];
            for (int i = threadIdx.x; i < num; i += kRowsPerCta) {
                TPos p = out_pos[o + i];
                if constexpr (kExcl)
                    if (x) p = excl_real(excl_pos + excl_off[tl], x, rowptr[r], p);
                out_gcol[o + i] = csr_col[p];
                out_w[o + i] = w_csr ? w_csr[p] : 1.0f;
            }
        }
    }
}

__global__ void __launch_bounds__(kRowsPerCta)
sample_rows_fill_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                        int32_t n_list, int k, double ratio, int padding, uint64_t seed, uint32_t stream,
                        const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                        int32_t *__restrict__ out_pos) {
    sample_rows_fill_body<false, int32_t>(rowptr, n_rows, rows, n_list, k, ratio, padding, seed, stream, out_rowptr, out_row,
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

// listed rows past the device count contribute 0, so the scan over the capacity ends in the hop's edge total; kExcl
// counts over the kept entries of rows with exclusions (sample_rows_fill_body)
template <bool kExcl>
__device__ __forceinline__ void block_count_body(const int64_t *__restrict__ rowptr, int32_t n_rows,
                                                 const int32_t *__restrict__ rows, const int32_t *__restrict__ n_list,
                                                 int32_t cap, int k, int padding, int32_t *__restrict__ cnt,
                                                 const int64_t *__restrict__ excl_off, int32_t n_excl) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cap) return;
    int num = 0;
    if (t < *n_list) {
        const int32_t r = rows[t];
        if (r >= 0 && r < n_rows)
            sample_rule((int)(rowptr[r + 1] - rowptr[r]) - (kExcl ? excl_count(excl_off, n_excl, t) : 0), k, -1.0,
                        padding, num);
    }
    cnt[t] = num;
}

__global__ void block_count_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                                   const int32_t *__restrict__ n_list, int32_t cap, int k, int padding,
                                   int32_t *__restrict__ cnt) {
    block_count_body<false>(rowptr, n_rows, rows, n_list, cap, k, padding, cnt, nullptr, 0);
}

__global__ void block_count_excl_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows,
                                        const int32_t *__restrict__ rows, const int32_t *__restrict__ n_list, int32_t cap,
                                        int k, int padding, int32_t *__restrict__ cnt,
                                        const int64_t *__restrict__ excl_off, int32_t n_excl) {
    block_count_body<true>(rowptr, n_rows, rows, n_list, cap, k, padding, cnt, excl_off, n_excl);
}

__global__ void __launch_bounds__(kRowsPerCta)
block_fill_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                  const int32_t *__restrict__ n_list, int k, int padding, uint64_t seed, uint32_t stream,
                  const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row, int32_t *__restrict__ out_pos,
                  const int32_t *__restrict__ csr_col, const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol,
                  float *__restrict__ out_w) {
    sample_rows_fill_body<true, int32_t>(rowptr, n_rows, rows, *n_list, k, -1.0, padding, seed, stream, out_rowptr,
                                         out_row, out_pos, csr_col, w_csr, out_gcol, out_w);
}

// the same fill over a CSR in host memory: csr_col and w_csr (or null: every weight 1.0f) are read over the host link,
// one 4-byte column (and weight) per sampled edge, at int64 positions.  The minimum of 4 CTAs per SM leaves ptxas room
// for the 64-bit positions (left to itself it chose 40 registers and spilled).
__global__ void __launch_bounds__(kRowsPerCta, 4)
block_fill_mapped_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                         const int32_t *__restrict__ n_list, int k, int padding, uint64_t seed, uint32_t stream,
                         const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                         int64_t *__restrict__ out_pos, const int32_t *__restrict__ csr_col,
                         const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol, float *__restrict__ out_w) {
    sample_rows_fill_body<true, int64_t>(rowptr, n_rows, rows, *n_list, k, -1.0, padding, seed, stream, out_rowptr,
                                         out_row, out_pos, csr_col, w_csr, out_gcol, out_w);
}

// the minimum of 4 CTAs per SM, as for block_fill_mapped_kernel: left to itself ptxas chose 40 registers and spilled
__global__ void __launch_bounds__(kRowsPerCta, 4)
block_fill_excl_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                       const int32_t *__restrict__ n_list, int k, int padding, uint64_t seed, uint32_t stream,
                       const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row, int32_t *__restrict__ out_pos,
                       const int32_t *__restrict__ csr_col, const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol,
                       float *__restrict__ out_w, const int64_t *__restrict__ excl_off,
                       const int32_t *__restrict__ excl_pos, int32_t n_excl) {
    sample_rows_fill_body<true, int32_t, true>(rowptr, n_rows, rows, *n_list, k, -1.0, padding, seed, stream, out_rowptr,
                                               out_row, out_pos, csr_col, w_csr, out_gcol, out_w, excl_off, excl_pos,
                                               n_excl);
}

__global__ void __launch_bounds__(kRowsPerCta, 4)
block_fill_mapped_excl_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                              const int32_t *__restrict__ n_list, int k, int padding, uint64_t seed, uint32_t stream,
                              const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                              int64_t *__restrict__ out_pos, const int32_t *__restrict__ csr_col,
                              const float *__restrict__ w_csr, int32_t *__restrict__ out_gcol, float *__restrict__ out_w,
                              const int64_t *__restrict__ excl_off, const int64_t *__restrict__ excl_pos, int32_t n_excl) {
    sample_rows_fill_body<true, int64_t, true>(rowptr, n_rows, rows, *n_list, k, -1.0, padding, seed, stream, out_rowptr,
                                               out_row, out_pos, csr_col, w_csr, out_gcol, out_w, excl_off, excl_pos,
                                               n_excl);
}

// ---- weighted fan-outs (include/tfgk.h, "weighted block sampler") -------------------------------------------------
// A listed row's candidates are its kept entries with weight > 0, numbered by virtual position v as excl_real numbers
// them; d+ counts them.  Without replacement the draw is the num = min(k, d+) candidates of smallest (E, v), E the key of
// weighted_key with j = 0, written in ascending CSR position; with padding and k >= d+, draw j is the candidate of smallest
// (E_j, v) with j + 1 in the key's counter.  (E, v) and (E, p) order the same way, since v grows with the real position p.
constexpr int kWeightedRowsPerCta = 64;        // rows per CTA: eight per warp
constexpr int kWarps = kRowsPerCta / 32;
constexpr int kWarpSlots = kThreadRowMax / 32;  // a row of up to kThreadRowMax entries is held by one warp, 4 per lane
constexpr uint64_t kNoKey = ~0ull;              // above every key (keys have no sign bit): entries that cannot be drawn
enum { kWeightedNone = 0, kWeightedAll = 1, kWeightedReplace = 2, kWeightedSelect = 3 };

// sample_rule on d+ for an integer fan-out k >= 0 and padding 0 / 1
__device__ __forceinline__ int weighted_rule(int dplus, int k, int padding, int &num) {
    sample_rule(dplus, k, -1.0, padding, num);
    if (num == 0) return kWeightedNone;
    if (padding && k >= dplus) return kWeightedReplace;
    return num == dplus ? kWeightedAll : kWeightedSelect;
}

// d+ of list row t (global row r): the row's positive entries less its excluded entries of positive weight
template <typename TPos, bool kExcl>
__device__ __forceinline__ int positive_degree(const int32_t *__restrict__ pos_deg, int32_t r,
                                               const float *__restrict__ w_csr, int64_t t,
                                               const int64_t *__restrict__ excl_off, const TPos *__restrict__ excl_pos,
                                               int32_t n_excl) {
    int d = pos_deg[r];
    if constexpr (kExcl)
        if (t < n_excl)
            for (int64_t j = excl_off[t]; j < excl_off[t + 1]; ++j) d -= w_csr[excl_pos[j]] > 0.0f ? 1 : 0;
    return d;
}

template <typename TPos>
struct WeightedRow {
    int64_t t, start, end, o;
    int32_t r;
    int x, num, rule;
    const TPos *ex;
};

template <typename TPos, bool kExcl>
__device__ __forceinline__ WeightedRow<TPos> weighted_row(int64_t t, int32_t r, const int64_t *__restrict__ rowptr,
                                                          const int32_t *__restrict__ pos_deg,
                                                          const float *__restrict__ w_csr, int k, int padding,
                                                          const int64_t *__restrict__ out_rowptr,
                                                          const int64_t *__restrict__ excl_off,
                                                          const TPos *__restrict__ excl_pos, int32_t n_excl) {
    WeightedRow<TPos> R;
    R.t = t;
    R.r = r;
    R.start = rowptr[r];
    R.end = rowptr[r + 1];
    R.o = out_rowptr[t];
    R.x = kExcl ? excl_count(excl_off, n_excl, t) : 0;
    R.ex = kExcl && R.x ? excl_pos + excl_off[t] : nullptr;
    R.rule = weighted_rule(positive_degree<TPos, kExcl>(pos_deg, r, w_csr, t, excl_off, excl_pos, n_excl), k, padding,
                           R.num);
    return R;
}

// the weight of the entry at real position p (0 when it is excluded) and its virtual position v
template <typename TPos, bool kExcl>
__device__ __forceinline__ float entry_weight(const WeightedRow<TPos> &R, const float *__restrict__ w_csr, int64_t p,
                                              uint32_t &v) {
    int before = 0;
    bool hit = false;
    if constexpr (kExcl)
        if (R.x) {
            int lo = 0, hi = R.x;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if ((int64_t)R.ex[mid] < p) lo = mid + 1;
                else hi = mid;
            }
            before = lo;
            hit = lo < R.x && (int64_t)R.ex[lo] == p;
        }
    v = (uint32_t)(p - R.start - before);
    return hit ? 0.0f : w_csr[p];
}

template <bool kBlock, typename TPos>
__device__ __forceinline__ void weighted_emit(const WeightedRow<TPos> &R, int64_t slot, int64_t p, float w,
                                              int32_t *__restrict__ out_row, TPos *__restrict__ out_pos,
                                              const int32_t *__restrict__ csr_col, int32_t *__restrict__ out_gcol,
                                              float *__restrict__ out_w) {
    const int64_t o = R.o + slot;
    if (out_row) out_row[o] = (int32_t)R.t;
    out_pos[o] = (TPos)p;
    if constexpr (kBlock) {
        out_gcol[o] = csr_col[p];
        out_w[o] = w;
    }
}

// (a, pa) < (b, pb) lexicographically
__device__ __forceinline__ bool key_less(uint64_t a, int64_t pa, uint64_t b, int64_t pb) {
    return a < b || (a == b && pa < pb);
}

// exclusive count of `flag` over the CTA in thread order; *total gets the CTA's count
__device__ __forceinline__ int cta_exclusive_count(bool flag, int *s_warp, int &total) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
        const int c = s_warp[w];
        if (w < warp) before += c;
        total += c;
    }
    __syncthreads();                   // s_warp is reused by the next call
    return before + __popc(m & ((1u << lane) - 1u));
}

// a row of at most kThreadRowMax entries on one warp: weights read once, in 128-byte segments, and kept in registers
template <bool kBlock, typename TPos, bool kExcl>
__device__ __forceinline__ void weighted_warp_row(const WeightedRow<TPos> &R, const float *__restrict__ w_csr,
                                                  uint64_t seed, uint32_t stream, int32_t *__restrict__ out_row,
                                                  TPos *__restrict__ out_pos, const int32_t *__restrict__ csr_col,
                                                  int32_t *__restrict__ out_gcol, float *__restrict__ out_w) {
    const int lane = threadIdx.x & 31;
    const int nchunks = (int)((R.end - R.start + 31) >> 5);
    float wt[kWarpSlots];
    uint32_t vv[kWarpSlots];
#pragma unroll
    for (int i = 0; i < kWarpSlots; ++i) {
        const int64_t p = R.start + lane + 32 * i;
        wt[i] = 0.0f;
        vv[i] = 0;
        if (i < nchunks && p < R.end) wt[i] = entry_weight<TPos, kExcl>(R, w_csr, p, vv[i]);
    }
    if (R.rule == kWeightedReplace) {
        for (int j = 0; j < R.num; ++j) {
            uint64_t best = kNoKey;
            int64_t bp = INT64_MAX;
            float bw = 0.0f;
#pragma unroll
            for (int i = 0; i < kWarpSlots; ++i)
                if (wt[i] > 0.0f) {
                    const uint64_t key = weighted_key(seed, stream, vv[i], (uint32_t)R.r, (uint32_t)j + 1u, wt[i]);
                    if (key < best) {          // positions grow with i: a tie keeps the earlier one
                        best = key;
                        bp = lane + 32 * i;
                        bw = wt[i];
                    }
                }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
                const int64_t op = __shfl_xor_sync(0xffffffffu, bp, off);
                const float ow = __shfl_xor_sync(0xffffffffu, bw, off);
                if (key_less(ok, op, best, bp)) {
                    best = ok;
                    bp = op;
                    bw = ow;
                }
            }
            if (lane == 0)
                weighted_emit<kBlock, TPos>(R, j, R.start + bp, bw, out_row, out_pos, csr_col, out_gcol, out_w);
        }
        return;
    }
    bool sel[kWarpSlots];
    if (R.rule == kWeightedSelect) {
        uint64_t key[kWarpSlots];
        int rank[kWarpSlots];
#pragma unroll
        for (int i = 0; i < kWarpSlots; ++i) {
            key[i] = wt[i] > 0.0f ? weighted_key(seed, stream, vv[i], (uint32_t)R.r, 0u, wt[i]) : kNoKey;
            rank[i] = 0;
        }
        // rank of every entry among the row's: the number of entries of smaller (key, position)
#pragma unroll
        for (int i2 = 0; i2 < kWarpSlots; ++i2) {
            if (i2 >= nchunks) break;
            for (int s = 0; s < 32; ++s) {
                const uint64_t kb = __shfl_sync(0xffffffffu, key[i2], s);
                const int pb = s + 32 * i2;
#pragma unroll
                for (int i = 0; i < kWarpSlots; ++i) rank[i] += key_less(kb, pb, key[i], lane + 32 * i) ? 1 : 0;
            }
        }
#pragma unroll
        for (int i = 0; i < kWarpSlots; ++i) sel[i] = key[i] != kNoKey && rank[i] < R.num;
    } else {
#pragma unroll
        for (int i = 0; i < kWarpSlots; ++i) sel[i] = wt[i] > 0.0f;
    }
    int base = 0;
#pragma unroll
    for (int i = 0; i < kWarpSlots; ++i) {
        const unsigned m = __ballot_sync(0xffffffffu, sel[i]);
        if (sel[i])
            weighted_emit<kBlock, TPos>(R, base + __popc(m & ((1u << lane) - 1u)), R.start + lane + 32 * i, wt[i],
                                        out_row, out_pos, csr_col, out_gcol, out_w);
        base += __popc(m);
    }
}

struct WeightedShared {
    int hist[256];
    int warp_count[kWarps];
    uint64_t key[kWarps];
    int64_t pos[kWarps];
    float w[kWarps];
    uint64_t prefix;
    int need, done;
};

// a longer row on the whole CTA.  Without replacement: a radix select of the num smallest keys, eight bits a pass from
// the top, each pass recomputing the keys from their counters (no workspace grows with the row), stopping once the
// bucket of the num-th key is taken whole; then one ordered pass writes the entries below the found prefix and, of those
// equal to it (ties after all 64 bits only), the first in position order.  With replacement: one CTA argmin per draw.
template <bool kBlock, typename TPos, bool kExcl>
__device__ __forceinline__ void weighted_cta_row(const WeightedRow<TPos> &R, const float *__restrict__ w_csr,
                                                 uint64_t seed, uint32_t stream, WeightedShared &sh,
                                                 int32_t *__restrict__ out_row, TPos *__restrict__ out_pos,
                                                 const int32_t *__restrict__ csr_col, int32_t *__restrict__ out_gcol,
                                                 float *__restrict__ out_w) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (R.rule == kWeightedReplace) {
        for (int j = 0; j < R.num; ++j) {
            uint64_t best = kNoKey;
            int64_t bp = INT64_MAX;
            float bw = 0.0f;
            for (int64_t p = R.start + threadIdx.x; p < R.end; p += kRowsPerCta) {
                uint32_t v;
                const float w = entry_weight<TPos, kExcl>(R, w_csr, p, v);
                if (w > 0.0f) {
                    const uint64_t key = weighted_key(seed, stream, v, (uint32_t)R.r, (uint32_t)j + 1u, w);
                    if (key < best) {
                        best = key;
                        bp = p;
                        bw = w;
                    }
                }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
                const int64_t op = __shfl_xor_sync(0xffffffffu, bp, off);
                const float ow = __shfl_xor_sync(0xffffffffu, bw, off);
                if (key_less(ok, op, best, bp)) {
                    best = ok;
                    bp = op;
                    bw = ow;
                }
            }
            if (lane == 0) {
                sh.key[warp] = best;
                sh.pos[warp] = bp;
                sh.w[warp] = bw;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                for (int w = 1; w < kWarps; ++w)
                    if (key_less(sh.key[w], sh.pos[w], best, bp)) {
                        best = sh.key[w];
                        bp = sh.pos[w];
                        bw = sh.w[w];
                    }
                weighted_emit<kBlock, TPos>(R, j, bp, bw, out_row, out_pos, csr_col, out_gcol, out_w);
            }
            __syncthreads();
        }
        return;
    }
    uint64_t prefix = 0;
    int shift = 64, need = R.num;
    if (R.rule == kWeightedSelect) {
        for (int s = 56; s >= 0; s -= 8) {
            sh.hist[threadIdx.x] = 0;
            __syncthreads();
            for (int64_t p = R.start + threadIdx.x; p < R.end; p += kRowsPerCta) {
                uint32_t v;
                const float w = entry_weight<TPos, kExcl>(R, w_csr, p, v);
                if (w > 0.0f) {
                    const uint64_t key = weighted_key(seed, stream, v, (uint32_t)R.r, 0u, w);
                    if (s == 56 || (key >> (s + 8)) == prefix) atomicAdd(&sh.hist[(key >> s) & 255], 1);
                }
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                int b = 0, cum = 0;
                while (cum + sh.hist[b] < need) cum += sh.hist[b++];
                sh.prefix = (prefix << 8) | (uint64_t)b;
                sh.need = need - cum;
                sh.done = sh.hist[b] == need - cum;
            }
            __syncthreads();
            prefix = sh.prefix;
            need = sh.need;
            shift = s;
            const bool done = sh.done;
            __syncthreads();               // every thread has read the pass's result before the next one writes it
            if (done) break;
        }
    }
    int64_t base = 0;
    int eq_base = 0;
    for (int64_t c = R.start; c < R.end; c += kRowsPerCta) {
        const int64_t p = c + threadIdx.x;
        bool lt = false, eq = false;
        float w = 0.0f;
        if (p < R.end) {
            uint32_t v;
            w = entry_weight<TPos, kExcl>(R, w_csr, p, v);
            if (w > 0.0f) {
                if (R.rule == kWeightedAll) {
                    lt = true;
                } else {
                    const uint64_t kp = weighted_key(seed, stream, v, (uint32_t)R.r, 0u, w) >> shift;
                    lt = kp < prefix;
                    eq = kp == prefix;
                }
            }
        }
        int n_eq, n_sel;
        const int eq_rank = eq_base + cta_exclusive_count(eq, sh.warp_count, n_eq);
        const bool sel = lt || (eq && eq_rank < need);
        const int slot = cta_exclusive_count(sel, sh.warp_count, n_sel);
        if (sel) weighted_emit<kBlock, TPos>(R, base + slot, p, w, out_row, out_pos, csr_col, out_gcol, out_w);
        eq_base += n_eq;
        base += n_sel;
    }
}

// The weighted fill: kWeightedRowsPerCta listed rows per CTA, a warp per row up to kThreadRowMax entries, then the
// longer rows one after another on the whole CTA.  n_list_dev (the block sampler's device count) overrides n_list.
// The explicit minimum of one CTA per SM lets ptxas take the 74-80 registers the keys need: left to itself it chose 64
// and spilled 4-20 bytes.
template <bool kBlock, typename TPos, bool kExcl>
__global__ void __launch_bounds__(kRowsPerCta, 1)
weighted_fill_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                     const int32_t *__restrict__ n_list_dev, int32_t n_list, int k, int padding,
                     const int32_t *__restrict__ pos_deg, const float *__restrict__ w_csr, uint64_t seed, uint32_t stream,
                     const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row, TPos *__restrict__ out_pos,
                     const int32_t *__restrict__ csr_col, int32_t *__restrict__ out_gcol, float *__restrict__ out_w,
                     const int64_t *__restrict__ excl_off, const TPos *__restrict__ excl_pos, int32_t n_excl) {
    __shared__ int32_t long_rows[kWeightedRowsPerCta];
    __shared__ int n_long;
    __shared__ WeightedShared sh;
    if (n_list_dev) n_list = *n_list_dev;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    for (int q = warp; q < kWeightedRowsPerCta; q += kWarps) {
        const int64_t t = (int64_t)blockIdx.x * kWeightedRowsPerCta + q;
        if (t >= n_list) break;
        const int32_t r = rows[t];
        if (r < 0 || r >= n_rows) continue;
        const WeightedRow<TPos> R = weighted_row<TPos, kExcl>(t, r, rowptr, pos_deg, w_csr, k, padding, out_rowptr,
                                                              excl_off, excl_pos, n_excl);
        if (R.rule == kWeightedNone) continue;
        if (R.end - R.start > kThreadRowMax) {
            if (lane == 0) long_rows[atomicAdd(&n_long, 1)] = q;     // rows write disjoint ranges: any order
            continue;
        }
        weighted_warp_row<kBlock, TPos, kExcl>(R, w_csr, seed, stream, out_row, out_pos, csr_col, out_gcol, out_w);
    }
    __syncthreads();
    const int nl = n_long;
    for (int i = 0; i < nl; ++i) {
        const int64_t t = (int64_t)blockIdx.x * kWeightedRowsPerCta + long_rows[i];
        const WeightedRow<TPos> R = weighted_row<TPos, kExcl>(t, rows[t], rowptr, pos_deg, w_csr, k, padding, out_rowptr,
                                                              excl_off, excl_pos, n_excl);
        weighted_cta_row<kBlock, TPos, kExcl>(R, w_csr, seed, stream, sh, out_row, out_pos, csr_col, out_gcol, out_w);
    }
}

// per-row counts of the weighted rule; K13's form (n_list on the host, listed rows outside [0, n_rows) counted in n_bad)
// when n_bad is set, the block sampler's otherwise (rows past the device count contribute 0)
template <typename TPos, bool kExcl>
__global__ void weighted_count_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
                                      const int32_t *__restrict__ n_list_dev, int32_t cap, int k, int padding,
                                      const int32_t *__restrict__ pos_deg, const float *__restrict__ w_csr,
                                      int32_t *__restrict__ cnt, int32_t *__restrict__ n_bad,
                                      const int64_t *__restrict__ excl_off, const TPos *__restrict__ excl_pos,
                                      int32_t n_excl) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cap) return;
    int num = 0;
    if (!n_list_dev || t < *n_list_dev) {
        const int32_t r = rows[t];
        if (r >= 0 && r < n_rows)
            weighted_rule(positive_degree<TPos, kExcl>(pos_deg, r, w_csr, t, excl_off, excl_pos, n_excl), k, padding,
                          num);
        else if (n_bad)
            atomicAdd(n_bad, 1);
    }
    cnt[t] = num;
}

// one warp per row: the entries of weight > 0, and (atomically, into n_invalid) those negative, NaN or infinite
__global__ void positive_degree_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const float *__restrict__ w,
                                       int64_t w_base, int32_t *__restrict__ pos_deg, int32_t *__restrict__ n_invalid) {
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return;                    // whole warps
    int pos = 0, bad = 0;
    for (int64_t p = rowptr[r] + lane; p < rowptr[r + 1]; p += 32) {
        const float x = w[p - w_base];
        pos += x > 0.0f && x <= FLT_MAX ? 1 : 0;
        bad += !(x >= 0.0f && x <= FLT_MAX) ? 1 : 0;
    }
    pos = __reduce_add_sync(0xffffffffu, pos);
    bad = __reduce_add_sync(0xffffffffu, bad);
    if (lane == 0) {
        pos_deg[r] = pos;
        if (bad) atomicAdd(n_invalid, bad);
    }
}

// ---- layer-neighbour (LABOR-0) fan-outs (include/tfgk.h, "LABOR block sampler") ------------------------------------
// Row t keeps its candidate (t, c) iff u_c * d < k 2^32, u_c one variate per column node id c under the hop key, so rows
// that share a neighbour keep it together.  Rows of d <= k keep every candidate; k = 0 keeps none.  The count and the
// fill visit a row with the same predicate, in CSR order: one warp for a row of up to kThreadRowMax entries (columns
// read 32 at a time, 128 bytes), the whole CTA for a longer one (kRowsPerCta at a time).
enum { kLaborNone = 0, kLaborAll = 1, kLaborDraw = 2 };

__device__ __forceinline__ bool labor_keep(int32_t c, uint64_t seed, uint32_t stream, int d, int k) {
    const uint32_t u = philox4x32_10((uint32_t)c, 0u, stream, 0u, (uint32_t)seed, (uint32_t)(seed >> 32)).v[0];
    return (uint64_t)u * (uint64_t)d < ((uint64_t)k << 32);
}

// whether real position p is one of the row's x excluded positions ex[0, x) (ascending)
template <typename TPos>
__device__ __forceinline__ bool excl_hit(const TPos *__restrict__ ex, int x, int64_t p) {
    int lo = 0, hi = x;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((int64_t)ex[mid] < p) lo = mid + 1;
        else hi = mid;
    }
    return lo < x && (int64_t)ex[lo] == p;
}

// listed row t's rule: WeightedRow with num = d (its candidates) and rule kLabor*
template <typename TPos, bool kExcl>
__device__ __forceinline__ WeightedRow<TPos> labor_row(int64_t t, int32_t r, const int64_t *__restrict__ rowptr, int k,
                                                       const int64_t *__restrict__ excl_off,
                                                       const TPos *__restrict__ excl_pos, int32_t n_excl) {
    WeightedRow<TPos> R;
    R.t = t;
    R.r = r;
    R.start = rowptr[r];
    R.end = rowptr[r + 1];
    R.o = 0;
    R.x = kExcl ? excl_count(excl_off, n_excl, t) : 0;
    R.ex = kExcl && R.x ? excl_pos + excl_off[t] : nullptr;
    R.num = (int)(R.end - R.start) - R.x;
    R.rule = (k == 0 || R.num == 0) ? kLaborNone : R.num <= k ? kLaborAll : kLaborDraw;
    return R;
}

// Visits row R's entries kWidth at a time (32: the calling warp, kRowsPerCta: the CTA) and returns how many it keeps;
// kFill writes them at R.o + slot in CSR order, with their list row, global column and weight (w_csr null: 1.0f).
template <bool kFill, int kWidth, typename TPos, bool kExcl>
__device__ __forceinline__ int labor_visit(const WeightedRow<TPos> &R, const int32_t *__restrict__ csr_col,
                                           const float *__restrict__ w_csr, int k, uint64_t seed, uint32_t stream,
                                           int *s_warp, int32_t *__restrict__ out_row, int32_t *__restrict__ out_gcol,
                                           float *__restrict__ out_w) {
    const int i = kWidth == 32 ? (int)(threadIdx.x & 31) : (int)threadIdx.x;
    int base = 0;
    for (int64_t c0 = R.start; c0 < R.end; c0 += kWidth) {
        const int64_t p = c0 + i;
        bool keep = false;
        int32_t c = 0;
        if (p < R.end && !(kExcl && R.x && excl_hit(R.ex, R.x, p))) {
            c = csr_col[p];
            keep = R.rule == kLaborAll || labor_keep(c, seed, stream, R.num, k);
        }
        int slot, n;
        if constexpr (kWidth == 32) {
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            slot = __popc(m & ((1u << i) - 1u));
            n = __popc(m);
        } else {
            slot = cta_exclusive_count(keep, s_warp, n);
        }
        if (kFill && keep) {
            const int64_t o = R.o + base + slot;
            out_row[o] = (int32_t)R.t;
            out_gcol[o] = c;
            out_w[o] = w_csr ? w_csr[p] : 1.0f;
        }
        base += n;
    }
    return base;
}

// The count (kFill false: cnt[t] for every t < cap, 0 past the device count n_list) and the fill of the LABOR rule over
// kWeightedRowsPerCta listed rows per CTA: a warp per row, then the rows longer than kThreadRowMax one after another on
// the CTA.  The count skips the column reads of rows that keep every candidate or none.  The minimum of 4 CTAs per SM,
// as for block_fill_mapped_kernel: left to itself ptxas chose 40-48 registers and spilled 4-8 bytes.
template <bool kFill, typename TPos, bool kExcl>
__global__ void __launch_bounds__(kRowsPerCta, 4)
labor_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ rows,
             const int32_t *__restrict__ n_list_dev, int32_t cap, int k, uint64_t seed, uint32_t stream,
             const int32_t *__restrict__ csr_col, const float *__restrict__ w_csr, int32_t *__restrict__ cnt,
             const int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row, int32_t *__restrict__ out_gcol,
             float *__restrict__ out_w, const int64_t *__restrict__ excl_off, const TPos *__restrict__ excl_pos,
             int32_t n_excl) {
    __shared__ int32_t long_rows[kWeightedRowsPerCta];
    __shared__ int n_long;
    __shared__ int s_warp[kWarps];
    const int n_list = *n_list_dev;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) n_long = 0;
    __syncthreads();
    for (int q = warp; q < kWeightedRowsPerCta; q += kWarps) {
        const int64_t t = (int64_t)blockIdx.x * kWeightedRowsPerCta + q;
        if (t >= cap) break;
        const int32_t r = t < n_list ? rows[t] : -1;
        int num = 0;
        if (r >= 0 && r < n_rows) {
            WeightedRow<TPos> R = labor_row<TPos, kExcl>(t, r, rowptr, k, excl_off, excl_pos, n_excl);
            if (!kFill && R.rule == kLaborAll) {
                num = R.num;
            } else if (R.rule != kLaborNone) {
                if (R.end - R.start > kThreadRowMax) {
                    if (lane == 0) long_rows[atomicAdd(&n_long, 1)] = q;     // rows write disjoint ranges: any order
                    continue;
                }
                if constexpr (kFill) R.o = out_rowptr[t];
                num = labor_visit<kFill, 32, TPos, kExcl>(R, csr_col, w_csr, k, seed, stream, nullptr, out_row,
                                                          out_gcol, out_w);
            }
        }
        if (!kFill && lane == 0) cnt[t] = num;
    }
    __syncthreads();
    const int nl = n_long;
    for (int j = 0; j < nl; ++j) {
        const int64_t t = (int64_t)blockIdx.x * kWeightedRowsPerCta + long_rows[j];
        WeightedRow<TPos> R = labor_row<TPos, kExcl>(t, rows[t], rowptr, k, excl_off, excl_pos, n_excl);
        if constexpr (kFill) R.o = out_rowptr[t];
        const int num = labor_visit<kFill, kRowsPerCta, TPos, kExcl>(R, csr_col, w_csr, k, seed, stream, s_warp,
                                                                     out_row, out_gcol, out_w);
        if (!kFill && threadIdx.x == 0) cnt[t] = num;
    }
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

// items [0, S) move edge p of row r to p + r; items [S, S + n_dst] write out_rowptr[r] and, for r < n_dst, the self edge
// (r, r) after the row's sampled edges.  Every output slot has exactly one writer.
__global__ void block_self_loops_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ row,
                                        const int32_t *__restrict__ col, int64_t S, int32_t n_dst,
                                        int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row,
                                        int32_t *__restrict__ out_col) {
    const int64_t n = S + n_dst + 1;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        if (t < S) {
            const int32_t r = row[t];
            out_row[t + r] = r;
            out_col[t + r] = col[t];
        } else {
            const int32_t r = (int32_t)(t - S);
            out_rowptr[r] = rowptr[r] + r;
            if (r < n_dst) {
                const int64_t q = rowptr[r + 1] + r;
                out_row[q] = r;
                out_col[q] = r;
            }
        }
    }
}

// f(v) of tfgk_block_gcn_values_f32: deg_inv_kernel's arithmetic on the full graph's degree d = rowsum + deg_fill
__device__ __forceinline__ float gcn_degree_factor(float rowsum, float deg_fill, int norm) {
    const float d = __fadd_rn(rowsum, deg_fill);
    float v = norm == TFGK_GCN_NORM_BOTH ? __frsqrt_rn(d) : __frcp_rn(d);
    if (isinf(v) || isnan(v)) v = 0.0f;
    return v;
}

// v times the factors of its row (fr) and column (fc) in scale_edges_kernel's order: dl on the left, dr on the right
__device__ __forceinline__ float gcn_scale(float v, int norm, float fr, float fc) {
    if (norm != TFGK_GCN_NORM_RIGHT) v = __fmul_rn(fr, v);
    if (norm != TFGK_GCN_NORM_LEFT) v = __fmul_rn(v, fc);
    return v;
}

// items [0, S): edge t, whose row is the last r with rowptr[r] <= t; items [S, S + n_dst) (loop modes only): the self
// loop of row t - S.  Every output slot has exactly one writer.  kExcl: row r < n_excl had x_r of its n_g entries
// excluded, and its scale is (n_g - x_r) / k_r.
template <bool kExcl>
__device__ __forceinline__ void block_gcn_values_body(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ gcol,
                                                      const float *__restrict__ w, int64_t S,
                                                      const int32_t *__restrict__ dst, int32_t n_dst,
                                                      const int64_t *__restrict__ g_rowptr,
                                                      const float *__restrict__ g_rowsum, int norm, int loop,
                                                      float deg_fill, float fill, float *__restrict__ out,
                                                      const int64_t *__restrict__ excl_off, int32_t n_excl) {
    const int64_t n = S + (loop != TFGK_GCN_LOOP_NONE ? n_dst : 0);
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
        if (t < S) {
            int32_t lo = 0, hi = n_dst - 1;
            while (lo < hi) {
                const int32_t mid = lo + ((hi - lo + 1) >> 1);
                if (rowptr[mid] <= t) lo = mid;
                else hi = mid - 1;
            }
            const int32_t g = dst[lo];
            const float fr = norm != TFGK_GCN_NORM_RIGHT ? gcn_degree_factor(g_rowsum[g], deg_fill, norm) : 0.0f;
            const float fc = norm != TFGK_GCN_NORM_LEFT ? gcn_degree_factor(g_rowsum[gcol[t]], deg_fill, norm) : 0.0f;
            const float v = gcn_scale(w ? w[t] : 1.0f, norm, fr, fc);
            const float s = __fdiv_rn((float)(g_rowptr[g + 1] - g_rowptr[g] - (kExcl ? excl_count(excl_off, n_excl, lo) : 0)),
                                      (float)(rowptr[lo + 1] - rowptr[lo]));
            out[loop != TFGK_GCN_LOOP_NONE ? t + lo : t] = __fmul_rn(s, v);
        } else {
            const int32_t r = (int32_t)(t - S);
            float v = fill;
            if (loop == TFGK_GCN_LOOP_NORMED) {
                const float f = gcn_degree_factor(g_rowsum[dst[r]], deg_fill, norm);
                v = gcn_scale(fill, norm, f, f);
            }
            out[rowptr[r + 1] + r] = v;
        }
    }
}

__global__ void block_gcn_values_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ gcol,
                                        const float *__restrict__ w, int64_t S, const int32_t *__restrict__ dst,
                                        int32_t n_dst, const int64_t *__restrict__ g_rowptr,
                                        const float *__restrict__ g_rowsum, int norm, int loop, float deg_fill, float fill,
                                        float *__restrict__ out) {
    block_gcn_values_body<false>(rowptr, gcol, w, S, dst, n_dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, out,
                                 nullptr, 0);
}

__global__ void block_gcn_values_excl_kernel(const int64_t *__restrict__ rowptr, const int32_t *__restrict__ gcol,
                                             const float *__restrict__ w, int64_t S, const int32_t *__restrict__ dst,
                                             int32_t n_dst, const int64_t *__restrict__ g_rowptr,
                                             const float *__restrict__ g_rowsum, int norm, int loop, float deg_fill,
                                             float fill, const int64_t *__restrict__ excl_off, int32_t n_excl,
                                             float *__restrict__ out) {
    block_gcn_values_body<true>(rowptr, gcol, w, S, dst, n_dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, out,
                                excl_off, n_excl);
}

// ---- link prediction on blocks: pair begin, tail negatives and the exclusion lists ---------------------------------
// endpoint e of a pair list is pair e >> 1's source (e even) or destination (e odd): the seeds' first-occurrence order
__global__ void pair_ends_kernel(const int32_t *__restrict__ pair_row, const int32_t *__restrict__ pair_col, int64_t P,
                                 int32_t *__restrict__ ends) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P; e += (int64_t)gridDim.x * blockDim.x)
        ends[e] = (e & 1) ? pair_col[e >> 1] : pair_row[e >> 1];
}

// the pairs relabelled, int32 [2, P / 2]: sources, then destinations
__global__ void pair_gather_kernel(const int32_t *__restrict__ ends, int64_t P, int32_t N, const int32_t *__restrict__ map,
                                   int32_t *__restrict__ local) {
    const int64_t n_pairs = P >> 1;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P; e += (int64_t)gridDim.x * blockDim.x) {
        const int32_t id = ends[e];
        local[(e & 1) * n_pairs + (e >> 1)] = (id >= 0 && id < N) ? map[id] : -1;
    }
}

// 64-bit multiply-shift: a 32-bit one gives ceil(2^32 / N) preimages to 2^32 mod N of the ids and one fewer to the rest,
// a relative over-weight of N / 2^32 (5.9 % at N = 244 M); over 64 bits it is at most N / 2^64
__global__ void tail_negatives_kernel(const int32_t *__restrict__ src, int64_t n, int32_t q, uint32_t N, uint64_t seed,
                                      uint32_t stream, int32_t *__restrict__ out_row, int32_t *__restrict__ out_col) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        out_row[i] = src[i / q];
        out_col[i] = (int32_t)random_below64(seed, stream, (uint64_t)i, N);
    }
}

// [tbeg[s], tend[s]): the targets of seed s in the list sorted by (source, destination); sources outside [0, cap) (-1:
// an endpoint outside the graph) are skipped
__global__ void excl_mark_kernel(const int32_t *__restrict__ ts, int64_t T, int32_t cap, int32_t *__restrict__ tbeg,
                                 int32_t *__restrict__ tend) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < T; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t s = ts[i];
        if (s < 0 || s >= cap) continue;
        if (i == 0 || ts[i - 1] != s) tbeg[s] = (int32_t)i;
        if (i == T - 1 || ts[i + 1] != s) tend[s] = (int32_t)(i + 1);
    }
}

// one warp per seed row with targets, 32 entries at a time: an entry is excluded when its column is among the row's
// sorted target destinations (binary search, so a repeated target excludes an entry once).  The count pass writes x_t;
// the fill pass writes the excluded positions in CSR order from excl_off[t] (ballot and prefix count).
template <bool kFill, typename TPos>
__global__ void excl_scan_kernel(const int64_t *__restrict__ rowptr, int32_t n_rows, const int32_t *__restrict__ col,
                                 const int32_t *__restrict__ nodes, int32_t cap, const int32_t *__restrict__ td,
                                 const int32_t *__restrict__ tbeg, const int32_t *__restrict__ tend,
                                 int32_t *__restrict__ cnt, const int64_t *__restrict__ excl_off, TPos *__restrict__ out) {
    const int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (t >= cap) return;                       // whole warps
    const int32_t b = tbeg[t], e = tend[t];
    int64_t n = kFill ? excl_off[t] : 0;
    if (e > b) {
        const int32_t r = nodes[t];
        if (r >= 0 && r < n_rows) {
            const int64_t end = rowptr[r + 1];
            for (int64_t p0 = rowptr[r]; p0 < end; p0 += 32) {
                const int64_t p = p0 + lane;
                bool hit = false;
                if (p < end) {
                    const int32_t c = col[p];
                    int32_t lo = b, hi = e;
                    while (lo < hi) {
                        const int32_t mid = (lo + hi) >> 1;
                        if (td[mid] < c) lo = mid + 1;
                        else hi = mid;
                    }
                    hit = lo < e && td[lo] == c;
                }
                const unsigned mask = __ballot_sync(0xffffffffu, hit);
                if constexpr (kFill)
                    if (hit) out[n + __popc(mask & ((1u << lane) - 1u))] = (TPos)p;
                n += __popc(mask);
            }
        }
    }
    if constexpr (!kFill)
        if (lane == 0) cnt[t] = (int32_t)n;
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

int tfgk_neighbor_sample_rows_count_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list,
                                             int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                             int64_t *out_rowptr, int64_t *total_host, void *workspace,
                                             size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n_rows >= 0 && n_list >= 0, "neighbor_sample_rows_count_weighted: bad size");
    TFGK_CHECK_ARG(k >= 0 && (padding == 0 || padding == 1), "neighbor_sample_rows_count_weighted: the weighted rule "
                   "takes an integer fan-out and padding 0 or 1");
    TFGK_CHECK_ARG(total_host != nullptr && out_rowptr != nullptr, "neighbor_sample_rows_count_weighted: null pointer");
    *total_host = 0;
    cudaStream_t st = as_stream(stream);
    if (n_list == 0) {
        TFGK_CUDA(cudaMemsetAsync(out_rowptr, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr && rows && pos_deg && w_csr, "neighbor_sample_rows_count_weighted: null pointer");
    size_t need = 0;
    tfgk_neighbor_sample_workspace_bytes(n_list, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "neighbor_sample_rows_count_weighted: workspace too small (%zu < %zu bytes)",
                         workspace_bytes, need);
    char *ws = static_cast<char *>(workspace);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + align_up(((size_t)n_list + 1) * 4));
    int32_t *n_bad = reinterpret_cast<int32_t *>(ws + need - 256);
    TFGK_CUDA(cudaMemsetAsync(n_bad, 0, 4, st));
    weighted_count_kernel<int32_t, false><<<(unsigned)ceil_div64(n_list, 256), 256, 0, st>>>(
        rowptr, n_rows, rows, nullptr, n_list, k, padding, pos_deg, w_csr, cnt, n_bad, nullptr, nullptr, 0);
    TFGK_LAUNCH_CHECK();
    int rc = exclusive_scan<int32_t, int64_t>(cnt, n_list, (int64_t)n_list + 1, out_rowptr, sums, st);
    if (rc != TFGK_OK) return rc;
    int32_t bad = 0;
    TFGK_CUDA(cudaMemcpyAsync(total_host, out_rowptr + n_list, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(&bad, n_bad, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (bad) {
        *total_host = 0;
        return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "neighbor_sample_rows_count_weighted: %d listed rows outside [0, %d)",
                         bad, n_rows);
    }
    TFGK_CHECK_ARG(*total_host < (1ll << 31) - 1, "neighbor_sample_rows_count_weighted: %lld sampled edges exceed int32 "
                   "positions", (long long)*total_host);
    return TFGK_OK;
}

int tfgk_neighbor_sample_rows_fill_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *rows, int32_t n_list,
                                            int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                            uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                            int32_t *out_row, int32_t *out_pos, void *stream) {
    TFGK_CHECK_ARG(n_rows >= 0 && n_list >= 0, "neighbor_sample_rows_fill_weighted: bad size");
    TFGK_CHECK_ARG(k >= 0 && (padding == 0 || padding == 1), "neighbor_sample_rows_fill_weighted: the weighted rule "
                   "takes an integer fan-out and padding 0 or 1");
    if (n_list == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && rows && pos_deg && w_csr && out_rowptr && out_pos,
                   "neighbor_sample_rows_fill_weighted: null pointer");
    weighted_fill_kernel<false, int32_t, false><<<(unsigned)ceil_div64(n_list, kWeightedRowsPerCta), kRowsPerCta, 0,
                                                  as_stream(stream)>>>(
        rowptr, n_rows, rows, nullptr, n_list, k, padding, pos_deg, w_csr, seed, rng_stream, out_rowptr, out_row, out_pos,
        nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_csr_positive_degree_f32(const int64_t *rowptr, int32_t n_rows, const float *w, int64_t w_base,
                                 int32_t *pos_deg, int32_t *n_invalid, void *stream) {
    TFGK_CHECK_ARG(n_rows >= 0 && w_base >= 0, "csr_positive_degree: bad size");
    if (n_rows == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && w && pos_deg && n_invalid, "csr_positive_degree: null pointer");
    positive_degree_kernel<<<(unsigned)ceil_div64((int64_t)n_rows * 32, 256), 256, 0, as_stream(stream)>>>(
        rowptr, n_rows, w, w_base, pos_deg, n_invalid);
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

}  // extern "C"

// the frontier's relabelling once the list nodes[0, n_nodes) is in the map and the counters are cleared: the ids of
// cols[0, S) not in the list are appended in first-occurrence order and local_col written; then the map is reset and
// the three counters read back into c (one synchronisation).  ws / need: tfgk_relabel_workspace_bytes(S)'s layout.
static int frontier_relabel(const int32_t *cols, int64_t S, int32_t N, int32_t *nodes, int32_t n_nodes, int32_t *map,
                            int32_t *local_col, char *ws, size_t need, int32_t *c, cudaStream_t st) {
    int32_t *flag = reinterpret_cast<int32_t *>(ws);
    int32_t *off = reinterpret_cast<int32_t *>(ws + align_up((size_t)(S + 1) * 4));
    int32_t *sums = reinterpret_cast<int32_t *>(ws + 2 * align_up((size_t)(S + 1) * 4));
    int32_t *counters = reinterpret_cast<int32_t *>(ws + need - 256);
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
    return read_counters(counters, c, st);
}

extern "C" {

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
    int32_t *counters = reinterpret_cast<int32_t *>(ws + need - 256);
    TFGK_CUDA(cudaMemsetAsync(counters, 0, 3 * 4, st));
    if (n_nodes) {
        node_scatter_kernel<<<grid_for(n_nodes), 256, 0, st>>>(nodes, n_nodes, N, map, counters);
        TFGK_LAUNCH_CHECK();
    }
    int32_t c[3];
    int rc = frontier_relabel(cols, S, N, nodes, n_nodes, map, local_col, ws, need, c, st);
    if (rc != TFGK_OK) return rc;
    if (c[kBadIds]) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "frontier: %d node ids outside [0, %d)", c[kBadIds], N);
    *n_dup_host = c[kDupIds];
    *n_new_host = c[kNewIds];
    return TFGK_OK;
}

// ---- block sampler (include/tfgk.h) -----------------------------------------------------------------------------
namespace {
// pos_bytes: the size of a CSR position, 4 on the device, 8 for a CSR in host memory
struct BlockWorkspace {
    size_t off_sums, off_pos, off_flag, off_off, total;
    BlockWorkspace(int32_t cap_list, int64_t cap_edges, size_t pos_bytes = 4) {
        size_t sums = scan_scratch_bytes((int64_t)cap_list + 1);
        if (scan_scratch_bytes(cap_edges + 1) > sums) sums = scan_scratch_bytes(cap_edges + 1);
        off_sums = align_up(((size_t)cap_list + 1) * 4);                   // per-row counts first
        off_pos = off_sums + sums;
        off_flag = off_pos + align_up((size_t)(cap_edges > 0 ? cap_edges : 1) * pos_bytes);
        off_off = off_flag + align_up((size_t)(cap_edges + 1) * 4);
        total = off_off + align_up((size_t)(cap_edges + 1) * 4);
    }
};
}  // namespace

static int block_workspace_check(const char *fn, int32_t cap_list, int64_t cap_edges, void *workspace,
                                 size_t workspace_bytes, size_t pos_bytes = 4) {
    const size_t need = BlockWorkspace(cap_list, cap_edges, pos_bytes).total;
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

int tfgk_block_sample_mapped_workspace_bytes(int32_t cap_list, int64_t cap_edges, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && cap_list >= 0 && cap_edges >= 0 && cap_edges < (1ll << 31) - 1,
                   "block_sample_mapped_workspace_bytes: bad argument");
    *out_bytes = BlockWorkspace(cap_list, cap_edges, 8).total;
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

}  // extern "C"

// tfgk_block_sample_count, _count_excl (excl_off null: no exclusions), their _weighted twins (pos_deg set: the
// weighted rule over d+, which reads the weights w_csr at the excluded positions excl_pos) and their _labor twins
// (labor_col set: the LABOR rule over the CSR columns labor_col under hop key seed)
template <typename TPos = int32_t>
static int block_sample_count(const char *fn, const int64_t *rowptr, int32_t n_rows, const int32_t *nodes,
                              const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding,
                              const int64_t *excl_off, int32_t n_excl, int64_t *out_rowptr, void *workspace,
                              size_t workspace_bytes, void *stream, const int32_t *pos_deg = nullptr,
                              const float *w_csr = nullptr, const TPos *excl_pos = nullptr,
                              const int32_t *labor_col = nullptr, uint64_t seed = 0, uint32_t rng_stream = 0) {
    int rc = check_sample_mode(fn, k, -1.0, padding);
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(n_rows >= 0 && hop >= 0 && hop < n_hops && cap_list >= 0 && n_excl >= 0, "%s: bad size", fn);
    TFGK_CHECK_ARG(state != nullptr && out_rowptr != nullptr, "%s: null pointer", fn);
    cudaStream_t st = as_stream(stream);
    if (cap_list == 0) {
        TFGK_CUDA(cudaMemsetAsync(out_rowptr, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr != nullptr && nodes != nullptr, "%s: null rowptr or node list", fn);
    if ((rc = block_workspace_check(fn, cap_list, 0, workspace, workspace_bytes)) != TFGK_OK) return rc;
    char *ws = static_cast<char *>(workspace);
    const BlockWorkspace L(cap_list, 0);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws);
    const unsigned grid = (unsigned)ceil_div64(cap_list, 256);
    if (labor_col) {
        TFGK_CHECK_ARG(k >= 0 && padding == 0, "%s: the LABOR rule takes an integer fan-out and no padding", fn);
        TFGK_CHECK_ARG(!excl_off || excl_pos, "%s: null exclusion positions", fn);
        const unsigned lgrid = (unsigned)ceil_div64(cap_list, kWeightedRowsPerCta);
        if (excl_off)
            labor_kernel<false, TPos, true><<<lgrid, kRowsPerCta, 0, st>>>(
                rowptr, n_rows, nodes, state + kStateSizes + hop, cap_list, k, seed, rng_stream, labor_col, nullptr, cnt,
                nullptr, nullptr, nullptr, nullptr, excl_off, excl_pos, n_excl);
        else
            labor_kernel<false, TPos, false><<<lgrid, kRowsPerCta, 0, st>>>(
                rowptr, n_rows, nodes, state + kStateSizes + hop, cap_list, k, seed, rng_stream, labor_col, nullptr, cnt,
                nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0);
    } else if (pos_deg) {
        TFGK_CHECK_ARG(k >= 0 && padding != TFGK_SAMPLE_HEAD, "%s: the weighted rule takes an integer fan-out and no "
                       "head rule", fn);
        TFGK_CHECK_ARG(!excl_off || (w_csr && excl_pos), "%s: null weights or exclusion list", fn);
        if (excl_off)
            weighted_count_kernel<TPos, true><<<grid, 256, 0, st>>>(rowptr, n_rows, nodes, state + kStateSizes + hop,
                                                                    cap_list, k, padding, pos_deg, w_csr, cnt, nullptr,
                                                                    excl_off, excl_pos, n_excl);
        else
            weighted_count_kernel<TPos, false><<<grid, 256, 0, st>>>(rowptr, n_rows, nodes, state + kStateSizes + hop,
                                                                     cap_list, k, padding, pos_deg, w_csr, cnt, nullptr,
                                                                     nullptr, nullptr, 0);
    } else if (excl_off)
        block_count_excl_kernel<<<grid, 256, 0, st>>>(rowptr, n_rows, nodes, state + kStateSizes + hop, cap_list, k,
                                                      padding, cnt, excl_off, n_excl);
    else
        block_count_kernel<<<grid, 256, 0, st>>>(rowptr, n_rows, nodes, state + kStateSizes + hop, cap_list, k, padding,
                                                 cnt);
    TFGK_LAUNCH_CHECK();
    return exclusive_scan<int32_t, int64_t>(cnt, cap_list, (int64_t)cap_list + 1, out_rowptr,
                                            reinterpret_cast<int64_t *>(ws + L.off_sums), st);
}

extern "C" {

int tfgk_block_sample_count(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                            int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding, int64_t *out_rowptr,
                            void *workspace, size_t workspace_bytes, void *stream) {
    return block_sample_count("block_sample_count", rowptr, n_rows, nodes, state, hop, n_hops, cap_list, k, padding,
                              nullptr, 0, out_rowptr, workspace, workspace_bytes, stream);
}

int tfgk_block_sample_count_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                                 int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding,
                                 const int64_t *excl_off, int32_t n_excl, int64_t *out_rowptr, void *workspace,
                                 size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr, "block_sample_count_excl: null exclusion offsets");
    return block_sample_count("block_sample_count_excl", rowptr, n_rows, nodes, state, hop, n_hops, cap_list, k, padding,
                              excl_off, n_excl, out_rowptr, workspace, workspace_bytes, stream);
}

int tfgk_block_sample_count_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes, const int32_t *state,
                                     int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k, int padding,
                                     const int32_t *pos_deg, const float *w_csr, int64_t *out_rowptr, void *workspace,
                                     size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr, "block_sample_count_weighted: null positive degrees");
    return block_sample_count<int32_t>("block_sample_count_weighted", rowptr, n_rows, nodes, state, hop, n_hops,
                                       cap_list, k, padding, nullptr, 0, out_rowptr, workspace, workspace_bytes, stream,
                                       pos_deg, w_csr, nullptr);
}

int tfgk_block_sample_count_weighted_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes,
                                          const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                          int padding, const int32_t *pos_deg, const float *w_csr,
                                          const int64_t *excl_off, const int32_t *excl_pos, int32_t n_excl,
                                          int64_t *out_rowptr, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr && excl_off != nullptr, "block_sample_count_weighted_excl: null positive degrees "
                   "or exclusion offsets");
    return block_sample_count<int32_t>("block_sample_count_weighted_excl", rowptr, n_rows, nodes, state, hop, n_hops,
                                       cap_list, k, padding, excl_off, n_excl, out_rowptr, workspace, workspace_bytes,
                                       stream, pos_deg, w_csr, excl_pos);
}

int tfgk_block_sample_count_weighted_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *nodes,
                                                 const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                                                 int32_t k, int padding, const int32_t *pos_deg, const float *w_csr,
                                                 const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                                 int64_t *out_rowptr, void *workspace, size_t workspace_bytes,
                                                 void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr && excl_off != nullptr, "block_sample_count_weighted_mapped_excl: null positive "
                   "degrees or exclusion offsets");
    return block_sample_count<int64_t>("block_sample_count_weighted_mapped_excl", rowptr, n_rows, nodes, state, hop,
                                       n_hops, cap_list, k, padding, excl_off, n_excl, out_rowptr, workspace,
                                       workspace_bytes, stream, pos_deg, w_csr, excl_pos);
}

int tfgk_block_sample_count_labor(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                  const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                  uint64_t seed, uint32_t rng_stream, int64_t *out_rowptr, void *workspace,
                                  size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(col != nullptr, "block_sample_count_labor: null columns");
    return block_sample_count<int32_t>("block_sample_count_labor", rowptr, n_rows, nodes, state, hop, n_hops, cap_list,
                                       k, 0, nullptr, 0, out_rowptr, workspace, workspace_bytes, stream, nullptr, nullptr,
                                       nullptr, col, seed, rng_stream);
}

int tfgk_block_sample_count_labor_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                       const int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list, int32_t k,
                                       uint64_t seed, uint32_t rng_stream, const int64_t *excl_off,
                                       const int32_t *excl_pos, int32_t n_excl, int64_t *out_rowptr, void *workspace,
                                       size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(col != nullptr && excl_off != nullptr, "block_sample_count_labor_excl: null columns or exclusion "
                   "offsets");
    return block_sample_count<int32_t>("block_sample_count_labor_excl", rowptr, n_rows, nodes, state, hop, n_hops,
                                       cap_list, k, 0, excl_off, n_excl, out_rowptr, workspace, workspace_bytes, stream,
                                       nullptr, nullptr, excl_pos, col, seed, rng_stream);
}

int tfgk_block_sample_count_labor_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                              const int32_t *nodes, const int32_t *state, int32_t hop, int32_t n_hops,
                                              int32_t cap_list, int32_t k, uint64_t seed, uint32_t rng_stream,
                                              const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                              int64_t *out_rowptr, void *workspace, size_t workspace_bytes,
                                              void *stream) {
    TFGK_CHECK_ARG(col != nullptr && excl_off != nullptr, "block_sample_count_labor_mapped_excl: null columns or "
                   "exclusion offsets");
    return block_sample_count<int64_t>("block_sample_count_labor_mapped_excl", rowptr, n_rows, nodes, state, hop,
                                       n_hops, cap_list, k, 0, excl_off, n_excl, out_rowptr, workspace, workspace_bytes,
                                       stream, nullptr, nullptr, excl_pos, col, seed, rng_stream);
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

}  // extern "C"

// tfgk_block_sample_fill, _fill_mapped and their _excl twins (excl_off null: no exclusions): K13's fill at positions of
// type TPos, then the frontier
template <typename TPos>
static int block_sample_fill(const char *fn, const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                             const float *w_csr, int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                             int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, int padding, uint64_t seed,
                             uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                             int32_t *out_gcol, float *out_w, const int64_t *excl_off, const TPos *excl_pos,
                             int32_t n_excl, void *workspace, size_t workspace_bytes, void *stream,
                             const int32_t *pos_deg = nullptr, bool labor = false) {
    constexpr bool kMapped = sizeof(TPos) == 8;
    int rc = check_sample_mode(fn, k, -1.0, padding);
    if (rc != TFGK_OK) return rc;
    TFGK_CHECK_ARG(!pos_deg || (k >= 0 && padding != TFGK_SAMPLE_HEAD),
                   "%s: the weighted rule takes an integer fan-out and no head rule", fn);
    TFGK_CHECK_ARG(!labor || (k >= 0 && padding == 0), "%s: the LABOR rule takes an integer fan-out and no padding", fn);
    TFGK_CHECK_ARG(n_rows >= 0 && N >= 0 && hop >= 0 && hop < n_hops && cap_list >= 0 && cap_edges >= 0 &&
                   cap_edges < (1ll << 31) - 1 && n_excl >= 0, "%s: bad size", fn);
    TFGK_CHECK_ARG(state && out_rowptr, "%s: null pointer", fn);
    if ((rc = block_workspace_check(fn, cap_list, cap_edges, workspace, workspace_bytes, sizeof(TPos))) != TFGK_OK)
        return rc;
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    const BlockWorkspace L(cap_list, cap_edges, sizeof(TPos));
    TPos *pos = reinterpret_cast<TPos *>(ws + L.off_pos);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int32_t *off = reinterpret_cast<int32_t *>(ws + L.off_off);
    const int32_t *n_list = state + kStateSizes + hop;
    const int64_t *S = out_rowptr + cap_list;               // listed rows past the count add no edges
    if (cap_list > 0 && cap_edges > 0) {
        TFGK_CHECK_ARG(rowptr && col && (w_csr || (kMapped && !pos_deg)) && nodes && map && out_row && out_local &&
                       out_gcol && out_w,
                       "%s: null pointer", fn);
        const unsigned grid = (unsigned)ceil_div64(cap_list, kRowsPerCta);
        if (labor) {
            const unsigned lgrid = (unsigned)ceil_div64(cap_list, kWeightedRowsPerCta);
            if (excl_off)
                labor_kernel<true, TPos, true><<<lgrid, kRowsPerCta, 0, st>>>(
                    rowptr, n_rows, nodes, n_list, cap_list, k, seed, rng_stream, col, w_csr, nullptr, out_rowptr,
                    out_row, out_gcol, out_w, excl_off, excl_pos, n_excl);
            else
                labor_kernel<true, TPos, false><<<lgrid, kRowsPerCta, 0, st>>>(
                    rowptr, n_rows, nodes, n_list, cap_list, k, seed, rng_stream, col, w_csr, nullptr, out_rowptr,
                    out_row, out_gcol, out_w, nullptr, nullptr, 0);
        } else if (pos_deg) {
            const unsigned wgrid = (unsigned)ceil_div64(cap_list, kWeightedRowsPerCta);
            if (excl_off)
                weighted_fill_kernel<true, TPos, true><<<wgrid, kRowsPerCta, 0, st>>>(
                    rowptr, n_rows, nodes, n_list, 0, k, padding, pos_deg, w_csr, seed, rng_stream, out_rowptr, out_row,
                    pos, col, out_gcol, out_w, excl_off, excl_pos, n_excl);
            else
                weighted_fill_kernel<true, TPos, false><<<wgrid, kRowsPerCta, 0, st>>>(
                    rowptr, n_rows, nodes, n_list, 0, k, padding, pos_deg, w_csr, seed, rng_stream, out_rowptr, out_row,
                    pos, col, out_gcol, out_w, nullptr, nullptr, 0);
        } else if constexpr (kMapped) {
            if (excl_off)
                block_fill_mapped_excl_kernel<<<grid, kRowsPerCta, 0, st>>>(rowptr, n_rows, nodes, n_list, k, padding,
                                                                           seed, rng_stream, out_rowptr, out_row, pos,
                                                                           col, w_csr, out_gcol, out_w, excl_off,
                                                                           excl_pos, n_excl);
            else
                block_fill_mapped_kernel<<<grid, kRowsPerCta, 0, st>>>(rowptr, n_rows, nodes, n_list, k, padding, seed,
                                                                      rng_stream, out_rowptr, out_row, pos, col, w_csr,
                                                                      out_gcol, out_w);
        } else {
            if (excl_off)
                block_fill_excl_kernel<<<grid, kRowsPerCta, 0, st>>>(rowptr, n_rows, nodes, n_list, k, padding, seed,
                                                                    rng_stream, out_rowptr, out_row, pos, col, w_csr,
                                                                    out_gcol, out_w, excl_off, excl_pos, n_excl);
            else
                block_fill_kernel<<<grid, kRowsPerCta, 0, st>>>(rowptr, n_rows, nodes, n_list, k, padding, seed,
                                                               rng_stream, out_rowptr, out_row, pos, col, w_csr, out_gcol,
                                                               out_w);
        }
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

extern "C" {

int tfgk_block_sample_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr, int32_t N,
                           int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                           int64_t cap_edges, int32_t k, int padding, uint64_t seed, uint32_t rng_stream,
                           const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local, int32_t *out_gcol,
                           float *out_w, void *workspace, size_t workspace_bytes, void *stream) {
    return block_sample_fill<int32_t>("block_sample_fill", rowptr, n_rows, col, w_csr, N, nodes, map, state, hop, n_hops,
                                      cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr, out_row, out_local,
                                      out_gcol, out_w, nullptr, nullptr, 0, workspace, workspace_bytes, stream);
}

int tfgk_block_sample_fill_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                int32_t cap_list, int64_t cap_edges, int32_t k, int padding, uint64_t seed,
                                uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                int32_t *out_gcol, float *out_w, const int64_t *excl_off, const int32_t *excl_pos,
                                int32_t n_excl, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr && excl_pos != nullptr, "block_sample_fill_excl: null exclusion lists");
    return block_sample_fill<int32_t>("block_sample_fill_excl", rowptr, n_rows, col, w_csr, N, nodes, map, state, hop,
                                      n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, excl_off, excl_pos, n_excl, workspace, workspace_bytes,
                                      stream);
}

int tfgk_block_sample_fill_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                  int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                  int32_t cap_list, int64_t cap_edges, int32_t k, int padding, uint64_t seed,
                                  uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                  int32_t *out_gcol, float *out_w, void *workspace, size_t workspace_bytes,
                                  void *stream) {
    return block_sample_fill<int64_t>("block_sample_fill_mapped", rowptr, n_rows, col, w_csr, N, nodes, map, state, hop,
                                      n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, nullptr, nullptr, 0, workspace, workspace_bytes, stream);
}

int tfgk_block_sample_fill_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                       int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                       int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, int padding,
                                       uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                       int32_t *out_local, int32_t *out_gcol, float *out_w, const int64_t *excl_off,
                                       const int64_t *excl_pos, int32_t n_excl, void *workspace, size_t workspace_bytes,
                                       void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr && excl_pos != nullptr, "block_sample_fill_mapped_excl: null exclusion lists");
    return block_sample_fill<int64_t>("block_sample_fill_mapped_excl", rowptr, n_rows, col, w_csr, N, nodes, map, state,
                                      hop, n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, excl_off, excl_pos, n_excl, workspace, workspace_bytes,
                                      stream);
}

int tfgk_block_sample_fill_weighted(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                    const int32_t *pos_deg, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                    int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                    int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                    int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                    void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr, "block_sample_fill_weighted: null positive degrees");
    return block_sample_fill<int32_t>("block_sample_fill_weighted", rowptr, n_rows, col, w_csr, N, nodes, map, state, hop,
                                      n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, nullptr, nullptr, 0, workspace, workspace_bytes, stream,
                                      pos_deg);
}

int tfgk_block_sample_fill_weighted_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                         const int32_t *pos_deg, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                         int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                         int padding, uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                         int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                         const int64_t *excl_off, const int32_t *excl_pos, int32_t n_excl,
                                         void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr && excl_off != nullptr && excl_pos != nullptr,
                   "block_sample_fill_weighted_excl: null positive degrees or exclusion lists");
    return block_sample_fill<int32_t>("block_sample_fill_weighted_excl", rowptr, n_rows, col, w_csr, N, nodes, map,
                                      state, hop, n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr,
                                      out_row, out_local, out_gcol, out_w, excl_off, excl_pos, n_excl, workspace,
                                      workspace_bytes, stream, pos_deg);
}

int tfgk_block_sample_fill_weighted_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                           const float *w_csr, const int32_t *pos_deg, int32_t N, int32_t *nodes,
                                           int32_t *map, int32_t *state, int32_t hop, int32_t n_hops, int32_t cap_list,
                                           int64_t cap_edges, int32_t k, int padding, uint64_t seed, uint32_t rng_stream,
                                           const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                                           int32_t *out_gcol, float *out_w, void *workspace, size_t workspace_bytes,
                                           void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr, "block_sample_fill_weighted_mapped: null positive degrees");
    return block_sample_fill<int64_t>("block_sample_fill_weighted_mapped", rowptr, n_rows, col, w_csr, N, nodes, map,
                                      state, hop, n_hops, cap_list, cap_edges, k, padding, seed, rng_stream, out_rowptr,
                                      out_row, out_local, out_gcol, out_w, nullptr, nullptr, 0, workspace,
                                      workspace_bytes, stream, pos_deg);
}

int tfgk_block_sample_fill_weighted_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                                const float *w_csr, const int32_t *pos_deg, int32_t N, int32_t *nodes,
                                                int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                                int32_t cap_list, int64_t cap_edges, int32_t k, int padding,
                                                uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                                int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                                const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                                void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(pos_deg != nullptr && excl_off != nullptr && excl_pos != nullptr,
                   "block_sample_fill_weighted_mapped_excl: null positive degrees or exclusion lists");
    return block_sample_fill<int64_t>("block_sample_fill_weighted_mapped_excl", rowptr, n_rows, col, w_csr, N, nodes,
                                      map, state, hop, n_hops, cap_list, cap_edges, k, padding, seed, rng_stream,
                                      out_rowptr, out_row, out_local, out_gcol, out_w, excl_off, excl_pos, n_excl,
                                      workspace, workspace_bytes, stream, pos_deg);
}

int tfgk_block_sample_fill_labor(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                 int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop, int32_t n_hops,
                                 int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed, uint32_t rng_stream,
                                 const int64_t *out_rowptr, int32_t *out_row, int32_t *out_local, int32_t *out_gcol,
                                 float *out_w, void *workspace, size_t workspace_bytes, void *stream) {
    return block_sample_fill<int32_t>("block_sample_fill_labor", rowptr, n_rows, col, w_csr, N, nodes, map, state, hop,
                                      n_hops, cap_list, cap_edges, k, 0, seed, rng_stream, out_rowptr, out_row, out_local,
                                      out_gcol, out_w, nullptr, nullptr, 0, workspace, workspace_bytes, stream, nullptr,
                                      true);
}

int tfgk_block_sample_fill_labor_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                      int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                      int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed,
                                      uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                      int32_t *out_local, int32_t *out_gcol, float *out_w, const int64_t *excl_off,
                                      const int32_t *excl_pos, int32_t n_excl, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr && excl_pos != nullptr, "block_sample_fill_labor_excl: null exclusion lists");
    return block_sample_fill<int32_t>("block_sample_fill_labor_excl", rowptr, n_rows, col, w_csr, N, nodes, map, state,
                                      hop, n_hops, cap_list, cap_edges, k, 0, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, excl_off, excl_pos, n_excl, workspace, workspace_bytes,
                                      stream, nullptr, true);
}

int tfgk_block_sample_fill_labor_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const float *w_csr,
                                        int32_t N, int32_t *nodes, int32_t *map, int32_t *state, int32_t hop,
                                        int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k, uint64_t seed,
                                        uint32_t rng_stream, const int64_t *out_rowptr, int32_t *out_row,
                                        int32_t *out_local, int32_t *out_gcol, float *out_w, void *workspace,
                                        size_t workspace_bytes, void *stream) {
    return block_sample_fill<int64_t>("block_sample_fill_labor_mapped", rowptr, n_rows, col, w_csr, N, nodes, map, state,
                                      hop, n_hops, cap_list, cap_edges, k, 0, seed, rng_stream, out_rowptr, out_row,
                                      out_local, out_gcol, out_w, nullptr, nullptr, 0, workspace, workspace_bytes, stream,
                                      nullptr, true);
}

int tfgk_block_sample_fill_labor_mapped_excl(const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                             const float *w_csr, int32_t N, int32_t *nodes, int32_t *map, int32_t *state,
                                             int32_t hop, int32_t n_hops, int32_t cap_list, int64_t cap_edges, int32_t k,
                                             uint64_t seed, uint32_t rng_stream, const int64_t *out_rowptr,
                                             int32_t *out_row, int32_t *out_local, int32_t *out_gcol, float *out_w,
                                             const int64_t *excl_off, const int64_t *excl_pos, int32_t n_excl,
                                             void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr && excl_pos != nullptr, "block_sample_fill_labor_mapped_excl: null exclusion "
                   "lists");
    return block_sample_fill<int64_t>("block_sample_fill_labor_mapped_excl", rowptr, n_rows, col, w_csr, N, nodes, map,
                                      state, hop, n_hops, cap_list, cap_edges, k, 0, seed, rng_stream, out_rowptr,
                                      out_row, out_local, out_gcol, out_w, excl_off, excl_pos, n_excl, workspace,
                                      workspace_bytes, stream, nullptr, true);
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

int tfgk_block_self_loops_i32(const int64_t *rowptr, const int32_t *row, const int32_t *col, int64_t S, int32_t n_dst,
                              int64_t *out_rowptr, int32_t *out_row, int32_t *out_col, void *stream) {
    TFGK_CHECK_ARG(S >= 0 && n_dst >= 0, "block_self_loops: bad size (S=%lld, n_dst=%d)", (long long)S, n_dst);
    if (S + n_dst >= (1ll << 31))
        return set_error(TFGK_ERR_UNSUPPORTED, "block_self_loops: %lld looped edges exceed int32 positions",
                         (long long)(S + n_dst));
    TFGK_CHECK_ARG(rowptr && out_rowptr && (S == 0 || (row && col)) && (S + n_dst == 0 || (out_row && out_col)),
                   "block_self_loops: null pointer");
    block_self_loops_kernel<<<grid_for(S + n_dst + 1), 256, 0, as_stream(stream)>>>(rowptr, row, col, S, n_dst, out_rowptr,
                                                                                     out_row, out_col);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // extern "C"

// tfgk_block_gcn_values_f32 and _excl_f32 (excl_off null: no exclusions)
static int block_gcn_values(const int64_t *rowptr, const int32_t *gcol, const float *w, int64_t S, const int32_t *dst,
                            int32_t n_dst, const int64_t *g_rowptr, const float *g_rowsum, int norm, int loop,
                            float deg_fill, float fill, const int64_t *excl_off, int32_t n_excl, float *out,
                            void *stream) {
    TFGK_CHECK_ARG(S >= 0 && n_dst >= 0 && n_excl >= 0, "block_gcn_values: bad size (S=%lld, n_dst=%d)", (long long)S,
                   n_dst);
    TFGK_CHECK_ARG(norm == TFGK_GCN_NORM_BOTH || norm == TFGK_GCN_NORM_LEFT || norm == TFGK_GCN_NORM_RIGHT,
                   "block_gcn_values: unknown norm %d", norm);
    TFGK_CHECK_ARG(loop == TFGK_GCN_LOOP_NONE || loop == TFGK_GCN_LOOP_NORMED || loop == TFGK_GCN_LOOP_FILL,
                   "block_gcn_values: unknown loop mode %d", loop);
    TFGK_CHECK_ARG(S == 0 || n_dst > 0, "block_gcn_values: %lld edges and no output rows", (long long)S);
    if (S + n_dst >= (1ll << 31))
        return set_error(TFGK_ERR_UNSUPPORTED, "block_gcn_values: %lld looped edges exceed int32 positions",
                         (long long)(S + n_dst));
    const int64_t n = S + (loop != TFGK_GCN_LOOP_NONE ? n_dst : 0);
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && dst && g_rowptr && g_rowsum && out && (S == 0 || gcol), "block_gcn_values: null pointer");
    if (excl_off)
        block_gcn_values_excl_kernel<<<grid_for(n), 256, 0, as_stream(stream)>>>(rowptr, gcol, w, S, dst, n_dst, g_rowptr,
                                                                                  g_rowsum, norm, loop, deg_fill, fill,
                                                                                  excl_off, n_excl, out);
    else
        block_gcn_values_kernel<<<grid_for(n), 256, 0, as_stream(stream)>>>(rowptr, gcol, w, S, dst, n_dst, g_rowptr,
                                                                             g_rowsum, norm, loop, deg_fill, fill, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

extern "C" {

int tfgk_block_gcn_values_f32(const int64_t *rowptr, const int32_t *gcol, const float *w, int64_t S, const int32_t *dst,
                              int32_t n_dst, const int64_t *g_rowptr, const float *g_rowsum, int norm, int loop,
                              float deg_fill, float fill, float *out, void *stream) {
    return block_gcn_values(rowptr, gcol, w, S, dst, n_dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, nullptr, 0,
                            out, stream);
}

int tfgk_block_gcn_values_excl_f32(const int64_t *rowptr, const int32_t *gcol, const float *w, int64_t S,
                                   const int32_t *dst, int32_t n_dst, const int64_t *g_rowptr, const float *g_rowsum,
                                   int norm, int loop, float deg_fill, float fill, const int64_t *excl_off,
                                   int32_t n_excl, float *out, void *stream) {
    TFGK_CHECK_ARG(excl_off != nullptr || n_dst == 0, "block_gcn_values_excl: null exclusion offsets");
    return block_gcn_values(rowptr, gcol, w, S, dst, n_dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, excl_off,
                            n_excl, out, stream);
}

// ---- link prediction on blocks ----------------------------------------------------------------------------------
int tfgk_block_pairs_workspace_bytes(int32_t n_pairs, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n_pairs >= 0 && n_pairs < (1 << 30) - 1, "block_pairs_workspace_bytes: bad argument");
    const int64_t P = 2 * (int64_t)n_pairs;
    *out_bytes = 3 * align_up((size_t)(P + 1) * 4) + scan_scratch_bytes(P + 1);
    return TFGK_OK;
}

int tfgk_block_sample_begin_pairs(const int32_t *pair_row, const int32_t *pair_col, int32_t n_pairs, int32_t N,
                                  int32_t *nodes, int32_t *map, int32_t *state, int32_t n_hops, int32_t *local,
                                  void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n_pairs >= 0 && n_pairs < (1 << 30) - 1 && N >= 0 && n_hops >= 0, "block_sample_begin_pairs: bad size");
    TFGK_CHECK_ARG(state != nullptr && (n_pairs == 0 || (pair_row && pair_col && nodes && map && local)),
                   "block_sample_begin_pairs: null pointer");
    size_t need = 0;
    tfgk_block_pairs_workspace_bytes(n_pairs, &need);
    if (n_pairs > 0 && (workspace == nullptr || workspace_bytes < need))
        return set_error(TFGK_ERR_WORKSPACE, "block_sample_begin_pairs: workspace too small (%zu < %zu bytes)",
                         workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    TFGK_CUDA(cudaMemsetAsync(state, 0, (size_t)(4 + 2 * n_hops) * 4, st));
    if (n_pairs == 0) return TFGK_OK;
    const int64_t P = 2 * (int64_t)n_pairs;
    char *ws = static_cast<char *>(workspace);
    int32_t *ends = reinterpret_cast<int32_t *>(ws);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + align_up((size_t)(P + 1) * 4));
    int32_t *off = reinterpret_cast<int32_t *>(ws + 2 * align_up((size_t)(P + 1) * 4));
    int32_t *sums = reinterpret_cast<int32_t *>(ws + 3 * align_up((size_t)(P + 1) * 4));
    // the frontier of an empty list: first occurrences (ids outside [0, N) counted in state[0]), flags, scan, emit
    pair_ends_kernel<<<grid_for(P), 256, 0, st>>>(pair_row, pair_col, P, ends);
    TFGK_LAUNCH_CHECK();
    frontier_first_kernel<<<grid_for(P), 256, 0, st>>>(ends, P, N, map, state);
    TFGK_LAUNCH_CHECK();
    frontier_flag_kernel<<<grid_for(P), 256, 0, st>>>(ends, P, N, map, flag);
    TFGK_LAUNCH_CHECK();
    int rc = exclusive_scan<int32_t, int32_t>(flag, P, P + 1, off, sums, st);
    if (rc != TFGK_OK) return rc;
    frontier_emit_kernel<<<grid_for(P), 256, 0, st>>>(ends, P, flag, off, 0, nodes, map);
    TFGK_LAUNCH_CHECK();
    pair_gather_kernel<<<grid_for(P), 256, 0, st>>>(ends, P, N, map, local);
    TFGK_LAUNCH_CHECK();
    TFGK_CUDA(cudaMemcpyAsync(state + kStateSizes, off + P, 4, cudaMemcpyDeviceToDevice, st));
    return TFGK_OK;
}

int tfgk_link_tail_negatives_i32(const int32_t *src, int32_t n_src, int32_t q, int32_t N, uint64_t seed,
                                 uint32_t rng_stream, int32_t *out_row, int32_t *out_col, void *stream) {
    TFGK_CHECK_ARG(n_src >= 0 && q >= 0 && (int64_t)n_src * q < (1ll << 31) - 1, "link_tail_negatives: bad size");
    const int64_t n = (int64_t)n_src * q;
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(N > 0, "link_tail_negatives: no nodes to draw from");
    TFGK_CHECK_ARG(src && out_row && out_col, "link_tail_negatives: null pointer");
    tail_negatives_kernel<<<grid_for(n), 256, 0, as_stream(stream)>>>(src, n, q, (uint32_t)N, seed, rng_stream, out_row,
                                                                       out_col);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

namespace {
struct ExclWorkspace {
    size_t off_tend, off_cnt, off_sums, total;
    explicit ExclWorkspace(int32_t cap) {
        const size_t row = align_up(((size_t)cap + 1) * 4);
        off_tend = row;
        off_cnt = 2 * row;
        off_sums = 3 * row;
        total = off_sums + scan_scratch_bytes((int64_t)cap + 1);
    }
};
}  // namespace

int tfgk_block_exclusion_workspace_bytes(int32_t cap, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && cap >= 0, "block_exclusion_workspace_bytes: bad argument");
    *out_bytes = ExclWorkspace(cap).total;
    return TFGK_OK;
}

int tfgk_block_exclusion_count(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                               int32_t cap, const int32_t *target_src, const int32_t *target_dst, int64_t n_targets,
                               int64_t *excl_off, int64_t *total_host, void *workspace, size_t workspace_bytes,
                               void *stream) {
    TFGK_CHECK_ARG(n_rows >= 0 && cap >= 0 && n_targets >= 0 && n_targets < (1ll << 31) - 1,
                   "block_exclusion_count: bad size");
    TFGK_CHECK_ARG(total_host != nullptr && excl_off != nullptr, "block_exclusion_count: null pointer");
    *total_host = 0;
    cudaStream_t st = as_stream(stream);
    if (cap == 0) {
        TFGK_CUDA(cudaMemsetAsync(excl_off, 0, 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(rowptr && col && nodes && (n_targets == 0 || (target_src && target_dst)),
                   "block_exclusion_count: null pointer");
    const ExclWorkspace L(cap);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "block_exclusion_count: workspace too small (%zu < %zu bytes)",
                         workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    int32_t *tbeg = reinterpret_cast<int32_t *>(ws);
    int32_t *tend = reinterpret_cast<int32_t *>(ws + L.off_tend);
    int32_t *cnt = reinterpret_cast<int32_t *>(ws + L.off_cnt);
    TFGK_CUDA(cudaMemsetAsync(ws, 0, L.off_cnt, st));            // tbeg = tend = 0: no targets
    if (n_targets) {
        excl_mark_kernel<<<grid_for(n_targets), 256, 0, st>>>(target_src, n_targets, cap, tbeg, tend);
        TFGK_LAUNCH_CHECK();
    }
    excl_scan_kernel<false, int32_t><<<(unsigned)ceil_div64((int64_t)cap * 32, 256), 256, 0, st>>>(
        rowptr, n_rows, col, nodes, cap, target_dst, tbeg, tend, cnt, nullptr, nullptr);
    TFGK_LAUNCH_CHECK();
    int rc = exclusive_scan<int32_t, int64_t>(cnt, cap, (int64_t)cap + 1, excl_off,
                                              reinterpret_cast<int64_t *>(ws + L.off_sums), st);
    if (rc != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(total_host, excl_off + cap, 8, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

}  // extern "C"

template <typename TPos>
static int block_exclusion_fill(const char *fn, const int64_t *rowptr, int32_t n_rows, const int32_t *col,
                                const int32_t *nodes, int32_t cap, const int32_t *target_dst, const int64_t *excl_off,
                                TPos *excl_pos, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n_rows >= 0 && cap >= 0, "%s: bad size", fn);
    if (cap == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && col && nodes && excl_off, "%s: null pointer", fn);
    const ExclWorkspace L(cap);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "%s: workspace too small (%zu < %zu bytes)", fn, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    excl_scan_kernel<true, TPos><<<(unsigned)ceil_div64((int64_t)cap * 32, 256), 256, 0, as_stream(stream)>>>(
        rowptr, n_rows, col, nodes, cap, target_dst, reinterpret_cast<const int32_t *>(ws),
        reinterpret_cast<const int32_t *>(ws + L.off_tend), nullptr, excl_off, excl_pos);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

extern "C" {

int tfgk_block_exclusion_fill(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                              int32_t cap, const int32_t *target_dst, const int64_t *excl_off, int32_t *excl_pos,
                              void *workspace, size_t workspace_bytes, void *stream) {
    return block_exclusion_fill<int32_t>("block_exclusion_fill", rowptr, n_rows, col, nodes, cap, target_dst, excl_off,
                                         excl_pos, workspace, workspace_bytes, stream);
}

int tfgk_block_exclusion_fill_mapped(const int64_t *rowptr, int32_t n_rows, const int32_t *col, const int32_t *nodes,
                                     int32_t cap, const int32_t *target_dst, const int64_t *excl_off, int64_t *excl_pos,
                                     void *workspace, size_t workspace_bytes, void *stream) {
    return block_exclusion_fill<int64_t>("block_exclusion_fill_mapped", rowptr, n_rows, col, nodes, cap, target_dst,
                                         excl_off, excl_pos, workspace, workspace_bytes, stream);
}

}  // extern "C"

// ---- row blocks: every in-neighbour of a range of rows (layer-wise inference) --------------------------------------
namespace tfgk {
namespace {

// items [0, n): output row i is node r0 + i, at position i of the list and of the map, with its rebased rowptr; item n:
// the closing rowptr; items n + 1 + e: edge e's output row, the last row i with rowptr[r0 + i] <= rowptr[r0] + e (a
// binary search, so that no thread walks a row and a hub's edges spread over as many threads as it has edges)
__global__ void row_block_begin_kernel(const int64_t *__restrict__ rowptr, int32_t r0, int32_t n, int64_t S,
                                       int32_t *__restrict__ nodes, int32_t *__restrict__ map,
                                       int64_t *__restrict__ out_rowptr, int32_t *__restrict__ out_row) {
    const int64_t *__restrict__ rp = rowptr + r0;
    const int64_t e0 = rp[0];
    const int64_t total = (int64_t)n + 1 + S;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        if (t <= n) {
            out_rowptr[t] = rp[t] - e0;
            if (t < n) {
                nodes[t] = r0 + (int32_t)t;
                map[r0 + t] = (int32_t)t;
            }
        } else {
            const int64_t p = e0 + (t - n - 1);
            int32_t lo = 0, hi = n - 1;
            while (lo < hi) {
                const int32_t mid = lo + (hi - lo + 1) / 2;
                if (rp[mid] <= p) lo = mid;
                else hi = mid - 1;
            }
            out_row[t - n - 1] = lo;
        }
    }
}

}  // namespace
}  // namespace tfgk

extern "C" {

int tfgk_row_block_i32(const int64_t *rowptr, int32_t N, int32_t r0, int32_t r1, const int32_t *cols, int64_t S,
                       int32_t *nodes, int32_t *map, int64_t *out_rowptr, int32_t *out_row, int32_t *out_local,
                       int32_t *num_src_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(N >= 0 && r0 >= 0 && r0 <= r1 && r1 <= N, "row_block: bad range [%d, %d) of %d rows", r0, r1, N);
    TFGK_CHECK_ARG(S >= 0 && S < (1ll << 31) - 1, "row_block: %lld edges; a row block takes fewer than 2^31 - 1",
                   (long long)S);
    TFGK_CHECK_ARG(S == 0 || r0 < r1, "row_block: %lld edges and no rows", (long long)S);
    TFGK_CHECK_ARG(num_src_host != nullptr && rowptr != nullptr && out_rowptr != nullptr, "row_block: null pointer");
    const int32_t n = r1 - r0;
    *num_src_host = n;
    TFGK_CHECK_ARG(n == 0 || (nodes && map), "row_block: null node list or map");
    TFGK_CHECK_ARG(S == 0 || (cols && out_row && out_local), "row_block: null edge array");
    size_t need = 0;
    int rc = tfgk_relabel_workspace_bytes(S, &need);
    if (rc != TFGK_OK) return rc;
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "row_block: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int32_t *counters = reinterpret_cast<int32_t *>(ws + need - 256);
    row_block_begin_kernel<<<grid_for((int64_t)n + 1 + S), 256, 0, st>>>(rowptr, r0, n, S, nodes, map, out_rowptr,
                                                                        out_row);
    TFGK_LAUNCH_CHECK();
    if (S == 0) {                       // no columns: the list is the range, and nothing is read back
        if (n) {
            node_reset_kernel<<<grid_for(n), 256, 0, st>>>(nodes, n, nullptr, N, map);
            TFGK_LAUNCH_CHECK();
        }
        return TFGK_OK;
    }
    // the frontier's relabelling after the range's rows: columns outside the list appended in first-occurrence order
    TFGK_CUDA(cudaMemsetAsync(counters, 0, 3 * 4, st));
    int32_t c[3];
    if ((rc = frontier_relabel(cols, S, N, nodes, n, map, out_local, ws, need, c, st)) != TFGK_OK) return rc;
    if (c[kBadIds]) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "row_block: %d column ids outside [0, %d)", c[kBadIds], N);
    *num_src_host = n + c[kNewIds];
    return TFGK_OK;
}

int tfgk_copy_async(void *dst, const void *src, size_t bytes, void *stream) {
    if (bytes == 0) return TFGK_OK;
    TFGK_CHECK_ARG(dst != nullptr && src != nullptr, "copy_async: null pointer");
    TFGK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, as_stream(stream)));
    return TFGK_OK;
}

}  // extern "C"
