// K11: max aggregation that can be trained without per-edge messages (tfgk_spmm_max_f32, tfgk_spmm_max_bwd_f32).
//
//   K11a  out[r,d] = max_{e in row r} w_e h[col_e,d]          (fmaxf in CSR order from -FLT_MAX, products __fmul_rn)
//         cnt[r,d] = #{e in row r : w_e h[col_e,d] == out[r,d]}   (IEEE ==: +0 == -0, NaN never, -inf != -FLT_MAX)
//   K11b  dh[c,d]  = sum_{e: c -> r} ((Gn[r,d] * sel_e) * w_e),   sel_e = (w_e h[c,d] == out[r,d]),
//         Gn = g / max(cnt, 1)
//
// K11a is K1's MAX with a tie counter next to every accumulator: the running maximum is the same fmaxf chain, and the
// count restarts at 1 when a product exceeds it and grows by 1 when a product equals it, so at every step it counts the
// products equal to the running maximum.  K11b walks the transposed CSR (one row per source c, its out-edges in stable
// edge order), loads h[c] once and gathers out[r] and Gn[r] per edge from one [N, 2D] table that a first elementwise pass
// writes.  Every edge adds its term, selected or not (0 * inf = NaN reaches the neighbours of a row with an inf upstream
// entry, as the product of the gradient with the 0/1 selection does); sums start at 0 and run in edge order, with
// separate roundings.  No atomics anywhere; every output row is written once.
//
// Both take the work plan of their CSR exactly where tfgk_spmm_f32 takes it: K11a for the same h and out, K11b for a
// dense [E, D] table (the per-edge gradient the composition TakeRows + SegmentReduce sums).  A hub slice reduces its part
// of the row into the plan's scratch and a fix-up merges the slices in order: (max, count) pairs for K11a, sums from 0
// for K11b.  The results are therefore bit-identical to K1 MAX and to that composition.
//
// Mapping (both kernels): a group of G lanes owns one row and each lane NC vectors of VEC consecutive columns; the edge
// ids (and weights) are read G at a time, coalesced, and broadcast by shuffles within the group; U gathers are in flight
// before any is consumed.  A warp owns 32 / G rows, or one task of the plan (its groups take the task's rows in turn).
//
// Algorithmic bytes (unweighted; +4 per edge with weights):
//   K11a  E*(4*D + 4) + N*(8*D + 8)          K11b  E*(8*D + 4) + N*(8*D + 8)   (+ the pass writing [out | Gn]: 20*D*N)
#include "common.cuh"

namespace tfgk {
namespace {

constexpr int kMaxThreads = 256;

struct MaxParams {
    const int64_t *rowptr;
    const int32_t *col;        // K11a: source of every CSR edge; K11b: destination row of every transposed edge
    const float *w;            // weights in the same order, or nullptr (= 1)
    const float *h;            // [rows of col / sources, ldh]
    int64_t ldh;
    const float *pk;           // K11b: [n_dst, 2 * D_full] = [out | Gn]
    int64_t ldpk;
    int32_t gn_off;            // K11b: column of Gn within a pk row (D_full)
    int32_t n_rows;
    int32_t D;                 // columns of this launch
    float *out;                // K11a: out;  K11b: dh
    int64_t ldo;
    int32_t *cnt;              // K11a only
    int64_t ldc;
    // optional work plan; task_row == nullptr -> implicit tasks of 32 / G consecutive rows per warp
    int32_t n_tasks;
    const int32_t *task_row, *task_nrows;
    const int64_t *task_e0, *task_e1;
    const int32_t *task_slot;
    int32_t n_hubs;
    const int32_t *hub_row, *hub_slot0, *hub_nslots;
    float *scratch;            // K11a: n_slots * D maxima, then n_slots * D counts (int32); K11b: n_slots * D sums
    int32_t n_slots;
};

template <int VEC>
__device__ __forceinline__ void ld_vec(const float *p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        v[0] = __ldg(p);
    }
}

template <int VEC>
__device__ __forceinline__ void st_vec(float *p, const float (&v)[VEC]) {
    if constexpr (VEC == 4) *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else p[0] = v[0];
}

template <int VEC>
__device__ __forceinline__ void st_vec(int32_t *p, const int (&v)[VEC]) {
    if constexpr (VEC == 4) *reinterpret_cast<int4 *>(p) = make_int4(v[0], v[1], v[2], v[3]);
    else p[0] = v[0];
}

// The rows of the warp's task: [r0, r1) with edges clipped to [e0, e1) (a hub slice: one row, part of its edges) and the
// scratch slot of a hub slice (-1 for whole rows).  False when the warp has no task.
template <int G>
__device__ __forceinline__ bool warp_task(const MaxParams &p, int64_t &r0, int64_t &r1, int64_t &e0, int64_t &e1,
                                          int &slot) {
    const int64_t warp = (int64_t)blockIdx.x * (kMaxThreads / 32) + (threadIdx.x >> 5);
    if (p.task_row != nullptr) {
        if (warp >= p.n_tasks) return false;
        r0 = p.task_row[warp];
        r1 = r0 + p.task_nrows[warp];
        e0 = p.task_e0[warp];
        e1 = p.task_e1[warp];
        slot = p.task_slot[warp];
        return true;
    }
    r0 = warp * (32 / G);
    if (r0 >= p.n_rows) return false;
    r1 = min((int64_t)p.n_rows, r0 + 32 / G);
    e0 = 0;
    e1 = INT64_MAX;
    slot = -1;
    return true;
}

// K11a.  G lanes per row (power of two), NC vectors of VEC columns per lane, U gathered rows in flight.
template <int VEC, int G, int NC, int U>
__global__ void __launch_bounds__(kMaxThreads) max_fwd_kernel(const MaxParams p) {
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int grp = lane / G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    int64_t r0, r1, t0, t1;
    int slot;
    if (!warp_task<G>(p, r0, r1, t0, t1, slot)) return;

    int coff[NC];
    bool cok[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        coff[k] = (gl + k * G) * VEC;
        cok[k] = coff[k] < p.D;
    }
    const bool weighted = p.w != nullptr;

    for (int64_t r = r0 + grp; r < r1; r += 32 / G) {
        const int64_t s = max(p.rowptr[r], t0);
        const int64_t t = min(p.rowptr[r + 1], t1);
        float acc[NC][VEC];
        int cn[NC][VEC];
#pragma unroll
        for (int k = 0; k < NC; ++k)
#pragma unroll
            for (int x = 0; x < VEC; ++x) { acc[k][x] = -FLT_MAX; cn[k][x] = 0; }

        for (int64_t b = s; b < t; b += G) {
            const int64_t e = b + gl;
            int my_c = 0;
            float my_w = 1.0f;
            if (e < t) {
                my_c = ld_stream_i32(p.col + e);
                if (weighted) my_w = ld_stream_f32(p.w + e);
            }
            const int nb = (int)min((int64_t)G, t - b);
            for (int j = 0; j < nb; j += U) {
                float v[U][NC][VEC];
                float ww[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int c = __shfl_sync(gmask, my_c, j + u, G);
                    ww[u] = __shfl_sync(gmask, my_w, j + u, G);
                    if (j + u < nb) {
                        const float *rowp = p.h + (int64_t)c * p.ldh;
#pragma unroll
                        for (int k = 0; k < NC; ++k)
                            if (cok[k]) ld_vec<VEC>(rowp + coff[k], v[u][k]);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (j + u < nb) {
#pragma unroll
                        for (int k = 0; k < NC; ++k) {
                            if (cok[k]) {
#pragma unroll
                                for (int x = 0; x < VEC; ++x) {
                                    const float m = __fmul_rn(v[u][k][x], ww[u]);
                                    const float a = acc[k][x];
                                    cn[k][x] = m > a ? 1 : (m == a ? cn[k][x] + 1 : cn[k][x]);
                                    acc[k][x] = fmaxf(a, m);
                                }
                            }
                        }
                    }
                }
            }
        }

        float *dst = slot >= 0 ? p.scratch + (int64_t)slot * p.D : p.out + r * p.ldo;
        int32_t *dstc = slot >= 0 ? reinterpret_cast<int32_t *>(p.scratch) + (int64_t)p.n_slots * p.D + (int64_t)slot * p.D
                                  : p.cnt + r * p.ldc;
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            if (!cok[k]) continue;
            if (slot >= 0) {
#pragma unroll
                for (int x = 0; x < VEC; ++x) {         // scratch rows are D wide: no alignment promise for VEC == 4
                    dst[coff[k] + x] = acc[k][x];
                    dstc[coff[k] + x] = cn[k][x];
                }
            } else {
                st_vec<VEC>(dst + coff[k], acc[k]);
                st_vec<VEC>(dstc + coff[k], cn[k]);
            }
        }
    }
}

// K11a hub fix-up: one warp per hub row merges its slices' (max, count) pairs in slice order.
__global__ void __launch_bounds__(256) max_fwd_fixup_kernel(const MaxParams p) {
    const int lane = threadIdx.x & 31;
    const int hb = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (hb >= p.n_hubs) return;
    const int64_t r = p.hub_row[hb];
    const int s0 = p.hub_slot0[hb], ns = p.hub_nslots[hb];
    const int32_t *cs = reinterpret_cast<const int32_t *>(p.scratch) + (int64_t)p.n_slots * p.D;
    for (int c = lane; c < p.D; c += 32) {
        float a = -FLT_MAX;
        int n = 0;
        for (int s = 0; s < ns; ++s) {
            const float m = p.scratch[(int64_t)(s0 + s) * p.D + c];
            const int k = cs[(int64_t)(s0 + s) * p.D + c];
            n = m > a ? k : (m == a ? n + k : n);
            a = fmaxf(a, m);
        }
        p.out[r * p.ldo + c] = a;
        p.cnt[r * p.ldc + c] = n;
    }
}

// pk[r] = [out[r] | g[r] / max(cnt[r], 1)] (fp32 division, correctly rounded), all D_full columns.
__global__ void max_bwd_pack_kernel(const float *out, int64_t ldo, const int32_t *cnt, int64_t ldc, const float *g,
                                    int64_t ldg, float *pk, int32_t n, int32_t D) {
    const int64_t total = (int64_t)n * D;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / D;
        const int c = (int)(i - r * D);
        pk[r * 2 * D + c] = out[r * ldo + c];
        pk[r * 2 * D + D + c] = __fdiv_rn(g[r * ldg + c], (float)max(cnt[r * ldc + c], 1));
    }
}

// K11b over the transposed CSR: rows are sources, p.col their destination rows.
template <int VEC, int G, int NC, int U>
__global__ void __launch_bounds__(kMaxThreads) max_bwd_kernel(const MaxParams p) {
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int grp = lane / G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    int64_t r0, r1, t0, t1;
    int slot;
    if (!warp_task<G>(p, r0, r1, t0, t1, slot)) return;

    int coff[NC];
    bool cok[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        coff[k] = (gl + k * G) * VEC;
        cok[k] = coff[k] < p.D;
    }
    const bool weighted = p.w != nullptr;

    for (int64_t c = r0 + grp; c < r1; c += 32 / G) {
        const int64_t s = max(p.rowptr[c], t0);
        const int64_t t = min(p.rowptr[c + 1], t1);
        float hv[NC][VEC], acc[NC][VEC];
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            if (cok[k] && s < t) ld_vec<VEC>(p.h + c * p.ldh + coff[k], hv[k]);
#pragma unroll
            for (int x = 0; x < VEC; ++x) acc[k][x] = 0.0f;
        }

        for (int64_t b = s; b < t; b += G) {
            const int64_t e = b + gl;
            int my_r = 0;
            float my_w = 1.0f;
            if (e < t) {
                my_r = ld_stream_i32(p.col + e);
                if (weighted) my_w = ld_stream_f32(p.w + e);
            }
            const int nb = (int)min((int64_t)G, t - b);
            for (int j = 0; j < nb; j += U) {
                float o[U][NC][VEC], gn[U][NC][VEC];
                float ww[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const int r = __shfl_sync(gmask, my_r, j + u, G);
                    ww[u] = __shfl_sync(gmask, my_w, j + u, G);
                    if (j + u < nb) {
                        const float *rowp = p.pk + (int64_t)r * p.ldpk;
#pragma unroll
                        for (int k = 0; k < NC; ++k) {
                            if (cok[k]) {
                                ld_vec<VEC>(rowp + coff[k], o[u][k]);
                                ld_vec<VEC>(rowp + p.gn_off + coff[k], gn[u][k]);
                            }
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (j + u < nb) {
#pragma unroll
                        for (int k = 0; k < NC; ++k) {
                            if (cok[k]) {
#pragma unroll
                                for (int x = 0; x < VEC; ++x) {
                                    const float m = __fmul_rn(hv[k][x], ww[u]);
                                    const float sel = m == o[u][k][x] ? 1.0f : 0.0f;
                                    acc[k][x] = __fadd_rn(acc[k][x], __fmul_rn(__fmul_rn(gn[u][k][x], sel), ww[u]));
                                }
                            }
                        }
                    }
                }
            }
        }

        float *dst = slot >= 0 ? p.scratch + (int64_t)slot * p.D : p.out + c * p.ldo;
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            if (!cok[k]) continue;
            if (slot >= 0) {
#pragma unroll
                for (int x = 0; x < VEC; ++x) dst[coff[k] + x] = acc[k][x];
            } else {
                st_vec<VEC>(dst + coff[k], acc[k]);
            }
        }
    }
}

// K11b hub fix-up: the slices' partial sums added from 0 in slice order (K1's SUM fix-up).
__global__ void __launch_bounds__(256) max_bwd_fixup_kernel(const MaxParams p) {
    const int lane = threadIdx.x & 31;
    const int hb = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (hb >= p.n_hubs) return;
    const int64_t r = p.hub_row[hb];
    const int s0 = p.hub_slot0[hb], ns = p.hub_nslots[hb];
    for (int c = lane; c < p.D; c += 32) {
        float a = 0.0f;
        for (int s = 0; s < ns; ++s) a = __fadd_rn(a, p.scratch[(int64_t)(s0 + s) * p.D + c]);
        p.out[r * p.ldo + c] = a;
    }
}

template <bool BWD, int VEC, int G, int NC, int U>
int launch_max(const MaxParams &p, cudaStream_t st) {
    const int64_t warps = p.task_row ? p.n_tasks : ceil_div64(p.n_rows, 32 / G);
    const unsigned blocks = (unsigned)ceil_div64(warps, kMaxThreads / 32);
    if (blocks == 0) return TFGK_OK;
    if constexpr (BWD) max_bwd_kernel<VEC, G, NC, U><<<blocks, kMaxThreads, 0, st>>>(p);
    else max_fwd_kernel<VEC, G, NC, U><<<blocks, kMaxThreads, 0, st>>>(p);
    TFGK_LAUNCH_CHECK();
    if (p.task_row && p.n_hubs > 0) {
        const unsigned fb = (unsigned)ceil_div64(p.n_hubs, 8);
        if constexpr (BWD) max_bwd_fixup_kernel<<<fb, 256, 0, st>>>(p);
        else max_fwd_fixup_kernel<<<fb, 256, 0, st>>>(p);
        TFGK_LAUNCH_CHECK();
    }
    return TFGK_OK;
}

// lanes = VEC-wide vectors in this launch's columns (<= 128); the backward holds twice the gathered data per edge
template <bool BWD, int VEC>
int dispatch_max(const MaxParams &p, cudaStream_t st) {
    const int lanes = (p.D + VEC - 1) / VEC;
    if (lanes <= 1) return launch_max<BWD, VEC, 1, 1, 8>(p, st);
    if (lanes <= 2) return launch_max<BWD, VEC, 2, 1, 8>(p, st);
    if (lanes <= 4) return launch_max<BWD, VEC, 4, 1, 8>(p, st);
    if (lanes <= 8) return launch_max<BWD, VEC, 8, 1, 8>(p, st);
    if (lanes <= 16) return launch_max<BWD, VEC, 16, 1, 8>(p, st);
    if (lanes <= 32) return launch_max<BWD, VEC, 32, 1, BWD ? 4 : 8>(p, st);
    if (lanes <= 64) return launch_max<BWD, VEC, 32, 2, BWD ? 2 : 4>(p, st);
    if (lanes <= 96) return launch_max<BWD, VEC, 32, 3, 2>(p, st);
    return launch_max<BWD, VEC, 32, 4, BWD ? 1 : 2>(p, st);
}

MaxParams max_params(const int64_t *rowptr, const int32_t *col, const float *w, const float *h, int64_t ldh, int32_t n,
                     float *out, int64_t ldo) {
    MaxParams p;
    p.rowptr = rowptr; p.col = col; p.w = w; p.h = h; p.ldh = ldh;
    p.pk = nullptr; p.ldpk = 0; p.gn_off = 0;
    p.n_rows = n; p.D = 0; p.out = out; p.ldo = ldo; p.cnt = nullptr; p.ldc = 0;
    p.n_tasks = 0; p.task_row = nullptr; p.task_nrows = nullptr; p.task_e0 = nullptr; p.task_e1 = nullptr;
    p.task_slot = nullptr; p.n_hubs = 0; p.hub_row = nullptr; p.hub_slot0 = nullptr; p.hub_nslots = nullptr;
    p.scratch = nullptr; p.n_slots = 0;
    return p;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" int tfgk_spmm_max_f32(const int64_t *rowptr, const int32_t *col, const float *w, const float *h, int64_t ldh,
                                 int32_t n_dst, int32_t D, float *out, int64_t ldo, int32_t *cnt, int64_t ldc,
                                 const tfgk_plan *plan, void *stream) {
    TFGK_CHECK_ARG(n_dst >= 0 && D >= 0, "spmm_max: negative size (n_dst=%d, D=%d)", n_dst, D);
    if (n_dst == 0 || D == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && col && h && out && cnt, "spmm_max: null pointer");
    TFGK_CHECK_ARG(ldh >= D && ldo >= D && ldc >= D, "spmm_max: leading dimension < D");
    const bool vec4 = D % 4 == 0 && ldh % 4 == 0 && ldo % 4 == 0 && ldc % 4 == 0 && aligned16(h) && aligned16(out) &&
                      aligned16(cnt);
    // tfgk_spmm_f32's plan condition for the same h and out (one launch of the float4 ring kernels)
    const bool plan_on = plan != nullptr && plan->n_tasks > 0 && vec4 && D >= 32 && D <= 512;
    if (plan_on && plan->n_hubs > 0)
        TFGK_CHECK_ARG(plan->scratch != nullptr && plan->scratch_bytes >= (size_t)plan->n_slots * D * 8,
                       "spmm_max: plan scratch too small (need %zu bytes)", (size_t)plan->n_slots * D * 8);
    const int vec = vec4 ? 4 : 1;
    const int per_launch = 128 * vec;
    cudaStream_t st = as_stream(stream);
    for (int c0 = 0; c0 < D; c0 += per_launch) {
        MaxParams p = max_params(rowptr, col, w, h + c0, ldh, n_dst, out + c0, ldo);
        p.D = D - c0 < per_launch ? D - c0 : per_launch;
        p.cnt = cnt + c0; p.ldc = ldc;
        if (plan_on) {
            use_plan(p, plan);
            p.n_slots = plan->n_slots;
        }
        const int rc = vec4 ? dispatch_max<false, 4>(p, st) : dispatch_max<false, 1>(p, st);
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}

extern "C" int tfgk_spmm_max_bwd_f32(const int64_t *rowptr_t, const int32_t *dst_t, const float *w_t, const float *h,
                                     int64_t ldh, int32_t n_src, int32_t n_dst, int32_t D, const float *out, int64_t ldo,
                                     const int32_t *cnt, int64_t ldc, const float *g, int64_t ldg, float *pk, float *dh,
                                     int64_t lddh, const tfgk_plan *plan, void *stream) {
    TFGK_CHECK_ARG(n_src >= 0 && n_dst >= 0 && D >= 0, "spmm_max_bwd: negative size (n_src=%d, n_dst=%d, D=%d)", n_src,
                   n_dst, D);
    if (n_src == 0 || D == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr_t && dst_t && h && dh && (n_dst == 0 || (out && cnt && g && pk)), "spmm_max_bwd: null pointer");
    TFGK_CHECK_ARG(ldh >= D && lddh >= D && ldo >= D && ldc >= D && ldg >= D, "spmm_max_bwd: leading dimension < D");
    // the per-edge gradient of the composition is a dense [E, D] table: K1 sums it with the plan for 32 <= D <= 512, D % 4 == 0
    const bool plan_on = plan != nullptr && plan->n_tasks > 0 && D % 4 == 0 && D >= 32 && D <= 512;
    if (plan_on && plan->n_hubs > 0)
        TFGK_CHECK_ARG(plan->scratch != nullptr && plan->scratch_bytes >= (size_t)plan->n_slots * D * 4,
                       "spmm_max_bwd: plan scratch too small (need %zu bytes)", (size_t)plan->n_slots * D * 4);
    cudaStream_t st = as_stream(stream);
    if (n_dst > 0) {
        const int64_t total = (int64_t)n_dst * D;
        const unsigned blocks = (unsigned)min(ceil_div64(total, 256), (int64_t)sm_count() * 16);
        max_bwd_pack_kernel<<<blocks, 256, 0, st>>>(out, ldo, cnt, ldc, g, ldg, pk, n_dst, D);
        TFGK_LAUNCH_CHECK();
    }
    const bool vec4 = D % 4 == 0 && ldh % 4 == 0 && lddh % 4 == 0 && aligned16(h) && aligned16(dh) && aligned16(pk);
    const int vec = vec4 ? 4 : 1;
    const int per_launch = 128 * vec;
    for (int c0 = 0; c0 < D; c0 += per_launch) {
        MaxParams p = max_params(rowptr_t, dst_t, w_t, h + c0, ldh, n_src, dh + c0, lddh);
        p.D = D - c0 < per_launch ? D - c0 : per_launch;
        p.pk = pk + c0; p.ldpk = 2 * (int64_t)D; p.gn_off = D;
        if (plan_on) {
            use_plan(p, plan);
            p.n_slots = plan->n_slots;
        }
        const int rc = vec4 ? dispatch_max<true, 4>(p, st) : dispatch_max<true, 1>(p, st);
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}
