// K1: gather - edge-apply - segment-reduce over a destination-sorted CSR  (tfgk_spmm_f32).
//
//   out[r,:] = epilogue( REDUCE_{e in [rowptr[r], rowptr[r+1])} w[e] * h[col[e], :] )
//
// HBM-bound (0.25-0.5 flop/byte): no tensor cores.  Mapping: a group of G lanes owns one destination row and
// each lane owns NC vectors of VEC consecutive feature columns, so one gathered source row is one coalesced
// G*VEC*4-byte request (512 B for D=128).  Edge ids/weights are read once, coalesced, G at a time and broadcast
// with shuffles; U gathered rows are kept in flight per group before any of them is consumed.  Accumulation is
// fp32, strictly in CSR (= input) order with separate multiply and add roundings, which makes SUM/MEAN
// bit-identical to tf.math.unsorted_segment_sum's sequential CPU loop (no atomics anywhere => deterministic).
//
// Algorithmic bytes per launch (DESIGN.md): E*(4*D + 4 [+4 weighted]) + N*(4*D + 8).
#include "common.cuh"
#include <cuda_bf16.h>

namespace tfgk {

template <int VEC> struct Vec;
template <> struct Vec<4> { using T = float4; };
template <> struct Vec<1> { using T = float; };

template <int VEC>
__device__ __forceinline__ void load_vec(const float *p, float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
        v[0] = __ldg(p);
    }
}

// bf16 rows (scalar path only): one widened element
template <int VEC>
__device__ __forceinline__ void load_vec(const uint16_t *p, float (&v)[VEC]) {
    static_assert(VEC == 1, "bf16 rows take the scalar path");
    v[0] = bf16_to_f32(__ldg(p));
}

// fp8 rows (scalar path only): one widened element, scaled by the caller
template <int VEC>
__device__ __forceinline__ void load_vec(const uint8_t *p, float (&v)[VEC]) {
    static_assert(VEC == 1, "fp8 rows take the scalar path");
    v[0] = e4m3_to_f32(__ldg(p));
}

template <int VEC>
__device__ __forceinline__ void store_vec(float *p, const float (&v)[VEC]) {
    if constexpr (VEC == 4) {
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
        p[0] = v[0];
    }
}

struct SpmmParams {
    const int64_t *rowptr;
    const int32_t *col;
    const float *w;
    const float *h;
    const uint16_t *hb;    // bf16 rows (tfgk_spmm_bf16); the kernels instantiated for uint16_t read this one
    // fp8 rows (tfgk_spmm_fp8, the kernels instantiated for uint8_t): e4m3 bytes and the [N, n_grp] int8 exponents; the
    // scalar path covers the columns of group grp0 only
    const uint8_t *h8;
    const int8_t *hexp;
    int32_t n_grp, grp0;
    int64_t ldh;
    int32_t n_dst;
    int32_t D;
    int reduce;
    float alpha;
    const float *addend;
    int64_t ld_addend;
    float beta;
    const float *bias;
    int act;
    float *out;            // may be nullptr in tfgk_spmm_bf16_dual (bf16 output only)
    int64_t ldo;
    // tfgk_spmm_bf16_dual only (the kernels instantiated with DUAL): a bf16 copy of the output, the number of columns
    // stored (D may include pad columns that are computed and never stored) and whether addend / bias / out / outb may
    // be accessed four columns at a time
    uint16_t *outb;
    int64_t ldob;
    int32_t d_store;
    bool io4;
    // optional work plan (tfgk_plan): tasks + hub slices; task_row == nullptr -> implicit blocks of consecutive rows
    int32_t n_tasks;
    const int32_t *task_row, *task_nrows;
    const int64_t *task_e0, *task_e1;
    const int32_t *task_slot;
    int32_t n_hubs;
    const int32_t *hub_row, *hub_slot0, *hub_nslots;
    float *scratch;
    // tfgk_spmm_proj_f32 only (the kernels instantiated with PROJ): out = act(agg . pw + bias), pw [D, pu] row-major
    const float *pw;
    int32_t pu;
    bool pio4;             // bias and out may be accessed four columns at a time
};

// the message rows of a kernel instantiated for element type T (float or bf16 bits)
template <typename T> __device__ __forceinline__ const T *rows_of(const SpmmParams &p);
template <> __device__ __forceinline__ const float *rows_of<float>(const SpmmParams &p) { return p.h; }
template <> __device__ __forceinline__ const uint16_t *rows_of<uint16_t>(const SpmmParams &p) { return p.hb; }
template <> __device__ __forceinline__ const uint8_t *rows_of<uint8_t>(const SpmmParams &p) { return p.h8; }

// The epilogue of tfgk_spmm_bf16_dual for N consecutive columns c .. c+N-1 of row r: the arithmetic of every other
// epilogue in this file (mean, axpby, bias, activation, in that order and rounding), then the value is stored in fp32
// and/or rounded to nearest even into the bf16 copy.  Columns from p.d_store on are pad columns: never stored.
template <int N>
__device__ __forceinline__ void epilogue_dual(const SpmmParams &p, int64_t r, int c, const float (&acc)[N], float cnt) {
    if (c >= p.d_store) return;
    float ad[N], bs[N], o[N];
    if constexpr (N == 4) {
        if (p.io4) {                             // io4 implies d_store % 4 == 0: all four columns are stored
            if (p.addend) load_vec<4>(p.addend + r * p.ld_addend + c, ad);
            if (p.bias) load_vec<4>(p.bias + c, bs);
        }
    }
    if (N != 4 || !p.io4) {
#pragma unroll
        for (int x = 0; x < N; ++x) {
            if (c + x >= p.d_store) break;
            if (p.addend) ad[x] = p.addend[r * p.ld_addend + c + x];
            if (p.bias) bs[x] = p.bias[c + x];
        }
    }
#pragma unroll
    for (int x = 0; x < N; ++x) {
        float a = acc[x];
        if (p.reduce == TFGK_REDUCE_MEAN) a = __fdiv_rn(a, cnt);
        if (p.addend) a = __fadd_rn(__fmul_rn(a, p.alpha), __fmul_rn(ad[x], p.beta));
        else if (p.alpha != 1.0f) a = __fmul_rn(a, p.alpha);
        if (p.bias) a = __fadd_rn(a, bs[x]);
        o[x] = apply_act(a, p.act);
    }
    if constexpr (N == 4) {
        if (p.io4) {
            if (p.out) store_vec<4>(p.out + r * p.ldo + c, o);
            if (p.outb) {
                uint32_t b[4];
#pragma unroll
                for (int x = 0; x < 4; ++x) b[x] = __bfloat16_as_ushort(__float2bfloat16_rn(o[x]));
                *reinterpret_cast<uint2 *>(p.outb + r * p.ldob + c) = make_uint2(b[0] | (b[1] << 16), b[2] | (b[3] << 16));
            }
            return;
        }
    }
#pragma unroll
    for (int x = 0; x < N; ++x) {
        if (c + x >= p.d_store) break;
        if (p.out) p.out[r * p.ldo + c + x] = o[x];
        if (p.outb) p.outb[r * p.ldob + c + x] = __bfloat16_as_ushort(__float2bfloat16_rn(o[x]));
    }
}

constexpr int kSpmmThreads = 256;

// G: lanes per row (power of two), NC: vectors per lane, IS_MAX: max-reduce instead of sum/mean, U: rows in flight
template <int VEC, int G, int NC, bool IS_MAX, int U, typename T, bool DUAL = false>
__global__ void __launch_bounds__(kSpmmThreads) spmm_kernel(const SpmmParams p) {
    constexpr int RPW = 32 / G;   // rows per warp
    const int lane = threadIdx.x & 31;
    const int gl = lane & (G - 1);
    const int grp = lane / G;
    const int64_t warp_global = (int64_t)blockIdx.x * (kSpmmThreads / 32) + (threadIdx.x >> 5);
    const int64_t r = warp_global * RPW + grp;
    const bool row_ok = r < p.n_dst;

    int64_t start = 0;
    int deg = 0;
    if (row_ok) {
        start = p.rowptr[r];
        deg = (int)(p.rowptr[r + 1] - start);
    }
    int deg_max = deg;
    if constexpr (RPW > 1) {
#pragma unroll
        for (int off = 16; off >= G; off >>= 1) deg_max = max(deg_max, __shfl_xor_sync(0xffffffffu, deg_max, off));
    }

    int coff[NC];
    bool cok[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        coff[k] = (gl + k * G) * VEC;
        cok[k] = coff[k] < p.D;
    }

    float acc[NC][VEC];
#pragma unroll
    for (int k = 0; k < NC; ++k)
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[k][v] = IS_MAX ? -FLT_MAX : 0.0f;

    const bool weighted = p.w != nullptr;
    const T *__restrict__ h = rows_of<T>(p);

    for (int t = 0; t < deg_max; t += G) {
        // coalesced read of up to G (col, w) pairs of this row
        const int e = t + gl;
        int my_c = 0;
        float my_w = 1.0f;
        if (e < deg) {
            my_c = ld_stream_i32(p.col + start + e);
            if (weighted) my_w = ld_stream_f32(p.w + start + e);
        }
        const int nb = min(G, deg - t);           // edges of this row in the batch (may be <= 0)
        const int nb_max = min(G, deg_max - t);   // warp-uniform trip count
        for (int j = 0; j < nb_max; j += U) {
            float v[U][NC][VEC];
            float ww[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int src = j + u;
                const int c = __shfl_sync(0xffffffffu, my_c, src, G);
                ww[u] = __shfl_sync(0xffffffffu, my_w, src, G);
                const bool ok = src < nb;
                const T *rowp = h + (int64_t)c * p.ldh;
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    if (ok && cok[k]) load_vec<VEC>(rowp + coff[k], v[u][k]);
                }
                if constexpr (sizeof(T) == 1) {             // fp8: x^ = float(q) * 2^k of the source row's group
                    if (ok) {
                        const float s = pow2i(__ldg(p.hexp + (int64_t)c * p.n_grp + p.grp0));
#pragma unroll
                        for (int k = 0; k < NC; ++k) v[u][k][0] = __fmul_rn(v[u][k][0], s);
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
                                const float m = __fmul_rn(v[u][k][x], ww[u]);   // gcn_mapper rounding
                                acc[k][x] = IS_MAX ? fmaxf(acc[k][x], m) : __fadd_rn(acc[k][x], m);
                            }
                        }
                    }
                }
            }
        }
    }

    if (!row_ok) return;
    const bool is_mean = p.reduce == TFGK_REDUCE_MEAN;
    const float cnt = (float)max(deg, 1);
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        if (!cok[k]) continue;
        if constexpr (DUAL) {
            epilogue_dual<VEC>(p, r, coff[k], acc[k], cnt);
            continue;
        }
        float o[VEC];
        float ad[VEC];
        float bs[VEC];
        if (p.addend) load_vec<VEC>(p.addend + r * p.ld_addend + coff[k], ad);
        if (p.bias) load_vec<VEC>(p.bias + coff[k], bs);
#pragma unroll
        for (int x = 0; x < VEC; ++x) {
            float a = acc[k][x];
            if (is_mean) a = __fdiv_rn(a, cnt);
            if (p.addend) a = __fadd_rn(__fmul_rn(a, p.alpha), __fmul_rn(ad[x], p.beta));
            else if (p.alpha != 1.0f) a = __fmul_rn(a, p.alpha);
            if (p.bias) a = __fadd_rn(a, bs[x]);
            o[x] = apply_act(a, p.act);
        }
        store_vec<VEC>(p.out + r * p.ldo + coff[k], o);
    }
}


// ------------------------------------------------------------------------------------------------------------
// cp.async variant.  Register double-buffering cannot overlap two gather rounds: a warp has six counting scoreboard
// slots, ptxas puts the loads of both rounds on the same slots, and the first use of round g then also waits for
// round g+1 (visible in the SASS).  LDGSTS copies are tracked by commit groups instead, so a
// per-warp shared-memory ring of S stages x U rows keeps (S-1)*U rows in flight per warp with no register cost.
// Each lane copies - and later reads back - only its own 16-byte slices: shared memory is used as an asynchronous
// extension of the register file, no cross-lane traffic, no barriers.  Edge streaming: a warp owns kAsyncRows
// consecutive rows = a contiguous CSR range, walked in rounds of U edges regardless of row boundaries, so the memory
// pipe never drains at a row change.  Same rounding and order as spmm_kernel => same bits.
// ------------------------------------------------------------------------------------------------------------
constexpr int kAsyncRows = 32;
constexpr int kAsyncWarps = 4;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// one lane's slice of a row: four elements, 16 bytes of fp32 or 8 bytes of bf16
__device__ __forceinline__ void cp_async_slice(uint32_t dst, const float *src) { cp_async16(dst, src); }
__device__ __forceinline__ void cp_async_slice(uint32_t dst, const uint16_t *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}

template <int NC, bool IS_MAX, int U, int S, typename T, bool DUAL = false>
__global__ void __launch_bounds__(kAsyncWarps * 32) spmm_async_kernel(const SpmmParams p, uint32_t row_bytes) {
    static_assert(32 % U == 0, "a round must not straddle an index chunk");
    constexpr int RPC = 32 / U;
    extern __shared__ __align__(16) uint8_t ring_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t task = (int64_t)blockIdx.x * kAsyncWarps + warp;
    int64_t r0, r1, e_begin, e_stop;
    int slot = -1;
    if (p.task_row != nullptr) {
        if (task >= p.n_tasks) return;
        r0 = p.task_row[task];
        r1 = r0 + p.task_nrows[task];
        e_begin = p.task_e0[task];
        e_stop = p.task_e1[task];
        slot = p.task_slot[task];
    } else {
        r0 = task * kAsyncRows;
        if (r0 >= p.n_dst) return;
        r1 = min((int64_t)p.n_dst, r0 + kAsyncRows);
        e_begin = p.rowptr[r0];
        e_stop = p.rowptr[r1];
    }
    const int64_t rp_lo = p.rowptr[min(r0 + lane, r1)];
    const int64_t rp_hi = p.rowptr[min(r0 + lane + 1, r1)];
    const int n_edges = (int)(e_stop - e_begin);
    const int n_rounds = (n_edges + U - 1) / U;
    const bool weighted = p.w != nullptr;
    const uint32_t stage_bytes = U * row_bytes;
    uint8_t *my_ring = ring_raw + (size_t)warp * S * stage_bytes;
    const uint32_t ring_addr = (uint32_t)__cvta_generic_to_shared(my_ring);

    int coff[NC];
    bool cok[NC];
    float acc[NC][4];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        coff[k] = (lane + 32 * k) * 4;
        cok[k] = coff[k] < p.D;
#pragma unroll
        for (int x = 0; x < 4; ++x) acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
    }
    int64_t r = r0;
    // a hub slice (slot >= 0) never closes its row: the partial sum goes to the scratch slot instead
    int row_end = slot >= 0 ? 0x7fffffff : (int)(__shfl_sync(0xffffffffu, rp_hi, 0) - e_begin);
    const bool is_mean = p.reduce == TFGK_REDUCE_MEAN;

    auto finalize_row = [&]() {
        const int64_t row_start = __shfl_sync(0xffffffffu, rp_lo, (int)(r - r0));
        const int deg = (int)(row_end + e_begin - row_start);
        const float cnt = (float)max(deg, 1);
#pragma unroll
        for (int k = 0; k < NC; ++k) {
            if (DUAL && cok[k]) {
                epilogue_dual<4>(p, r, coff[k], acc[k], cnt);
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
            } else if (cok[k]) {
                float ad[4], bs[4], o[4];
                if (p.addend) load_vec<4>(p.addend + r * p.ld_addend + coff[k], ad);
                if (p.bias) load_vec<4>(p.bias + coff[k], bs);
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    float a = acc[k][x];
                    if (is_mean) a = __fdiv_rn(a, cnt);
                    if (p.addend) a = __fadd_rn(__fmul_rn(a, p.alpha), __fmul_rn(ad[x], p.beta));
                    else if (p.alpha != 1.0f) a = __fmul_rn(a, p.alpha);
                    if (p.bias) a = __fadd_rn(a, bs[x]);
                    o[x] = apply_act(a, p.act);
                    acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
                }
                store_vec<4>(p.out + r * p.ldo + coff[k], o);
            }
        }
        ++r;
        if (r < r1) row_end = (int)(__shfl_sync(0xffffffffu, rp_hi, (int)(r - r0)) - e_begin);
    };
    auto load_chunk = [&](int c, int &ci, float &wi) {
        const int e = c * 32 + lane;
        ci = 0;
        wi = 1.0f;
        if (e < n_edges) {
            ci = ld_stream_i32(p.col + e_begin + e);
            if (weighted) wi = ld_stream_f32(p.w + e_begin + e);
        }
    };
    // copy round g (edges [g*U, g*U+U)) into ring stage g % S; always commits one group (possibly empty)
    auto issue = [&](int g, int ci) {
        if (g < n_rounds) {
            const int base = (g % RPC) * U;
            const uint32_t dst0 = ring_addr + (uint32_t)(g % S) * stage_bytes;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int c = __shfl_sync(0xffffffffu, ci, base + u);
                if (g * U + u < n_edges) {
                    const T *rowp = rows_of<T>(p) + (int64_t)c * p.ldh;
#pragma unroll
                    for (int k = 0; k < NC; ++k)
                        if (cok[k]) cp_async_slice(dst0 + u * row_bytes + coff[k] * (uint32_t)sizeof(T), rowp + coff[k]);
                }
            }
        }
        cp_async_commit();
    };

    // Index registers (ca: even chunks, cb: odd chunks) are dead once the chunk's last round has been ISSUED; its
    // weights are needed until that round is CONSUMED, S-1 iterations later: wa/wb serve the consumer, wna/wnb hold the
    // weights fetched ahead together with the indices (requires S <= 2*RPC, asserted below).
    static_assert(S <= 2 * RPC, "weight look-ahead registers would be overwritten before they are consumed");
    int ca, cb;
    float wa, wb, wna = 1.0f, wnb = 1.0f;
    load_chunk(0, ca, wa);
    load_chunk(1, cb, wb);
    // prologue: S-1 rounds in flight (they all live in chunk 0 / 1 as long as (S-1)*U <= 64)
#pragma unroll
    for (int g = 0; g < S - 1; ++g) issue(g, ((g / RPC) & 1) ? cb : ca);
    if (S - 1 >= RPC) load_chunk(2, ca, wna);       // chunk 0 was issued completely by the prologue

    for (int g = 0; g < n_rounds; ++g) {
        // keep the pipe full: round g+S-1 goes into the stage consumed in the previous iteration
        {
            const int gn = g + S - 1;
            issue(gn, ((gn / RPC) & 1) ? cb : ca);
        }
        cp_async_wait<S - 1>();                     // round g has landed (groups retire in order)
        const int cc = g / RPC;
        const float wi = (cc & 1) ? wb : wa;
        const int base = (g % RPC) * U;
        const uint8_t *sbuf = my_ring + (size_t)(g % S) * stage_bytes;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int e = g * U + u;
            const float we = __shfl_sync(0xffffffffu, wi, base + u);
            if (e < n_edges) {
                while (e == row_end) finalize_row();
#pragma unroll
                for (int k = 0; k < NC; ++k) {
                    if (cok[k]) {
                        const float4 v = load_row4<T>(sbuf + (size_t)u * row_bytes + coff[k] * sizeof(T));
                        const float m0 = __fmul_rn(v.x, we), m1 = __fmul_rn(v.y, we), m2 = __fmul_rn(v.z, we), m3 = __fmul_rn(v.w, we);
                        acc[k][0] = IS_MAX ? fmaxf(acc[k][0], m0) : __fadd_rn(acc[k][0], m0);
                        acc[k][1] = IS_MAX ? fmaxf(acc[k][1], m1) : __fadd_rn(acc[k][1], m1);
                        acc[k][2] = IS_MAX ? fmaxf(acc[k][2], m2) : __fadd_rn(acc[k][2], m2);
                        acc[k][3] = IS_MAX ? fmaxf(acc[k][3], m3) : __fadd_rn(acc[k][3], m3);
                    }
                }
            }
        }
        // the index chunk that the LAST issued round (g+S-1) no longer needs can be refilled: chunk j is dead once
        // round (j+1)*RPC - 1 has been issued, i.e. when g + S - 1 == (j+1)*RPC - 1
        if ((g + 1) % RPC == 0) {                   // chunk cc fully consumed: promote the look-ahead weights
            if (cc & 1) wb = wnb; else wa = wna;
        }
        if ((g + S) % RPC == 0) {
            const int dead = (g + S) / RPC - 1;
            if (dead & 1) load_chunk(dead + 2, cb, wnb); else load_chunk(dead + 2, ca, wna);
        }
    }
    if (slot >= 0) {                                  // hub slice: raw partial, merged by spmm_hub_fixup_kernel
#pragma unroll
        for (int k = 0; k < NC; ++k)
            if (cok[k]) store_vec<4>(p.scratch + (int64_t)slot * p.D + coff[k], acc[k]);
        return;
    }
    while (r < r1) finalize_row();
}

// The epilogue of tfgk_spmm_proj_f32 for NB finished rows row0 .. row0+nrows-1 whose F-wide aggregates sit at agg
// (ldagg floats apart): out[r, c] = act(fmaf chain over k = 0 .. F-1 of agg[r, k] * W[k, c] from +0, + bias[c]).  Lane j
// computes columns 4j .. 4j+3, so one W row serves all NB rows; a row's bits depend on nothing but its own aggregate.
// W rows are ldw floats apart: PADDED = ldw is a multiple of 4 with zero columns from pu on (the shared-memory copy);
// otherwise W is read column by column with bounds checks (the hub fix-up reads it from global memory).
template <int NB, bool PADDED>
__device__ __forceinline__ void project_rows(const SpmmParams &p, const float *__restrict__ Wm, int ldw,
                                             const float *agg, int ldagg, int nrows, int F, int64_t row0, int lane) {
    const int c = lane * 4;
    if (c >= p.pu) return;
    float o[NB][4];
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
        for (int x = 0; x < 4; ++x) o[b][x] = 0.0f;
    for (int k = 0; k < F; k += 4) {
        float wk[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (PADDED) {
                const float4 t = *reinterpret_cast<const float4 *>(Wm + (k + i) * ldw + c);
                wk[i][0] = t.x; wk[i][1] = t.y; wk[i][2] = t.z; wk[i][3] = t.w;
            } else {
#pragma unroll
                for (int x = 0; x < 4; ++x) wk[i][x] = c + x < p.pu ? __ldg(Wm + (int64_t)(k + i) * ldw + c + x) : 0.0f;
            }
        }
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const float4 a = *reinterpret_cast<const float4 *>(agg + b * ldagg + k);
#pragma unroll
            for (int x = 0; x < 4; ++x) {
                o[b][x] = fmaf(a.x, wk[0][x], o[b][x]);
                o[b][x] = fmaf(a.y, wk[1][x], o[b][x]);
                o[b][x] = fmaf(a.z, wk[2][x], o[b][x]);
                o[b][x] = fmaf(a.w, wk[3][x], o[b][x]);
            }
        }
    }
    float bs[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.bias) {
        if (p.pio4) load_vec<4>(p.bias + c, bs);
        else
#pragma unroll
            for (int x = 0; x < 4; ++x) if (c + x < p.pu) bs[x] = p.bias[c + x];
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        if (b >= nrows) break;
        float v[4];
#pragma unroll
        for (int x = 0; x < 4; ++x) v[x] = apply_act(p.bias ? __fadd_rn(o[b][x], bs[x]) : o[b][x], p.act);
        float *dst = p.out + (row0 + b) * p.ldo + c;
        if (p.pio4) store_vec<4>(dst, v);
        else
#pragma unroll
            for (int x = 0; x < 4; ++x) if (c + x < p.pu) dst[x] = v[x];
    }
}

// ------------------------------------------------------------------------------------------------------------
// TMA ring variant (north_star: "staged through TMA into shared memory").  Same edge streaming, ring and arithmetic as
// spmm_async_kernel, but the neighbour rows of a round of U = 4 edges are fetched by the TMA unit: lane 0 arms the
// stage's mbarrier with the round's transaction bytes and lanes 0-3 each issue one 1-D cp.async.bulk of a whole row
// (row_bytes = 4 D), which leaves the LSU issue slots of the cp.async ring to the consumer.  Each warp owns S mbarriers;
// a stage is re-armed only after every lane has read it (__syncwarp before the copies are issued).  A short last round
// copies only its valid rows.  Same rounding and order => same bits.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_row(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

__device__ __forceinline__ void mbar_wait_parity(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (spin > (1u << 28)) __trap();     // a lost transaction becomes a launch failure, never a hang
    }
}

// PROJ (tfgk_spmm_proj_f32, fp32 SUM only): the finished rows of a warp are projected through W in batches of kProjRows
// (project_rows), with W copied into shared memory once per CTA of WARPS warps, behind the ring and its mbarriers.
constexpr int kProjRows = 4;
constexpr int kProjWarps = 8;

// shared memory of spmm_tma4_kernel: the ring, the mbarriers, fp8 exponents or (PROJ) W padded to pu rounded up to 4
// columns and kProjRows aggregate rows per warp
template <bool PROJ, typename T>
__host__ __device__ inline size_t tma4_smem_bytes(int warps, int S, uint32_t row_bytes, int D, int pu) {
    const size_t stage_pitch = ((size_t)4 * row_bytes + 127) & ~(size_t)127;
    size_t bytes = (size_t)warps * S * stage_pitch + (size_t)warps * S * 8 +
                   (sizeof(T) == 1 ? (size_t)warps * S * 4 * sizeof(uint16_t) : 0);
    if (PROJ) bytes = (bytes + 15) / 16 * 16 + ((size_t)D * ((pu + 3) / 4 * 4) + (size_t)warps * kProjRows * D) * 4;
    return bytes;
}

template <bool IS_MAX, int S, typename T, bool DUAL, bool PROJ, int WARPS>
__device__ __forceinline__ void spmm_tma4_body(const SpmmParams &p, uint32_t row_bytes) {
    constexpr int U = 4, RPC = 32 / U;
    constexpr bool FP8 = sizeof(T) == 1;
    static_assert(S <= 2 * RPC, "weight look-ahead registers would be overwritten before they are consumed");
    static_assert(!PROJ || (!IS_MAX && !DUAL && sizeof(T) == 4), "the projection epilogue follows an fp32 sum");
    extern __shared__ __align__(128) uint8_t g4_ring[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t stage_bytes = (U * row_bytes + 127u) & ~127u;
    uint8_t *my_ring = g4_ring + (size_t)warp * S * stage_bytes;
    const uint32_t ring_addr = (uint32_t)__cvta_generic_to_shared(my_ring);
    uint64_t *bars = reinterpret_cast<uint64_t *>(g4_ring + (size_t)WARPS * S * stage_bytes) + warp * S;
    // fp8: the exponents of every edge in the ring, [S][U] 16-bit entries per warp (group 0 low byte, group 1 high byte)
    uint16_t *sexp = reinterpret_cast<uint16_t *>(g4_ring + (size_t)WARPS * S * (stage_bytes + 8)) + warp * S * U;
    const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(bars);
    // PROJ: W [D][ldw] and this warp's kProjRows aggregate rows; every thread helps copy W before any warp can leave
    float *w_s = nullptr, *agg_s = nullptr;
    const int ldw = (p.pu + 3) & ~3;
    if constexpr (PROJ) {
        w_s = reinterpret_cast<float *>(g4_ring + ((size_t)WARPS * S * (stage_bytes + 8) + 15) / 16 * 16);
        agg_s = w_s + (size_t)p.D * ldw + (size_t)warp * kProjRows * p.D;
        for (int i = threadIdx.x; i < p.D * ldw; i += WARPS * 32) {
            const int k = i / ldw, c = i - k * ldw;
            w_s[i] = c < p.pu ? __ldg(p.pw + (int64_t)k * p.pu + c) : 0.0f;
        }
        __syncthreads();
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < S; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8 * i));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const int64_t task = (int64_t)blockIdx.x * WARPS + warp;
    int64_t r0, r1, e_begin, e_stop;
    int slot = -1;
    if (p.task_row != nullptr) {
        if (task >= p.n_tasks) return;
        r0 = p.task_row[task];
        r1 = r0 + p.task_nrows[task];
        e_begin = p.task_e0[task];
        e_stop = p.task_e1[task];
        slot = p.task_slot[task];
    } else {
        r0 = task * kAsyncRows;
        if (r0 >= p.n_dst) return;
        r1 = min((int64_t)p.n_dst, r0 + kAsyncRows);
        e_begin = p.rowptr[r0];
        e_stop = p.rowptr[r1];
    }
    const int64_t rp_lo = p.rowptr[min(r0 + lane, r1)];
    const int64_t rp_hi = p.rowptr[min(r0 + lane + 1, r1)];
    const int n_edges = (int)(e_stop - e_begin);
    const int n_rounds = (n_edges + U - 1) / U;
    const bool weighted = p.w != nullptr;
    constexpr int NCX = 2;                         // up to 256 columns: two float4 slices per lane
    int coff[NCX];
    bool cok[NCX];
    float acc[NCX][4];
#pragma unroll
    for (int k = 0; k < NCX; ++k) {
        coff[k] = (lane + 32 * k) * 4;
        cok[k] = coff[k] < p.D;
#pragma unroll
        for (int x = 0; x < 4; ++x) acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
    }
    int64_t r = r0;
    int row_end = slot >= 0 ? 0x7fffffff : (int)(__shfl_sync(0xffffffffu, rp_hi, 0) - e_begin);
    const bool is_mean = p.reduce == TFGK_REDUCE_MEAN;

    int n_done = 0;                                 // PROJ: finished rows r - n_done .. r-1 waiting in agg_s
    auto project_done = [&]() {
        __syncwarp();
        project_rows<kProjRows, true>(p, w_s, ldw, agg_s, p.D, n_done, p.D, r - n_done, lane);
        __syncwarp();
        n_done = 0;
    };
    auto finalize_row = [&]() {
        const int64_t row_start = __shfl_sync(0xffffffffu, rp_lo, (int)(r - r0));
        const int deg = (int)(row_end + e_begin - row_start);
        const float cnt = (float)max(deg, 1);
#pragma unroll
        for (int k = 0; k < NCX; ++k) {
            if (PROJ) {                             // D <= 128: the row is acc[0] of lanes 0 .. D/4-1
                if (k == 0 && cok[0])
                    *reinterpret_cast<float4 *>(agg_s + n_done * p.D + coff[0]) = make_float4(acc[0][0], acc[0][1], acc[0][2], acc[0][3]);
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[k][x] = 0.0f;
            } else if (DUAL && cok[k]) {
                epilogue_dual<4>(p, r, coff[k], acc[k], cnt);
#pragma unroll
                for (int x = 0; x < 4; ++x) acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
            } else if (cok[k]) {
                float ad[4], bs[4], o[4];
                if (p.addend) load_vec<4>(p.addend + r * p.ld_addend + coff[k], ad);
                if (p.bias) load_vec<4>(p.bias + coff[k], bs);
#pragma unroll
                for (int x = 0; x < 4; ++x) {
                    float a = acc[k][x];
                    if (is_mean) a = __fdiv_rn(a, cnt);
                    if (p.addend) a = __fadd_rn(__fmul_rn(a, p.alpha), __fmul_rn(ad[x], p.beta));
                    else if (p.alpha != 1.0f) a = __fmul_rn(a, p.alpha);
                    if (p.bias) a = __fadd_rn(a, bs[x]);
                    o[x] = apply_act(a, p.act);
                    acc[k][x] = IS_MAX ? -FLT_MAX : 0.0f;
                }
                store_vec<4>(p.out + r * p.ldo + coff[k], o);
            }
        }
        ++r;
        if constexpr (PROJ) {
            if (++n_done == kProjRows) project_done();
        }
        if (r < r1) row_end = (int)(__shfl_sync(0xffffffffu, rp_hi, (int)(r - r0)) - e_begin);
    };
    auto load_chunk = [&](int c, int &ci, float &wi) {
        const int e = c * 32 + lane;
        ci = 0;
        wi = 1.0f;
        if (e < n_edges) {
            ci = ld_stream_i32(p.col + e_begin + e);
            if (weighted) wi = ld_stream_f32(p.w + e_begin + e);
        }
    };
    // fp8: lanes 0-3 load the exponents of the round they copy into xpend, and store them into sexp at the next issue, a
    // round later (the load has landed by then and the warp never waits on it); the consumer reads them after a __syncwarp
    uint32_t xpend = 0;
    int xslot = -1;
    // round g (edges [4g, 4g+4)) -> ring stage g % S: armed by lane 0, one row copy from each of lanes 0 .. valid-1
    auto issue = [&](int g, int ci) {
        if constexpr (FP8) {
            if (xslot >= 0 && lane < U) sexp[xslot * U + lane] = (uint16_t)xpend;
            xslot = -1;
        }
        if (g < n_rounds) {
            const int base = (g % RPC) * U;
            const int valid = min(U, n_edges - g * U);
            const int c = __shfl_sync(0xffffffffu, ci, base + (lane < U ? lane : 0));
            const uint32_t bar = bar0 + 8 * (uint32_t)(g % S);
            if (lane == 0)
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((uint32_t)valid * row_bytes)
                             : "memory");
            if (lane < valid)
                tma_row(ring_addr + (uint32_t)(g % S) * stage_bytes + (uint32_t)lane * row_bytes,
                        rows_of<T>(p) + (int64_t)c * p.ldh, row_bytes, bar);
            if constexpr (FP8) {
                if (lane < valid)
                    xpend = p.n_grp == 1 ? (uint32_t)(uint8_t)__ldg(p.hexp + c)
                                         : (uint32_t)__ldg(reinterpret_cast<const uint16_t *>(p.hexp) + c);
                xslot = g % S;
            }
        }
    };

    int ca, cb;
    float wa, wb, wna = 1.0f, wnb = 1.0f;
    load_chunk(0, ca, wa);
    load_chunk(1, cb, wb);
#pragma unroll
    for (int g = 0; g < S - 1; ++g) issue(g, ((g / RPC) & 1) ? cb : ca);
    if (S - 1 >= RPC) load_chunk(2, ca, wna);

    for (int g = 0; g < n_rounds; ++g) {
        __syncwarp();                               // every lane has finished reading stage (g-1) % S, which is re-armed now
        {
            const int gn = g + S - 1;
            issue(gn, ((gn / RPC) & 1) ? cb : ca);
        }
        if constexpr (FP8) __syncwarp();            // the exponents stored by issue() are visible to every lane
        mbar_wait_parity(bar0 + 8 * (uint32_t)(g % S), (uint32_t)(g / S) & 1u);
        const int cc = g / RPC;
        const float wi = (cc & 1) ? wb : wa;
        const int base = (g % RPC) * U;
        const uint8_t *sbuf = my_ring + (size_t)(g % S) * stage_bytes;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int e = g * U + u;
            const float we = __shfl_sync(0xffffffffu, wi, base + u);
            if (e < n_edges) {
                while (e == row_end) finalize_row();
                float xs[NCX];                          // fp8: 2^k of the source row's groups 0 and 1
                if constexpr (FP8) {
                    const uint32_t xe = sexp[(g % S) * U + u];
                    xs[0] = pow2i((int8_t)(xe & 0xFFu));
                    xs[1] = pow2i((int8_t)(xe >> 8));
                }
#pragma unroll
                for (int k = 0; k < NCX; ++k) {
                    if (cok[k]) {
                        float4 v = load_row4<T>(sbuf + (size_t)u * row_bytes + coff[k] * sizeof(T));
                        if constexpr (FP8) v = scale4(v, xs[k]);
                        const float m0 = __fmul_rn(v.x, we), m1 = __fmul_rn(v.y, we), m2 = __fmul_rn(v.z, we), m3 = __fmul_rn(v.w, we);
                        acc[k][0] = IS_MAX ? fmaxf(acc[k][0], m0) : __fadd_rn(acc[k][0], m0);
                        acc[k][1] = IS_MAX ? fmaxf(acc[k][1], m1) : __fadd_rn(acc[k][1], m1);
                        acc[k][2] = IS_MAX ? fmaxf(acc[k][2], m2) : __fadd_rn(acc[k][2], m2);
                        acc[k][3] = IS_MAX ? fmaxf(acc[k][3], m3) : __fadd_rn(acc[k][3], m3);
                    }
                }
            }
        }
        if ((g + 1) % RPC == 0) {
            if (cc & 1) wb = wnb; else wa = wna;
        }
        if ((g + S) % RPC == 0) {
            const int dead = (g + S) / RPC - 1;
            if (dead & 1) load_chunk(dead + 2, cb, wnb); else load_chunk(dead + 2, ca, wna);
        }
    }
    if (slot >= 0) {
#pragma unroll
        for (int k = 0; k < NCX; ++k)
            if (cok[k]) store_vec<4>(p.scratch + (int64_t)slot * p.D + coff[k], acc[k]);
        return;
    }
    while (r < r1) finalize_row();
    if constexpr (PROJ) {
        if (n_done > 0) project_done();
    }
}

template <bool IS_MAX, int S, typename T, bool DUAL = false>
__global__ void __launch_bounds__(kAsyncWarps * 32) spmm_tma4_kernel(const SpmmParams p, uint32_t row_bytes) {
    spmm_tma4_body<IS_MAX, S, T, DUAL, false, kAsyncWarps>(p, row_bytes);
}

// tfgk_spmm_proj_f32: the fp32 SUM ring with the projection epilogue, WARPS warps sharing one copy of W
template <int S, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) spmm_proj_tma4_kernel(const SpmmParams p, uint32_t row_bytes) {
    spmm_tma4_body<false, S, float, false, true, WARPS>(p, row_bytes);
}

// merges the slices of every hub row in slice order (deterministic) and applies the epilogue; one warp per hub row
// (PROJ: D <= 128; the merged row goes through project_rows with W read from global memory)
template <bool IS_MAX, bool DUAL, bool PROJ>
__device__ __forceinline__ void spmm_hub_fixup_body(const SpmmParams &p, float (*agg_s)[128]) {
    const int lane = threadIdx.x & 31;
    const int h = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (h >= p.n_hubs) return;
    const int64_t r = p.hub_row[h];
    const int s0 = p.hub_slot0[h], ns = p.hub_nslots[h];
    const float cnt = (float)max((int)(p.rowptr[r + 1] - p.rowptr[r]), 1);
    for (int c = lane * 4; c < p.D; c += 128) {
        float acc[4] = {IS_MAX ? -FLT_MAX : 0.f, IS_MAX ? -FLT_MAX : 0.f, IS_MAX ? -FLT_MAX : 0.f, IS_MAX ? -FLT_MAX : 0.f};
        for (int s = 0; s < ns; ++s) {
            float v[4];
            load_vec<4>(p.scratch + (int64_t)(s0 + s) * p.D + c, v);
#pragma unroll
            for (int x = 0; x < 4; ++x) acc[x] = IS_MAX ? fmaxf(acc[x], v[x]) : __fadd_rn(acc[x], v[x]);
        }
        if constexpr (PROJ) {
            store_vec<4>(&agg_s[threadIdx.x >> 5][c], acc);
            continue;
        }
        if constexpr (DUAL) {
            epilogue_dual<4>(p, r, c, acc, cnt);
            continue;
        }
        float ad[4], bs[4], o[4];
        if (p.addend) load_vec<4>(p.addend + r * p.ld_addend + c, ad);
        if (p.bias) load_vec<4>(p.bias + c, bs);
#pragma unroll
        for (int x = 0; x < 4; ++x) {
            float a = acc[x];
            if (p.reduce == TFGK_REDUCE_MEAN) a = __fdiv_rn(a, cnt);
            if (p.addend) a = __fadd_rn(__fmul_rn(a, p.alpha), __fmul_rn(ad[x], p.beta));
            else if (p.alpha != 1.0f) a = __fmul_rn(a, p.alpha);
            if (p.bias) a = __fadd_rn(a, bs[x]);
            o[x] = apply_act(a, p.act);
        }
        store_vec<4>(p.out + r * p.ldo + c, o);
    }
    if constexpr (PROJ) {
        __syncwarp();
        project_rows<1, false>(p, p.pw, p.pu, agg_s[threadIdx.x >> 5], 128, 1, p.D, r, lane);
    }
}

template <bool IS_MAX, bool DUAL = false>
__global__ void __launch_bounds__(256) spmm_hub_fixup_kernel(const SpmmParams p) {
    spmm_hub_fixup_body<IS_MAX, DUAL, false>(p, nullptr);
}

__global__ void __launch_bounds__(256) spmm_hub_fixup_proj_kernel(const SpmmParams p) {
    __shared__ __align__(16) float agg_s[8][128];      // the merged row of each warp
    spmm_hub_fixup_body<false, false, true>(p, agg_s);
}

template <int NC, int U, int S, typename T = float, bool DUAL = false>
static int launch_spmm_async(const SpmmParams &p, cudaStream_t st) {
    const uint32_t row_bytes = (uint32_t)(p.D * sizeof(T));
    const size_t smem = (size_t)kAsyncWarps * S * U * row_bytes;
    if (smem > 200 * 1024) return TFGK_ERR_UNSUPPORTED;
    const int64_t n_tasks = p.task_row ? p.n_tasks : ceil_div64(p.n_dst, kAsyncRows);
    const unsigned blocks = (unsigned)ceil_div64(n_tasks, kAsyncWarps);
    if (p.reduce == TFGK_REDUCE_MAX) {
        TFGK_CUDA(ensure_dynamic_smem(spmm_async_kernel<NC, true, U, S, T, DUAL>, smem));
        spmm_async_kernel<NC, true, U, S, T, DUAL><<<blocks, kAsyncWarps * 32, smem, st>>>(p, row_bytes);
    } else {
        TFGK_CUDA(ensure_dynamic_smem(spmm_async_kernel<NC, false, U, S, T, DUAL>, smem));
        spmm_async_kernel<NC, false, U, S, T, DUAL><<<blocks, kAsyncWarps * 32, smem, st>>>(p, row_bytes);
    }
    TFGK_LAUNCH_CHECK();
    if (p.task_row && p.n_hubs > 0) {
        const unsigned fb = (unsigned)ceil_div64(p.n_hubs, 8);
        if (p.reduce == TFGK_REDUCE_MAX) spmm_hub_fixup_kernel<true, DUAL><<<fb, 256, 0, st>>>(p);
        else spmm_hub_fixup_kernel<false, DUAL><<<fb, 256, 0, st>>>(p);
        TFGK_LAUNCH_CHECK();
    }
    return TFGK_OK;
}

template <int S, typename T = float, bool DUAL = false, bool PROJ = false, int WARPS = kAsyncWarps>
static int launch_spmm_tma4(const SpmmParams &p, cudaStream_t st) {
    // cp.async.bulk wants 16-byte aligned rows: D, ldh multiples of 16 bytes' worth of elements and an aligned base
    constexpr int kPer16 = 16 / (int)sizeof(T);
    const void *base = sizeof(T) == 4 ? (const void *)p.h : sizeof(T) == 2 ? (const void *)p.hb : (const void *)p.h8;
    if (p.D > 256 || p.D % kPer16 != 0 || p.ldh % kPer16 != 0 || !aligned16(base)) return TFGK_ERR_UNSUPPORTED;
    const uint32_t row_bytes = (uint32_t)(p.D * sizeof(T));
    const size_t smem = tma4_smem_bytes<PROJ, T>(WARPS, S, row_bytes, p.D, PROJ ? p.pu : 0);
    if (smem > 200 * 1024) return TFGK_ERR_UNSUPPORTED;
    const int64_t n_tasks = p.task_row ? p.n_tasks : ceil_div64(p.n_dst, kAsyncRows);
    const unsigned blocks = (unsigned)ceil_div64(n_tasks, WARPS);
    if constexpr (PROJ) {
        TFGK_CUDA(ensure_dynamic_smem(spmm_proj_tma4_kernel<S, WARPS>, smem));
        spmm_proj_tma4_kernel<S, WARPS><<<blocks, WARPS * 32, smem, st>>>(p, row_bytes);
    } else if (p.reduce == TFGK_REDUCE_MAX) {
        TFGK_CUDA(ensure_dynamic_smem(spmm_tma4_kernel<true, S, T, DUAL>, smem));
        spmm_tma4_kernel<true, S, T, DUAL><<<blocks, kAsyncWarps * 32, smem, st>>>(p, row_bytes);
    } else {
        TFGK_CUDA(ensure_dynamic_smem(spmm_tma4_kernel<false, S, T, DUAL>, smem));
        spmm_tma4_kernel<false, S, T, DUAL><<<blocks, kAsyncWarps * 32, smem, st>>>(p, row_bytes);
    }
    TFGK_LAUNCH_CHECK();
    if (p.task_row && p.n_hubs > 0) {
        const unsigned fb = (unsigned)ceil_div64(p.n_hubs, 8);
        if (PROJ) spmm_hub_fixup_proj_kernel<<<fb, 256, 0, st>>>(p);
        else if (p.reduce == TFGK_REDUCE_MAX) spmm_hub_fixup_kernel<true, DUAL><<<fb, 256, 0, st>>>(p);
        else spmm_hub_fixup_kernel<false, DUAL><<<fb, 256, 0, st>>>(p);
        TFGK_LAUNCH_CHECK();
    }
    return TFGK_OK;
}

// the cp.async ring by width: four float4 slices of a row per lane at most, 512 columns
template <typename T, bool DUAL = false>
static int dispatch_spmm_async(const SpmmParams &p, cudaStream_t st) {
    const int lanes = (p.D + 3) / 4;
    return lanes <= 32 ? launch_spmm_async<1, 4, 3, T, DUAL>(p, st)
         : lanes <= 64 ? launch_spmm_async<2, 4, 4, T, DUAL>(p, st)
         : lanes <= 96 ? launch_spmm_async<3, 4, 3, T, DUAL>(p, st)
                       : launch_spmm_async<4, 2, 4, T, DUAL>(p, st);
}

template <int VEC, int G, int NC, int U, typename T, bool DUAL>
static int launch_spmm(const SpmmParams &p, cudaStream_t st) {
    constexpr int rows_per_block = (kSpmmThreads / 32) * (32 / G);
    const int64_t blocks = ceil_div64(p.n_dst, rows_per_block);
    if (p.reduce == TFGK_REDUCE_MAX)
        spmm_kernel<VEC, G, NC, true, U, T, DUAL><<<(unsigned)blocks, kSpmmThreads, 0, st>>>(p);
    else
        spmm_kernel<VEC, G, NC, false, U, T, DUAL><<<(unsigned)blocks, kSpmmThreads, 0, st>>>(p);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

template <int VEC, typename T = float, bool DUAL = false>
static int dispatch_spmm(const SpmmParams &p, int lanes, cudaStream_t st) {
    // lanes = number of VEC-wide vectors in a row (<= 128)
    if (lanes <= 1) return launch_spmm<VEC, 1, 1, 8, T, DUAL>(p, st);
    if (lanes <= 2) return launch_spmm<VEC, 2, 1, 8, T, DUAL>(p, st);
    if (lanes <= 4) return launch_spmm<VEC, 4, 1, 8, T, DUAL>(p, st);
    if (lanes <= 8) return launch_spmm<VEC, 8, 1, 8, T, DUAL>(p, st);
    if (lanes <= 16) return launch_spmm<VEC, 16, 1, 8, T, DUAL>(p, st);
    if (lanes <= 32) return launch_spmm<VEC, 32, 1, 8, T, DUAL>(p, st);
    if (lanes <= 64) return launch_spmm<VEC, 32, 2, 4, T, DUAL>(p, st);
    if (lanes <= 96) return launch_spmm<VEC, 32, 3, 2, T, DUAL>(p, st);
    return launch_spmm<VEC, 32, 4, 2, T, DUAL>(p, st);
}

// argument checks shared by the fp32 and bf16 entry points: TFGK_OK to go on (with *nothing_to_do set for an empty
// launch), or the error status
static int spmm_validate(const int64_t *rowptr, const void *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                         const float *addend, int64_t ld_addend, int act, const void *out, int64_t ldo,
                         const tfgk_plan *plan, bool *nothing_to_do) {
    *nothing_to_do = true;
    TFGK_CHECK_ARG(n_dst >= 0 && D >= 0, "spmm: negative size (n_dst=%d, D=%d)", n_dst, D);
    if (plan != nullptr && plan->n_hubs > 0)
        TFGK_CHECK_ARG(plan->scratch != nullptr && plan->scratch_bytes >= (size_t)plan->n_slots * D * sizeof(float),
                       "spmm: plan scratch too small (need %zu bytes)", (size_t)plan->n_slots * D * sizeof(float));
    TFGK_CHECK_ARG(reduce >= TFGK_REDUCE_SUM && reduce <= TFGK_REDUCE_MAX, "spmm: unknown reduce %d", reduce);
    TFGK_CHECK_ARG(act == TFGK_ACT_NONE || act == TFGK_ACT_RELU, "spmm: unknown activation %d", act);
    if (n_dst == 0 || D == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && out && h, "spmm: null pointer");
    TFGK_CHECK_ARG(ldh >= D && ldo >= D && (!addend || ld_addend >= D), "spmm: leading dimension < D");
    *nothing_to_do = false;
    return TFGK_OK;
}

static SpmmParams spmm_params(const int64_t *rowptr, const int32_t *col, const float *w, int64_t ldh, int32_t n_dst,
                              int reduce, float alpha, const float *addend, int64_t ld_addend, float beta,
                              const float *bias, int act, float *out, int64_t ldo, int c0, int width) {
    SpmmParams p;
    p.rowptr = rowptr; p.col = col; p.w = w;
    p.h = nullptr; p.hb = nullptr; p.ldh = ldh; p.n_dst = n_dst;
    p.h8 = nullptr; p.hexp = nullptr; p.n_grp = 0; p.grp0 = 0;
    p.D = width;
    p.reduce = reduce; p.alpha = alpha;
    p.addend = addend ? addend + c0 : nullptr; p.ld_addend = ld_addend; p.beta = beta;
    p.bias = bias ? bias + c0 : nullptr; p.act = act;
    p.out = out ? out + c0 : nullptr; p.ldo = ldo;
    p.outb = nullptr; p.ldob = 0; p.d_store = width; p.io4 = false;
    p.n_tasks = 0; p.task_row = nullptr; p.task_nrows = nullptr; p.task_e0 = nullptr; p.task_e1 = nullptr;
    p.task_slot = nullptr; p.n_hubs = 0; p.hub_row = nullptr; p.hub_slot0 = nullptr; p.hub_nslots = nullptr;
    p.scratch = nullptr;
    p.pw = nullptr; p.pu = 0; p.pio4 = false;
    return p;
}

}  // namespace tfgk

using namespace tfgk;

extern "C" int tfgk_spmm_f32(const int64_t *rowptr, const int32_t *col, const float *w,
                             const float *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                             float alpha, const float *addend, int64_t ld_addend, float beta,
                             const float *bias, int act,
                             float *out, int64_t ldo, const tfgk_plan *plan, void *stream) {
    bool nothing_to_do = true;
    const int vrc = spmm_validate(rowptr, h, ldh, n_dst, D, reduce, addend, ld_addend, act, out, ldo, plan, &nothing_to_do);
    if (vrc != TFGK_OK || nothing_to_do) return vrc;

    const bool vec4 = (D % 4 == 0) && (ldh % 4 == 0) && (ldo % 4 == 0) && aligned16(h) && aligned16(out) &&
                      (!addend || ((ld_addend % 4 == 0) && aligned16(addend))) && (!bias || aligned16(bias));
    const int vec = vec4 ? 4 : 1;
    const int cols_per_launch = 128 * vec;   // 32 lanes x NC<=4 vectors
    for (int c0 = 0; c0 < D; c0 += cols_per_launch) {
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   c0, (D - c0 < cols_per_launch) ? D - c0 : cols_per_launch);
        p.h = h + c0;
        // the plan applies when the whole width runs in one launch of a ring kernel (scratch rows are D wide)
        if (plan != nullptr && plan->n_tasks > 0 && vec4 && D >= 32 && D <= cols_per_launch) use_plan(p, plan);
        if (vec4 && p.D >= 32) {
            // the TMA row-copy ring with three stages up to 256 columns, the cp.async ring above
            int rcr = launch_spmm_tma4<3>(p, as_stream(stream));
            if (rcr == TFGK_ERR_UNSUPPORTED) rcr = dispatch_spmm_async<float>(p, as_stream(stream));
            if (rcr != TFGK_ERR_UNSUPPORTED) { if (rcr != TFGK_OK) return rcr; continue; }
        }
        const int lanes = (p.D + vec - 1) / vec;
        const int rc = vec4 ? dispatch_spmm<4>(p, lanes, as_stream(stream)) : dispatch_spmm<1>(p, lanes, as_stream(stream));
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}

// Aggregate, then project: out = act((A x) W + bias) with the aggregate A x never stored.  The aggregation is
// tfgk_spmm_f32's TMA ring over the F-wide rows of x, with its plan taken where tfgk_spmm_f32 takes it for x (F >= 32; x
// has 16-byte aligned rows here), so every aggregate is bit-identical to tfgk_spmm_f32's SUM; each finished row is then
// projected in the ring kernel's epilogue (project_rows), hub rows in the fix-up kernel after their slices are merged.
extern "C" int tfgk_spmm_proj_f32(const int64_t *rowptr, const int32_t *col, const float *w,
                                  const float *x, int64_t ldx, int32_t n_dst, int32_t F, const float *W, int32_t U,
                                  const float *bias, int act, float *out, int64_t ldo, const tfgk_plan *plan, void *stream) {
    TFGK_CHECK_ARG(n_dst >= 0 && F >= 0 && U >= 0, "spmm_proj: negative size (n_dst=%d, F=%d, U=%d)", n_dst, F, U);
    TFGK_CHECK_ARG(act == TFGK_ACT_NONE || act == TFGK_ACT_RELU, "spmm_proj: unknown activation %d", act);
    if (F < 4 || F % 4 != 0 || F >= U || U > 128 || ldx % 4 != 0 || !aligned16(x)) return TFGK_ERR_UNSUPPORTED;
    TFGK_CHECK_ARG(ldx >= F && ldo >= U, "spmm_proj: leading dimension too small (ldx=%lld, ldo=%lld)", (long long)ldx,
                   (long long)ldo);
    if (plan != nullptr && plan->n_hubs > 0 && F >= 32)
        TFGK_CHECK_ARG(plan->scratch != nullptr && plan->scratch_bytes >= (size_t)plan->n_slots * F * sizeof(float),
                       "spmm_proj: plan scratch too small (need %zu bytes)", (size_t)plan->n_slots * F * sizeof(float));
    if (n_dst == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && x && W && out, "spmm_proj: null pointer");
    SpmmParams p = spmm_params(rowptr, col, w, ldx, n_dst, TFGK_REDUCE_SUM, 1.0f, nullptr, 0, 0.0f, bias, act, out, ldo, 0, F);
    p.h = x;
    p.pw = W; p.pu = U;
    p.pio4 = U % 4 == 0 && ldo % 4 == 0 && aligned16(out) && (!bias || aligned16(bias));
    if (plan != nullptr && plan->n_tasks > 0 && F >= 32) use_plan(p, plan);
    return launch_spmm_tma4<3, float, false, true, kProjWarps>(p, as_stream(stream));
}

// bf16 rows.  The kernels are the fp32 ones with each element widened on the way from shared memory (or from global
// memory on the scalar path), with the same lane-to-column mapping, plan and order of operations: the output is the
// fp32 kernel's output over a widened table with the same leading dimension, bit for bit.  The rings (and the plan) need
// 8-byte aligned rows of D % 4 == 0 elements, 32 <= D <= 512, where the fp32 kernel needs 16-byte aligned ones: the two
// layouts correspond element for element, so both take the plan for the same shapes.
extern "C" int tfgk_spmm_bf16(const int64_t *rowptr, const int32_t *col, const float *w,
                              const uint16_t *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                              float alpha, const float *addend, int64_t ld_addend, float beta,
                              const float *bias, int act,
                              float *out, int64_t ldo, const tfgk_plan *plan, void *stream) {
    bool nothing_to_do = true;
    const int vrc = spmm_validate(rowptr, h, ldh, n_dst, D, reduce, addend, ld_addend, act, out, ldo, plan, &nothing_to_do);
    if (vrc != TFGK_OK || nothing_to_do) return vrc;

    // rows4: every lane moves four consecutive columns (8 bytes of h, 16 bytes of out / addend / bias)
    const bool rows4 = (D % 4 == 0) && (ldh % 4 == 0) && aligned8(h) && (ldo % 4 == 0) && aligned16(out) &&
                       (!addend || ((ld_addend % 4 == 0) && aligned16(addend))) && (!bias || aligned16(bias));
    cudaStream_t st = as_stream(stream);
    if (rows4 && D >= 32 && D <= 512) {                // the ring kernels: one launch over the whole width
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   0, D);
        p.hb = h;
        // the plan is taken exactly when the fp32 entry point takes it for the same shape
        if (plan != nullptr && plan->n_tasks > 0) use_plan(p, plan);
        // 256-byte rows at D = 128: six ring stages keep as many bytes in flight per warp as three stages of fp32 rows
        const int rc = launch_spmm_tma4<6, uint16_t>(p, st);        // TFGK_ERR_UNSUPPORTED unless 16-byte rows, D <= 256
        if (rc != TFGK_ERR_UNSUPPORTED) return rc;
        return dispatch_spmm_async<uint16_t>(p, st);
    }
    for (int c0 = 0; c0 < D; c0 += 128) {               // scalar path: 32 lanes x 4 single columns per launch
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   c0, D - c0 < 128 ? D - c0 : 128);
        p.hb = h + c0;
        const int rc = dispatch_spmm<1, uint16_t>(p, p.D, st);
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}

// bf16 rows, fp32 and/or bf16 output.  The kernels are tfgk_spmm_bf16's, instantiated with the dual-store epilogue
// (epilogue_dual), and take the plan exactly where tfgk_spmm_bf16 takes it for the same h, addend, bias and fp32 out (a
// dense fp32 out when only the bf16 copy is written): `out` is then bit-identical to tfgk_spmm_bf16's, and out_bf16 is
// its rounding.  Rows without the plan are summed strictly in CSR order by every kernel, so the ring kernels may also run
// where tfgk_spmm_bf16 takes the scalar path: a table whose rows are 16-byte (8-byte) aligned with ldh >= D rounded up to
// 8 (4) is read with its pad columns, which makes the TMA (cp.async) ring available to any D.  Pad columns never interact
// with the first D and are never stored.
extern "C" int tfgk_spmm_bf16_dual(const int64_t *rowptr, const int32_t *col, const float *w,
                                   const uint16_t *h, int64_t ldh, int32_t n_dst, int32_t D, int reduce,
                                   float alpha, const float *addend, int64_t ld_addend, float beta,
                                   const float *bias, int act,
                                   float *out, int64_t ldo, uint16_t *out_bf16, int64_t ldob,
                                   const tfgk_plan *plan, void *stream) {
    TFGK_CHECK_ARG(out != nullptr || out_bf16 != nullptr, "spmm_bf16_dual: both outputs are null");
    bool nothing_to_do = true;
    const int vrc = spmm_validate(rowptr, h, ldh, n_dst, D, reduce, addend, ld_addend, act,
                                  out ? (const void *)out : (const void *)out_bf16, out ? ldo : ldob, plan, &nothing_to_do);
    if (vrc != TFGK_OK || nothing_to_do) return vrc;
    TFGK_CHECK_ARG(!out_bf16 || ldob >= D, "spmm_bf16_dual: leading dimension < D (ldob=%lld)", (long long)ldob);
    TFGK_CHECK_ARG((reinterpret_cast<uintptr_t>(h) & 1u) == 0 && (reinterpret_cast<uintptr_t>(out_bf16) & 1u) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 3u) == 0, "spmm_bf16_dual: misaligned h, out or out_bf16");

    const bool in_aligned = (!addend || ((ld_addend % 4 == 0) && aligned16(addend))) && (!bias || aligned16(bias));
    const bool out4 = !out || ((ldo % 4 == 0) && aligned16(out));
    const bool outb4 = !out_bf16 || ((ldob % 4 == 0) && aligned8(out_bf16));
    // tfgk_spmm_bf16's ring condition (its rows4), with the fp32 out it would write
    const bool rows4 = (D % 4 == 0) && (ldh % 4 == 0) && aligned8(h) && out4 && in_aligned;
    const bool plan_on = rows4 && D >= 32 && D <= 512 && plan != nullptr && plan->n_tasks > 0;
    // width read per row: D, or D with its pad columns where that lets a ring run (the plan's scratch must hold them)
    const int32_t d8 = (D + 7) / 8 * 8, d4 = (D + 3) / 4 * 4;
    const bool scratch8 = !plan_on || plan->n_hubs == 0 || plan->scratch_bytes >= (size_t)plan->n_slots * d8 * sizeof(float);
    int32_t width = 0;                                   // 0: the scalar path
    if (ldh % 8 == 0 && ldh >= d8 && aligned16(h) && d8 >= 32 && d8 <= 256 && scratch8) width = d8;   // TMA ring
    else if (ldh % 4 == 0 && ldh >= d4 && aligned8(h) && d4 >= 32 && d4 <= 512) width = d4;            // cp.async ring
    cudaStream_t st = as_stream(stream);
    if (width > 0) {
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   0, width);
        p.hb = h;
        p.outb = out_bf16; p.ldob = ldob; p.d_store = D;
        p.io4 = D % 4 == 0 && out4 && outb4 && in_aligned;
        if (plan_on) use_plan(p, plan);
        const int rc = launch_spmm_tma4<6, uint16_t, true>(p, st);   // TFGK_ERR_UNSUPPORTED unless 16-byte rows, width <= 256
        if (rc != TFGK_ERR_UNSUPPORTED) return rc;
        return dispatch_spmm_async<uint16_t, true>(p, st);
    }
    for (int c0 = 0; c0 < D; c0 += 128) {               // scalar path: 32 lanes x 4 single columns per launch
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   c0, D - c0 < 128 ? D - c0 : 128);
        p.hb = h + c0;
        p.outb = out_bf16 ? out_bf16 + c0 : nullptr; p.ldob = ldob;
        const int rc = dispatch_spmm<1, uint16_t, true>(p, p.D, st);
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}

// fp8 rows (e4m3 bytes, exponents [N, ceil(D / 128)]).  The kernels are tfgk_spmm_bf16_dual's with a one-byte element:
// each element is widened to fp32 and scaled by 2^k of its row's group on its way out of shared memory (or global memory
// on the scalar path), then the fp32 arithmetic runs in the same order.  The plan is taken exactly where tfgk_spmm_f32
// takes it over the dequantised table with the same leading dimension, and every kernel sums rows without the plan
// strictly in CSR order, so the output is bit-identical to tfgk_spmm_f32 over x^ wherever both take the plan or neither
// does.  A table whose rows are 16-byte aligned with ldh >= D rounded up to 16, up to 256 columns, runs on the TMA ring,
// read with its pad columns (computed, never stored); every other shape takes the scalar path without the plan.
extern "C" int tfgk_spmm_fp8(const int64_t *rowptr, const int32_t *col, const float *w,
                             const uint8_t *h, int64_t ldh, const int8_t *h_exp, int32_t n_dst, int32_t D, int reduce,
                             float alpha, const float *addend, int64_t ld_addend, float beta,
                             const float *bias, int act,
                             float *out, int64_t ldo, const tfgk_plan *plan, void *stream) {
    bool nothing_to_do = true;
    const int vrc = spmm_validate(rowptr, h, ldh, n_dst, D, reduce, addend, ld_addend, act, out, ldo, plan, &nothing_to_do);
    if (vrc != TFGK_OK || nothing_to_do) return vrc;
    TFGK_CHECK_ARG(h_exp != nullptr, "spmm_fp8: null exponent array");
    const int32_t n_grp = (D + 127) / 128;
    TFGK_CHECK_ARG(n_grp == 1 || (reinterpret_cast<uintptr_t>(h_exp) & 1u) == 0, "spmm_fp8: exponents not 2-byte aligned");
    TFGK_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 3u) == 0, "spmm_fp8: misaligned out");

    const bool in_aligned = (!addend || ((ld_addend % 4 == 0) && aligned16(addend))) && (!bias || aligned16(bias));
    const bool out4 = (ldo % 4 == 0) && aligned16(out);
    // tfgk_spmm_f32's plan condition for the dequantised table (16-byte aligned fp32 rows, same ldh in elements)
    const bool plan_on = D % 4 == 0 && ldh % 4 == 0 && out4 && in_aligned && D >= 32 && D <= 512 && plan != nullptr &&
                         plan->n_tasks > 0;
    const int32_t d16 = (D + 15) / 16 * 16;
    cudaStream_t st = as_stream(stream);
    if (ldh % 16 == 0 && ldh >= d16 && aligned16(h) && d16 <= 256) {
        if (plan_on && plan->n_hubs > 0)
            TFGK_CHECK_ARG(plan->scratch != nullptr && plan->scratch_bytes >= (size_t)plan->n_slots * d16 * sizeof(float),
                           "spmm_fp8: plan scratch too small (need %zu bytes)", (size_t)plan->n_slots * d16 * sizeof(float));
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   0, d16);
        p.h8 = h; p.hexp = h_exp; p.n_grp = n_grp;
        p.d_store = D;
        p.io4 = D % 4 == 0 && out4 && in_aligned;
        if (plan_on) use_plan(p, plan);
        // 128-byte rows at D = 128: twelve stages keep as many bytes in flight per warp as six stages of bf16 rows
        return launch_spmm_tma4<12, uint8_t, true>(p, st);
    }
    for (int c0 = 0; c0 < D; c0 += 128) {               // scalar path: 32 lanes x 4 single columns = one group per launch
        SpmmParams p = spmm_params(rowptr, col, w, ldh, n_dst, reduce, alpha, addend, ld_addend, beta, bias, act, out, ldo,
                                   c0, D - c0 < 128 ? D - c0 : 128);
        p.h8 = h + c0; p.hexp = h_exp; p.n_grp = n_grp; p.grp0 = c0 / 128;
        const int rc = dispatch_spmm<1, uint8_t>(p, p.D, st);
        if (rc != TFGK_OK) return rc;
    }
    return TFGK_OK;
}
