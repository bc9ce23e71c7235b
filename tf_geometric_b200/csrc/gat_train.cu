// Backward pass of the fused GAT aggregation without the [E, H] coefficient table (round 2).
//
// The reference obtains these gradients from TensorFlow autodiff over nn/conv/gat.py:73-114 (demo/demo_gat.py).  Round 1
// kept the attention coefficients of the forward pass ([E', H] floats, which forced the slower register-staged forward
// kernel), then ran a softmax-backward kernel and three per-head aggregations.  Here the forward pass is the streaming
// cp.async kernel and keeps only (max, denominator) per (row, head); the backward pass RECOMPUTES every coefficient from
// Q, K and those two numbers - the FlashAttention recipe applied to an edge list:
//
//   a_e,h   = exp(<Q_r,h, K_c,h> / scale - m_r,h) / den_r,h                       (r = row_e, c = col_e)
//   delta_r,h = sum_e a_e,h <G_r,h, V_c,h> = <G_r,h, out_r,h>                        (out = aggregate before bias / activation)
//   ds_e,h  = a_e,h (<G_r,h, V_c,h> - delta_r,h)
//   dQ_r = (1/scale) sum_{e: row_e = r} ds_e K_c          pass 1, forward CSR, gathers K | V rows
//   dK_c = (1/scale) sum_{e: col_e = c} ds_e Q_r          pass 2, transposed CSR, gathers Q and G|stats rows
//   dV_c =             sum_{e: col_e = c} a_e  G_r
//
// tfgk_gat_bwd_prepare_f32 masks the upstream gradient with the activation, computes delta and packs
// [G (A floats) | m (8) | den (8) | delta (8) | pad (8)] per row so that pass 2 fetches everything it needs about a
// destination with one 640-byte gather.  Both passes reuse the edge-streaming cp.async ring of the forward kernels.
// Limits of this path (the caller falls back to the coefficient-table path otherwise): heads concatenated, dqk == dv,
// A = H * dqk <= 128, H <= 8 (gat_recompute_shape in common.cuh, which the stats forward checks too), no hub-row plan.
#include "common.cuh"

namespace tfgk {

constexpr int kBwdRows = 32;
constexpr int kBwdWarps = 4;
constexpr int kStatFloats = 32;          // [m(8) | den(8) | delta(8) | pad(8)]

__device__ __forceinline__ void bwd_cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ float4 bwd_ldg4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }

struct GatBwdParams {
    const int64_t *rowptr;
    const int32_t *col;
    const float *Q; int64_t ldq;
    const float *K; int64_t ldk;
    const float *V; int64_t ldv;
    const float *GS; int64_t ldgs;       // [N, A + 32]
    int32_t N, H, dqk;
    float scale;
    float *dQ; int64_t lddq;
    float *dK; int64_t lddk;
    float *dV; int64_t lddv;
};

// one warp per row: g_masked, delta and the packed row
__global__ void __launch_bounds__(256) gat_bwd_prepare_kernel(const float *__restrict__ G, int64_t ldg, const float *__restrict__ Y,
                                                              int64_t ldy, const float *__restrict__ bias, int act,
                                                              const float *__restrict__ stats, int32_t N, int32_t H, int32_t dqk,
                                                              float *__restrict__ GS, int64_t ldgs) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (r >= N) return;
    const int A = H * dqk, lph = dqk >> 2, ccol = lane * 4;
    float d = 0.0f;
    if (ccol < A) {
        float4 g = bwd_ldg4(G + r * ldg + ccol);
        const float4 y = bwd_ldg4(Y + r * ldy + ccol);
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (bias) b = bwd_ldg4(bias + ccol);
        if (act == TFGK_ACT_RELU) {           // dL/d(pre-activation): relu'(y) = [y > 0]
            g.x = y.x > 0.0f ? g.x : 0.0f; g.y = y.y > 0.0f ? g.y : 0.0f;
            g.z = y.z > 0.0f ? g.z : 0.0f; g.w = y.w > 0.0f ? g.w : 0.0f;
        }
        // aggregate before bias: out = y - b wherever the gradient survives (relu passes y = out + b > 0 through unchanged).
        // y - b is exact, but y = fl(out + b) kept out only to 2^-24 |y|: about 24 - log2(|b| / |out|) bits of out survive
        // (17 at |b| = 100 |out|, checked in tests/test_gpu_gat_backward.py)
        d = g.x * (y.x - b.x) + g.y * (y.y - b.y) + g.z * (y.z - b.z) + g.w * (y.w - b.w);
        *reinterpret_cast<float4 *>(GS + r * ldgs + ccol) = g;
    }
    for (int off = 1; off < lph; off <<= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
    if (ccol < A && (lane % lph) == 0) {
        const int h = lane / lph;
        GS[r * ldgs + A + h] = stats[r * 2 * H + h];
        GS[r * ldgs + A + 8 + h] = stats[r * 2 * H + H + h];
        GS[r * ldgs + A + 16 + h] = d;
    }
}

// MODE 0: rows = destinations (forward CSR), gathers K[c] | V[c], produces dQ.
// MODE 1: rows = sources (transposed CSR), gathers Q[r] | GS[r], produces dK and dV.
template <int MODE, int U, int S>
__global__ void __launch_bounds__(kBwdWarps * 32) gat_bwd_kernel(const GatBwdParams p) {
    static_assert(32 % U == 0, "a round must not straddle an index chunk");
    constexpr int RPC = 32 / U;
    static_assert(S <= RPC, "index chunk refill assumes the prologue stays inside chunk 0");
    extern __shared__ __align__(16) uint8_t bwd_ring[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t r0 = ((int64_t)blockIdx.x * kBwdWarps + warp) * kBwdRows;
    if (r0 >= p.N) return;
    const int64_t r1 = min((int64_t)p.N, r0 + kBwdRows);
    const int64_t e_begin = p.rowptr[r0], e_stop = p.rowptr[r1];
    const int64_t rp_hi = p.rowptr[min(r0 + lane + 1, r1)];
    const int n_edges = (int)(e_stop - e_begin);
    const int n_rounds = (n_edges + U - 1) / U;
    const int A = p.H * p.dqk, lph = p.dqk >> 2;
    const int ccol = lane * 4;
    const bool cok = ccol < A;
    const int head = min(lane / lph, p.H - 1);
    const uint32_t row_bytes = (uint32_t)A * 4u;
    // per edge: MODE 0 [K row | V row];  MODE 1 [Q row | G row | 32 stat floats]
    const uint32_t edge_bytes = MODE == 0 ? 2u * row_bytes : 2u * row_bytes + kStatFloats * 4u;
    const uint32_t stage_bytes = U * edge_bytes;
    uint8_t *my_ring = bwd_ring + (size_t)warp * S * stage_bytes;
    const uint32_t ring_addr = (uint32_t)__cvta_generic_to_shared(my_ring);
    const float inv_scale = 1.0f / p.scale;

    int64_t r = r0;
    int row_end = (int)(__shfl_sync(0xffffffffu, rp_hi, 0) - e_begin);
    // row-local operands: MODE 0: q, g, (m, den, delta);  MODE 1: k, v
    float4 la = make_float4(0.f, 0.f, 0.f, 0.f), lb = la;
    float m_r = 0.f, den_r = 1.f, delta_r = 0.f;
    auto load_row = [&](int64_t row) {
        if (row >= r1) return;
        if (MODE == 0) {
            if (cok) {
                la = bwd_ldg4(p.Q + row * p.ldq + ccol);
                lb = bwd_ldg4(p.GS + row * p.ldgs + ccol);
            }
            m_r = __ldg(p.GS + row * p.ldgs + A + head);
            den_r = __ldg(p.GS + row * p.ldgs + A + 8 + head);
            delta_r = __ldg(p.GS + row * p.ldgs + A + 16 + head);
        } else if (cok) {
            la = bwd_ldg4(p.K + row * p.ldk + ccol);
            lb = bwd_ldg4(p.V + row * p.ldv + ccol);
        }
    };
    load_row(r);
    float x0 = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f;      // dQ (MODE 0) or dK (MODE 1)
    float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;      // dV (MODE 1)

    auto finalize_row = [&]() {
        if (cok) {
            if (MODE == 0) {
                *reinterpret_cast<float4 *>(p.dQ + r * p.lddq + ccol) = make_float4(x0 * inv_scale, x1 * inv_scale, x2 * inv_scale, x3 * inv_scale);
            } else {
                *reinterpret_cast<float4 *>(p.dK + r * p.lddk + ccol) = make_float4(x0 * inv_scale, x1 * inv_scale, x2 * inv_scale, x3 * inv_scale);
                *reinterpret_cast<float4 *>(p.dV + r * p.lddv + ccol) = make_float4(y0, y1, y2, y3);
            }
        }
        x0 = x1 = x2 = x3 = 0.f;
        y0 = y1 = y2 = y3 = 0.f;
        ++r;
        if (r < r1) {
            row_end = (int)(__shfl_sync(0xffffffffu, rp_hi, (int)(r - r0)) - e_begin);
            load_row(r);
        }
    };
    auto load_chunk = [&](int c) {
        const int e = c * 32 + lane;
        return e < n_edges ? ld_stream_i32(p.col + e_begin + e) : 0;
    };
    auto issue = [&](int g, int ci) {
        if (g < n_rounds) {
            const int base = (g % RPC) * U;
            const uint32_t dst0 = ring_addr + (uint32_t)(g % S) * stage_bytes;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int c = __shfl_sync(0xffffffffu, ci, base + u);
                if (g * U + u < n_edges) {
                    const uint32_t dst = dst0 + (uint32_t)u * edge_bytes;
                    if (MODE == 0) {
                        if (cok) {
                            bwd_cp_async16(dst + ccol * 4, p.K + (int64_t)c * p.ldk + ccol);
                            bwd_cp_async16(dst + row_bytes + ccol * 4, p.V + (int64_t)c * p.ldv + ccol);
                        }
                    } else {
                        if (cok) {
                            bwd_cp_async16(dst + ccol * 4, p.Q + (int64_t)c * p.ldq + ccol);
                            bwd_cp_async16(dst + row_bytes + ccol * 4, p.GS + (int64_t)c * p.ldgs + ccol);
                        }
                        if (lane < kStatFloats / 4)
                            bwd_cp_async16(dst + 2u * row_bytes + lane * 16, p.GS + (int64_t)c * p.ldgs + A + lane * 4);
                    }
                }
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    int ca = load_chunk(0), cb = load_chunk(1);
#pragma unroll
    for (int g = 0; g < S - 1; ++g) issue(g, ca);

    for (int g = 0; g < n_rounds; ++g) {
        {
            const int gn = g + S - 1;
            issue(gn, ((gn / RPC) & 1) ? cb : ca);
        }
        asm volatile("cp.async.wait_group %0;" ::"n"(S - 1) : "memory");
        if (MODE == 1) __syncwarp();             // the stat floats were copied by lanes 0-7 and are read by every lane
        const uint8_t *sbuf = my_ring + (size_t)(g % S) * stage_bytes;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int e = g * U + u;
            if (e < n_edges) {
                while (e == row_end) finalize_row();
                const uint8_t *eb = sbuf + (size_t)u * edge_bytes;
                float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), gb = ga;
                if (cok) {
                    ga = *reinterpret_cast<const float4 *>(eb + ccol * 4);
                    gb = *reinterpret_cast<const float4 *>(eb + row_bytes + ccol * 4);
                }
                float m = m_r, dn = den_r, dl = delta_r;
                if (MODE == 1) {
                    const float *st = reinterpret_cast<const float *>(eb + 2u * row_bytes);
                    m = st[head]; dn = st[8 + head]; dl = st[16 + head];
                }
                // MODE 0: la = q_r, lb = g_r, ga = k_c, gb = v_c;  MODE 1: la = k_c, lb = v_c, ga = q_r, gb = g_r
                float d = la.x * ga.x + la.y * ga.y + la.z * ga.z + la.w * ga.w;                    // <q, k>
                float da = MODE == 0 ? lb.x * gb.x + lb.y * gb.y + lb.z * gb.z + lb.w * gb.w        // <g, v>
                                     : gb.x * lb.x + gb.y * lb.y + gb.z * lb.z + gb.w * lb.w;
                for (int off = 1; off < lph; off <<= 1) {
                    d += __shfl_xor_sync(0xffffffffu, d, off);
                    da += __shfl_xor_sync(0xffffffffu, da, off);
                }
                const float s = __fdiv_rn(d, p.scale);
                const float a = __fdiv_rn(expf(s - m), dn);
                const float ds = a * (da - dl);
                x0 = fmaf(ds, ga.x, x0); x1 = fmaf(ds, ga.y, x1); x2 = fmaf(ds, ga.z, x2); x3 = fmaf(ds, ga.w, x3);
                if (MODE == 1) {
                    y0 = fmaf(a, gb.x, y0); y1 = fmaf(a, gb.y, y1); y2 = fmaf(a, gb.z, y2); y3 = fmaf(a, gb.w, y3);
                }
            }
        }
        if (MODE == 1) __syncwarp();             // all lanes are done with the stage before lanes 0-7 overwrite its stat floats
        if ((g + S) % RPC == 0) {
            const int dead = (g + S) / RPC - 1;
            if (dead & 1) cb = load_chunk(dead + 2); else ca = load_chunk(dead + 2);
        }
    }
    while (r < r1) finalize_row();
}

template <int MODE>
static int launch_gat_bwd(const GatBwdParams &p, cudaStream_t st) {
    constexpr int U = 2, S = 3;
    const size_t edge_bytes = (size_t)2 * p.H * p.dqk * 4 + (MODE == 1 ? kStatFloats * 4 : 0);
    const size_t smem = (size_t)kBwdWarps * S * U * edge_bytes;
    static int configured[2][16] = {{0}};
    int dev = 0;
    TFGK_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 16 || configured[MODE][dev] < (int)smem) {
        TFGK_CUDA(cudaFuncSetAttribute(gat_bwd_kernel<MODE, U, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (dev >= 0 && dev < 16) configured[MODE][dev] = (int)smem;
    }
    const unsigned blocks = (unsigned)ceil_div64(ceil_div64(p.N, kBwdRows), kBwdWarps);
    gat_bwd_kernel<MODE, U, S><<<blocks, kBwdWarps * 32, smem, st>>>(p);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

static int check_bwd_shape(int32_t N, int32_t H, int32_t dqk) {
    if (N < 0 || H < 1 || dqk < 1) return set_error(TFGK_ERR_INVALID_ARGUMENT, "gat_bwd: bad size (N=%d H=%d dqk=%d)", N, H, dqk);
    if (!gat_recompute_shape(H, dqk)) return TFGK_ERR_UNSUPPORTED;
    return TFGK_OK;
}

}  // namespace tfgk

using namespace tfgk;

extern "C" int tfgk_gat_bwd_prepare_f32(const float *G, int64_t ldg, const float *Y, int64_t ldy, const float *bias, int act,
                                        const float *stats, int32_t N, int32_t H, int32_t dqk, float *GS, int64_t ldgs,
                                        void *stream) {
    const int rc = check_bwd_shape(N, H, dqk);
    if (rc != TFGK_OK) return rc;
    if (N == 0) return TFGK_OK;
    const int A = H * dqk;
    TFGK_CHECK_ARG(G && Y && stats && GS, "gat_bwd_prepare: null pointer");
    TFGK_CHECK_ARG(act == TFGK_ACT_NONE || act == TFGK_ACT_RELU, "gat_bwd_prepare: unknown activation %d", act);
    TFGK_CHECK_ARG(ldg >= A && ldy >= A && ldgs >= A + kStatFloats, "gat_bwd_prepare: leading dimension too small");
    if (ldg % 4 || ldy % 4 || ldgs % 4 || !aligned16(G) || !aligned16(Y) || !aligned16(GS) || (bias && !aligned16(bias)))
        return TFGK_ERR_UNSUPPORTED;
    gat_bwd_prepare_kernel<<<(unsigned)ceil_div64(N, 8), 256, 0, as_stream(stream)>>>(G, ldg, Y, ldy, bias, act, stats, N, H, dqk, GS, ldgs);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

extern "C" int tfgk_gat_bwd_dst_f32(const int64_t *rowptr, const int32_t *col, const float *Q, int64_t ldq,
                                    const float *K, int64_t ldk, const float *V, int64_t ldv, const float *GS, int64_t ldgs,
                                    int32_t N, int32_t H, int32_t dqk, float scale, float *dQ, int64_t lddq, void *stream) {
    const int rc = check_bwd_shape(N, H, dqk);
    if (rc != TFGK_OK) return rc;
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && col && Q && K && V && GS && dQ && scale > 0.0f, "gat_bwd_dst: bad argument");
    if (ldq % 4 || ldk % 4 || ldv % 4 || ldgs % 4 || lddq % 4 || !aligned16(Q) || !aligned16(K) || !aligned16(V) || !aligned16(GS) ||
        !aligned16(dQ))
        return TFGK_ERR_UNSUPPORTED;
    GatBwdParams p;
    p.rowptr = rowptr; p.col = col; p.Q = Q; p.ldq = ldq; p.K = K; p.ldk = ldk; p.V = V; p.ldv = ldv; p.GS = GS; p.ldgs = ldgs;
    p.N = N; p.H = H; p.dqk = dqk; p.scale = scale; p.dQ = dQ; p.lddq = lddq; p.dK = nullptr; p.lddk = 0; p.dV = nullptr; p.lddv = 0;
    return launch_gat_bwd<0>(p, as_stream(stream));
}

extern "C" int tfgk_gat_bwd_src_f32(const int64_t *rowptr_t, const int32_t *col_t, const float *Q, int64_t ldq,
                                    const float *K, int64_t ldk, const float *V, int64_t ldv, const float *GS, int64_t ldgs,
                                    int32_t N, int32_t H, int32_t dqk, float scale, float *dK, int64_t lddk, float *dV, int64_t lddv,
                                    void *stream) {
    const int rc = check_bwd_shape(N, H, dqk);
    if (rc != TFGK_OK) return rc;
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr_t && col_t && Q && K && V && GS && dK && dV && scale > 0.0f, "gat_bwd_src: bad argument");
    if (ldq % 4 || ldk % 4 || ldv % 4 || ldgs % 4 || lddk % 4 || lddv % 4 || !aligned16(Q) || !aligned16(K) || !aligned16(V) ||
        !aligned16(GS) || !aligned16(dK) || !aligned16(dV))
        return TFGK_ERR_UNSUPPORTED;
    GatBwdParams p;
    p.rowptr = rowptr_t; p.col = col_t; p.Q = Q; p.ldq = ldq; p.K = K; p.ldk = ldk; p.V = V; p.ldv = ldv; p.GS = GS; p.ldgs = ldgs;
    p.N = N; p.H = H; p.dqk = dqk; p.scale = scale; p.dQ = nullptr; p.lddq = 0; p.dK = dK; p.lddk = lddk; p.dV = dV; p.lddv = lddv;
    return launch_gat_bwd<1>(p, as_stream(stream));
}
