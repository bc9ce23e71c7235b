// K4: the dense projections of the hot path on the Hopper tensor cores (wgmma), as ONE launch over several column blocks,
// optionally with the A operand gathered tile by tile from other GPUs' memory (fused all-gather -> GEMM over NVLink peer
// mappings, K5).
//
//   C_b[M, n_b] = act_b(A[M, K] @ W_b[K, n_b] + bias_b)     for b in 0..nb-1  (n_b <= 128, nb <= 4)
//
// replaces x@W at nn/conv/gcn.py:272 and the three projections x@Wq, x@Wk, x@W of nn/conv/gat.py:52,61,70, which would
// otherwise be three launches that each re-read x.  tfgk_gemm_f32 sends every tall projection here as well.
//
// Arithmetic: 3xTF32.  a = a_hi + a_lo and w = w_hi + w_lo with x_hi = rna_tf32(x) kept finite, and per k-step of 8
//     acc += a_lo * w_hi;  acc += a_hi * w_lo;  acc += a_hi * w_hi        (wgmma.m64n128k8.f32.tf32.tf32, fp32 accumulators)
// which keeps the error at the fp32 level, where a single TF32 pass is off by ~1e-3: every entry is within
// (K 2^-23 + 2^-19) S + 2^-23 |ref| of float64, S = |A| |W| + |bias| (tests/test_gpu_gemm_contract.py, every K up to the
// limit of 184 set by the shared-memory plan below).  The result of a row depends only on that row, the weights and K: the
// same bits whatever the number of blocks, the grid or the part layout of A.
//
// Layout (one CTA = 128 output rows x one column block of <= 128 columns, 256 threads = two warpgroups of 64 rows):
//   * W_b (hi | lo) resident in shared memory for the whole kernel, K rounded up to 8, in the K-major no-swizzle layout of
//     the wgmma descriptors: 8 x 16-byte core matrices, LBO = 128 B along K, SBO = 32 * Kpad bytes along N;
//   * A streams through a cp.async ring of BK = 32 columns per stage (rows padded to 36 floats: the fragment loads hit 32
//     distinct banks); each thread splits its own A fragment into hi / lo in registers, so A never goes back to shared memory
//     and the wgmma reads A from registers and W through the descriptors.  The fragments live in two register sets, so the
//     wait for the MMAs of k-block j comes after k-block j + 1 has been loaded and split into the other set (ptxas adds
//     warpgroup.arrive fences around the register operands; measured, this is 3-4 % faster than waiting after every
//     k-block, DESIGN.md section 4);
//   * persistent CTAs: CTA b handles block b % nb for the row tiles of its group b / nb; the nb CTAs of a group walk the
//     same tiles in the same order, so x is read from HBM once and from L2 nb-1 times.  The ring runs across tile
//     boundaries, so the loads of the next tile overlap the epilogue of the current one;
//   * A may be split into `n_parts` row blocks living at different base pointers (the other ranks' copies of x, mapped
//     through CUDA IPC): the cp.async then read straight over NVLink, tile by tile.  Tiles are walked starting at the tile
//     of part `first_part`, so that every rank pulls from a different peer at any moment.
#include "common.cuh"
#include <cuda_bf16.h>
#include <type_traits>

namespace tfgk {
namespace proj {

constexpr int BM = 128;                  // rows per tile (two warpgroups x 64)
constexpr int BK = 32;                   // A columns per ring stage
constexpr int kUN = 128;                 // output columns per CTA
constexpr int kThreads = 256;
constexpr int kApitch = BK + 4;          // floats per A row in a stage
constexpr int kStageBytes = BM * kApitch * 4;
constexpr int kMaxBlocks = 4;
constexpr int kMaxParts = 8;

struct Params {
    const float *A[kMaxParts];
    int64_t lda, part_rows;
    int first_tile;
    int M, K, kpad, nb, tiles_m, n_groups;
    const float *B[kMaxBlocks]; int64_t ldb[kMaxBlocks];
    const float *bias[kMaxBlocks]; int act[kMaxBlocks]; int ncols[kMaxBlocks]; int transb[kMaxBlocks];
    void *C[kMaxBlocks]; int64_t ldc[kMaxBlocks];
    int c_kind[kMaxBlocks];            // 0: fp32 C; 1: bf16 C, rounded to nearest even; 2: e4m3 C with exponents in E
    int8_t *E[kMaxBlocks]; int64_t lde[kMaxBlocks];
};

// shared memory: W hi | W lo | bias | ring of A stages.  With 1024 bytes of W per K (rounded up to 8), 18 432 per A stage
// and 227 KB in all: 4 stages for K <= 152, 3 for K 153..168, 2 for K 169..184, none (unsupported) from K = 185 on
struct Plan {
    uint32_t kpad, b_bytes, ring_off, stages, total;
    explicit Plan(int K) {
        kpad = (uint32_t)((K + 7) / 8) * 8;
        b_bytes = (uint32_t)kUN * kpad * 4u;
        ring_off = 2u * b_bytes + kUN * 4u;
        const uint32_t budget = 227u * 1024u;
        stages = 0;
        for (uint32_t st = 4; st >= 2; --st)
            if (ring_off + st * kStageBytes <= budget) { stages = st; break; }
        total = ring_off + stages * kStageBytes;
    }
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// byte offset of W[k][n] in the K-major core-matrix layout (8 rows of n x 16 bytes of k per core matrix)
__device__ __forceinline__ uint32_t w_offset(int n, int k, int kpad) {
    return (uint32_t)(n >> 3) * (uint32_t)(kpad * 32) + (uint32_t)(k >> 2) * 128u + (uint32_t)(n & 7) * 16u + (uint32_t)(k & 3) * 4u;
}

// wgmma shared-memory descriptor: K-major, no swizzle, LBO = 128 B (next core matrix along K), SBO (next 8 rows along N)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);          // start address,       bits [0,14)
    d |= (uint64_t)(128u >> 4) << 16;                  // leading byte offset, bits [16,30)
    d |= (uint64_t)(sbo_bytes >> 4) << 32;             // stride byte offset,  bits [32,46)
    return d;                                          // base offset 0, layout type 0 (no swizzle)
}

// hi = rna_tf32(a) (round half away from zero to 10 mantissa bits: add half a TF32 ulp to the magnitude bits, truncate),
// of a first clamped to +-0x7F7FEFFF, the largest magnitude that rounds to a finite TF32 number (2 - 2^-10) 2^127.  Without
// the clamp |a| >= (2 - 2^-11) 2^127 would round to inf and a = +-inf would give lo = inf - inf = NaN.  With it,
// lo = a - hi is finite for every finite a, +-inf for a = +-inf and NaN for a NaN (fmaxf takes the number), so the
// products give the IEEE result.  Every a below the threshold gets the bits of cvt.rna.tf32.f32, in as many instructions
// (two FMNMX instead of the inf test and select that cvt.rna, or .satfinite on top of it, compiles to).
__device__ __forceinline__ void split_tf32(float a, uint32_t &hi, uint32_t &lo) {
    const float lim = __uint_as_float(0x7F7FEFFFu);
    hi = (__float_as_uint(fminf(fmaxf(a, -lim), lim)) + 0x1000u) & 0xFFFFE000u;
    lo = __float_as_uint(a - __uint_as_float(hi));
}

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 128] (+)= A[64 x 8] (registers, tf32) * B[8 x 128] (shared memory descriptor, tf32); accumulate == 0 overwrites D
__device__ __forceinline__ void wgmma_m64n128k8(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ int tile_index(const Params &p, int group, int it) {
    int tl = group + it * p.n_groups + p.first_tile;
    return tl >= p.tiles_m ? tl - p.tiles_m : tl;
}

template <int STAGES>
__global__ void __launch_bounds__(kThreads, 1) gemm_proj_kernel(const Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cb = blockIdx.x % p.nb, group = blockIdx.x / p.nb;
    const int kpad = p.kpad;
    const uint32_t b_bytes = (uint32_t)kUN * kpad * 4u;
    uint8_t *w_hi = smem, *w_lo = smem + b_bytes;
    float *s_bias = reinterpret_cast<float *>(smem + 2 * b_bytes);
    uint8_t *ring = smem + 2 * b_bytes + kUN * 4;
    const uint32_t ring_addr = smem_u32(ring);

    const int ncols = p.ncols[cb];
    const int my_tiles = group < p.tiles_m ? (p.tiles_m - group + p.n_groups - 1) / p.n_groups : 0;
    const int kb_per_tile = (p.K + BK - 1) / BK;
    const int total = my_tiles * kb_per_tile;

    // A k-block j of this CTA (tile j / kb_per_tile) -> ring stage j % STAGES; rows beyond M and columns beyond K are zeros
    // (a tile never straddles two parts: part_rows is a multiple of BM)
    auto load_stage = [&](int j) {
        if (j < total) {
            const int64_t row0 = (int64_t)tile_index(p, group, j / kb_per_tile) * BM;
            const int part = (int)(row0 / p.part_rows);
            const float *a_tile = p.A[part] + (row0 - (int64_t)part * p.part_rows) * p.lda;
            const int rows = (int)min((int64_t)BM, (int64_t)p.M - row0);
            const int k0 = (j % kb_per_tile) * BK;
            const uint32_t dst0 = ring_addr + (uint32_t)(j % STAGES) * kStageBytes;
            const int ch = tid & 7, gk = k0 + ch * 4;
            const uint32_t bytes = gk < p.K ? (uint32_t)min(16, (p.K - gk) * 4) : 0u;
#pragma unroll
            for (int i = 0; i < (BM * BK / 4) / kThreads; ++i) {
                const int r = (tid >> 3) + i * (kThreads / 8);
                const bool ok = r < rows && bytes != 0;
                cp_async16_zfill(dst0 + (uint32_t)(r * kApitch + ch * 4) * 4u, ok ? a_tile + (int64_t)r * p.lda + gk : p.A[0],
                                 ok ? bytes : 0u);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) load_stage(s);

    {   // W_b: split into hi / lo, once per CTA; columns beyond n_b and rows beyond K are zeros
        const float *B = p.B[cb];
        const int64_t ldb = p.ldb[cb];
        const bool tb = p.transb[cb] != 0;
        for (int idx = tid; idx < kUN * kpad; idx += kThreads) {
            int n, k;
            if (tb) { n = idx / kpad; k = idx % kpad; } else { k = idx / kUN; n = idx % kUN; }     // coalesced reads of B
            const float w = (n < ncols && k < p.K) ? (tb ? B[(int64_t)n * ldb + k] : B[(int64_t)k * ldb + n]) : 0.0f;
            uint32_t hi, lo;
            split_tf32(w, hi, lo);
            const uint32_t off = w_offset(n, k, kpad);
            *reinterpret_cast<uint32_t *>(w_hi + off) = hi;
            *reinterpret_cast<uint32_t *>(w_lo + off) = lo;
        }
        if (tid < kUN) s_bias[tid] = (p.bias[cb] != nullptr && tid < ncols) ? p.bias[cb][tid] : 0.0f;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores of W -> visible to wgmma
    __syncthreads();

    const uint32_t w_hi_addr = smem_u32(w_hi), w_lo_addr = smem_u32(w_lo), sbo = (uint32_t)kpad * 32u;
    // fragment coordinates: warpgroup wg owns rows [64 wg, 64 wg + 64), warp w of it rows 16 w .. 16 w + 15
    const int frag_row = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
    const int frag_col = lane & 3;
    const int act = p.act[cb];
    float *C = static_cast<float *>(p.C[cb]);
    __nv_bfloat16 *Cb = static_cast<__nv_bfloat16 *>(p.C[cb]);
    const bool c_bf16 = p.c_kind[cb] == 1;
    const bool c_fp8 = p.c_kind[cb] == 2;
    const int64_t ldc = p.ldc[cb];
    // (col, col + 1) as one 8-byte store (fp32), one 4-byte store (bf16) or one 2-byte store (fp8)
    const bool vec2 = (ldc % 2) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.C[cb]) & (c_fp8 ? 1u : c_bf16 ? 3u : 7u)) == 0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;

    // A fragments (m16n8k8 layout per warp) of the stage's four k-steps, split into hi / lo, in two register sets: the MMAs of
    // stage j - 1 read one set while stage j loads and splits into the other, and are waited for only then
    uint32_t ah[2][BK / 8][4], al[2][BK / 8][4];
    auto stage = [&](auto parity, int j) {
        constexpr int P = decltype(parity)::value;
        asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 2) : "memory");
        __syncthreads();                          // stage j landed for every thread; stage j - 1 is no longer read
        load_stage(j + STAGES - 1);
        const int kb = j % kb_per_tile;
        const float *As = reinterpret_cast<const float *>(ring + (size_t)(j % STAGES) * kStageBytes);
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
            const float *a_r0 = As + frag_row * kApitch + ks * 8 + frag_col;
            const float *a_r8 = a_r0 + 8 * kApitch;
            split_tf32(a_r0[0], ah[P][ks][0], al[P][ks][0]);
            split_tf32(a_r8[0], ah[P][ks][1], al[P][ks][1]);
            split_tf32(a_r0[4], ah[P][ks][2], al[P][ks][2]);
            split_tf32(a_r8[4], ah[P][ks][3], al[P][ks][3]);
        }
        wgmma_wait_all();                         // the MMAs of stage j - 1 (the other register set) have retired
        wgmma_fence();                            // wgmma may only read registers written before the fence
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
            const int kg = kb * BK + ks * 8;
            if (kg < kpad) {                      // block-uniform: skips the k-steps beyond K rounded up to 8
                const uint32_t koff = (uint32_t)(kg >> 2) * 128u;
                const uint64_t dh = make_desc(w_hi_addr + koff, sbo), dl = make_desc(w_lo_addr + koff, sbo);
                wgmma_m64n128k8(acc, al[P][ks], dh, (kb | ks) != 0);
                wgmma_m64n128k8(acc, ah[P][ks], dl, 1u);
                wgmma_m64n128k8(acc, ah[P][ks], dh, 1u);
            }
        }
        wgmma_commit();
        if (kb == kb_per_tile - 1) {              // epilogue of the tile: + bias -> act -> C
            wgmma_wait_all();
            const int64_t row0 = (int64_t)tile_index(p, group, j / kb_per_tile) * BM + frag_row;
            if (c_fp8) {                          // block-uniform: a row's columns sit in the four threads of a quad
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t row = row0 + 8 * h;
                    float m = 0.0f;
#pragma unroll
                    for (int nb8 = 0; nb8 < kUN / 8; ++nb8) {
                        const int col = nb8 * 8 + 2 * frag_col;
                        if (col < ncols) m = fp8_amax(m, apply_act(acc[4 * nb8 + 2 * h] + s_bias[col], act));
                        if (col + 1 < ncols) m = fp8_amax(m, apply_act(acc[4 * nb8 + 2 * h + 1] + s_bias[col + 1], act));
                    }
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                    const int k = fp8_exponent(m);
                    const float inv = pow2i(-k);
                    if (row < p.M) {
                        uint8_t *crow = static_cast<uint8_t *>(p.C[cb]) + row * ldc;
#pragma unroll
                        for (int nb8 = 0; nb8 < kUN / 8; ++nb8) {
                            const int col = nb8 * 8 + 2 * frag_col;
                            const float v0 = apply_act(acc[4 * nb8 + 2 * h] + s_bias[col], act);
                            const float v1 = apply_act(acc[4 * nb8 + 2 * h + 1] + s_bias[col + 1], act);
                            const uint32_t q = fp8_pack2(v0, v1, inv);
                            if (vec2 && col + 1 < ncols) {
                                *reinterpret_cast<uint16_t *>(crow + col) = (uint16_t)q;
                            } else {
                                if (col < ncols) crow[col] = (uint8_t)(q & 0xFFu);
                                if (col + 1 < ncols) crow[col + 1] = (uint8_t)(q >> 8);
                            }
                        }
                        if (frag_col == 0) p.E[cb][row * p.lde[cb]] = (int8_t)k;
                    }
                }
            } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int64_t row = row0 + 8 * h;
                if (row < p.M && c_bf16) {        // block-uniform: the fp32 value, rounded once
                    __nv_bfloat16 *crow = Cb + row * ldc;
#pragma unroll
                    for (int nb8 = 0; nb8 < kUN / 8; ++nb8) {
                        const int col = nb8 * 8 + 2 * frag_col;
                        const float v0 = apply_act(acc[4 * nb8 + 2 * h] + s_bias[col], act);
                        const float v1 = apply_act(acc[4 * nb8 + 2 * h + 1] + s_bias[col + 1], act);
                        if (vec2 && col + 1 < ncols) {
                            *reinterpret_cast<__nv_bfloat162 *>(crow + col) = __floats2bfloat162_rn(v0, v1);
                        } else {
                            if (col < ncols) crow[col] = __float2bfloat16_rn(v0);
                            if (col + 1 < ncols) crow[col + 1] = __float2bfloat16_rn(v1);
                        }
                    }
                } else if (row < p.M) {
                    float *crow = C + row * ldc;
#pragma unroll
                    for (int nb8 = 0; nb8 < kUN / 8; ++nb8) {
                        const int col = nb8 * 8 + 2 * frag_col;
                        const float v0 = apply_act(acc[4 * nb8 + 2 * h] + s_bias[col], act);
                        const float v1 = apply_act(acc[4 * nb8 + 2 * h + 1] + s_bias[col + 1], act);
                        if (vec2 && col + 1 < ncols) {
                            *reinterpret_cast<float2 *>(crow + col) = make_float2(v0, v1);
                        } else {
                            if (col < ncols) crow[col] = v0;
                            if (col + 1 < ncols) crow[col + 1] = v1;
                        }
                    }
                }
            }
            }
        }
    };
    for (int j = 0; j < total; j += 2) {
        stage(std::integral_constant<int, 0>(), j);
        if (j + 1 < total) stage(std::integral_constant<int, 1>(), j + 1);
    }
    wgmma_wait_all();
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

template <int STAGES>
static int launch(const Params &p, int grid, uint32_t smem_bytes, cudaStream_t st) {
    TFGK_CUDA(ensure_dynamic_smem(gemm_proj_kernel<STAGES>, smem_bytes));
    gemm_proj_kernel<STAGES><<<grid, kThreads, smem_bytes, st>>>(p);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

// dst = bf16(src), round to nearest even, for the projections tfgk_gemm_proj_mixed cannot take (fp32 GEMM, then this)
__global__ void __launch_bounds__(256) round_bf16_kernel(const float *src, int64_t lds, int32_t rows, int32_t cols,
                                                         __nv_bfloat16 *dst, int64_t ldd) {
    const int64_t n = (int64_t)rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols, c = i % cols;
        dst[r * ldd + c] = __float2bfloat16_rn(src[r * lds + c]);
    }
}

// dst = e4m3(src) with one exponent per row and group of 128 columns, for the projections tfgk_gemm_proj_fp8 cannot take;
// one warp per (row, group), four columns a lane: the same exponent rule and rounding as the K4 epilogue
__global__ void __launch_bounds__(256) quantize_fp8_kernel(const float *src, int64_t lds, int32_t rows, int32_t cols,
                                                           uint8_t *dst, int64_t ldd, int8_t *exps, int64_t lde) {
    const int lane = threadIdx.x & 31;
    const int n_grp = (cols + 127) / 128;
    const int64_t n_tasks = (int64_t)rows * n_grp;
    for (int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; t < n_tasks;
         t += (int64_t)gridDim.x * blockDim.x / 32) {
        const int64_t r = t / n_grp;
        const int g = (int)(t % n_grp);
        const int c = g * 128 + lane * 4;
        float v[4];
        float m = 0.0f;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
            v[x] = c + x < cols ? src[r * lds + c + x] : 0.0f;
            if (c + x < cols) m = fp8_amax(m, v[x]);
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
        const int k = fp8_exponent(m);
        const float inv = pow2i(-k);
        const uint32_t q01 = fp8_pack2(v[0], v[1], inv), q23 = fp8_pack2(v[2], v[3], inv);
        const uint32_t q[4] = {q01 & 0xFFu, q01 >> 8, q23 & 0xFFu, q23 >> 8};
#pragma unroll
        for (int x = 0; x < 4; ++x)
            if (c + x < cols) dst[r * ldd + c + x] = (uint8_t)q[x];
        if (lane == 0) exps[r * lde + g] = (int8_t)k;
    }
}

}  // namespace proj
}  // namespace tfgk

using namespace tfgk;

// blocks: n_blocks entries (read only when blocks != nullptr); c_bf16[b] != 0 marks a bf16 output block
static int gemm_proj_impl(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda, int32_t M, int32_t K,
                          const tfgk_proj_block *blocks, const int *c_kind, int8_t *const *E, const int64_t *lde,
                          int32_t n_blocks, int32_t first_part, int32_t max_ctas, void *stream) {
    TFGK_CHECK_ARG(A_parts != nullptr && blocks != nullptr, "gemm_proj: null argument");
    TFGK_CHECK_ARG(n_parts >= 1 && n_parts <= proj::kMaxParts, "gemm_proj: n_parts=%d not in [1, %d]", n_parts, proj::kMaxParts);
    TFGK_CHECK_ARG(n_blocks >= 1 && n_blocks <= proj::kMaxBlocks, "gemm_proj: n_blocks=%d not in [1, %d]", n_blocks, proj::kMaxBlocks);
    TFGK_CHECK_ARG(M >= 0 && K >= 1, "gemm_proj: bad size (M=%d, K=%d)", M, K);
    TFGK_CHECK_ARG(first_part >= 0 && first_part < n_parts, "gemm_proj: first_part=%d out of range", first_part);
    if (M == 0) return TFGK_OK;
    if (n_parts > 1)
        TFGK_CHECK_ARG(part_rows > 0 && part_rows % proj::BM == 0 && (int64_t)n_parts * part_rows >= M,
                       "gemm_proj: part_rows=%lld must be a positive multiple of %d covering M=%d", (long long)part_rows, proj::BM, M);
    // K > 512 never fits (Plan below stops at K = 184, ops.GEMM_PROJ_MAX_K); refusing it here keeps Plan's byte counts
    // far from overflowing 32 bits
    if (K > 512 || (lda % 4) != 0 || lda < K) return TFGK_ERR_UNSUPPORTED;
    proj::Params p;
    for (int i = 0; i < proj::kMaxParts; ++i) {
        p.A[i] = A_parts[i < n_parts ? i : 0];
        if (!aligned16(p.A[i]) || p.A[i] == nullptr) return i < n_parts && A_parts[i] == nullptr
            ? set_error(TFGK_ERR_INVALID_ARGUMENT, "gemm_proj: A part %d is null", i) : TFGK_ERR_UNSUPPORTED;
    }
    p.lda = lda; p.part_rows = n_parts > 1 ? part_rows : (int64_t)1 << 40;
    p.M = M; p.K = K; p.nb = n_blocks;
    p.tiles_m = (int)ceil_div64(M, proj::BM);
    p.first_tile = n_parts > 1 ? (int)((int64_t)first_part * part_rows / proj::BM) : 0;
    if (p.first_tile >= p.tiles_m) p.first_tile = 0;
    for (int b = 0; b < proj::kMaxBlocks; ++b) {
        const tfgk_proj_block &blk = blocks[b < n_blocks ? b : 0];
        if (b < n_blocks) {
            TFGK_CHECK_ARG(blk.B != nullptr && blk.C != nullptr, "gemm_proj: block %d has a null operand", b);
            TFGK_CHECK_ARG(blk.ncols >= 1 && blk.ldb >= (blk.transB ? K : blk.ncols) && blk.ldc >= blk.ncols,
                           "gemm_proj: block %d has bad sizes", b);
            TFGK_CHECK_ARG(blk.act == TFGK_ACT_NONE || blk.act == TFGK_ACT_RELU, "gemm_proj: unknown activation %d", blk.act);
            if (blk.ncols > proj::kUN) return TFGK_ERR_UNSUPPORTED;
        }
        p.B[b] = blk.B; p.ldb[b] = blk.ldb; p.bias[b] = blk.bias; p.act[b] = blk.act; p.ncols[b] = blk.ncols;
        p.transb[b] = blk.transB;
        p.C[b] = blk.C; p.ldc[b] = blk.ldc; p.c_kind[b] = b < n_blocks ? c_kind[b] : 0;
        p.E[b] = b < n_blocks && E != nullptr ? E[b] : nullptr; p.lde[b] = b < n_blocks && lde != nullptr ? lde[b] : 0;
    }
    const proj::Plan L(K);
    if (L.stages == 0) return TFGK_ERR_UNSUPPORTED;     // W (hi | lo) does not fit next to two A stages
    p.kpad = (int)L.kpad;
    int dev = 0, sms = 0;
    TFGK_CUDA(cudaGetDevice(&dev));
    TFGK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (max_ctas > 0 && max_ctas < sms) sms = max_ctas;
    int n_groups = sms / n_blocks;
    if (n_groups < 1) n_groups = 1;
    if (n_groups > p.tiles_m) n_groups = p.tiles_m;
    p.n_groups = n_groups;
    const int grid = n_groups * n_blocks;
    cudaStream_t st = as_stream(stream);
    if (L.stages >= 4) return proj::launch<4>(p, grid, L.total, st);
    if (L.stages == 3) return proj::launch<3>(p, grid, L.total, st);
    return proj::launch<2>(p, grid, L.total, st);
}

extern "C" int tfgk_gemm_proj_f32(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                                  int32_t M, int32_t K, const tfgk_proj_block *blocks, int32_t n_blocks,
                                  int32_t first_part, int32_t max_ctas, void *stream) {
    const int all_f32[proj::kMaxBlocks] = {0, 0, 0, 0};
    return gemm_proj_impl(A_parts, n_parts, part_rows, lda, M, K, blocks, all_f32, nullptr, nullptr, n_blocks, first_part,
                          max_ctas, stream);
}

extern "C" int tfgk_gemm_proj_mixed(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                                    int32_t M, int32_t K, const tfgk_proj_block_out *blocks, int32_t n_blocks,
                                    int32_t first_part, int32_t max_ctas, void *stream) {
    TFGK_CHECK_ARG(A_parts != nullptr && blocks != nullptr, "gemm_proj: null argument");
    TFGK_CHECK_ARG(n_blocks >= 1 && n_blocks <= proj::kMaxBlocks, "gemm_proj: n_blocks=%d not in [1, %d]", n_blocks, proj::kMaxBlocks);
    tfgk_proj_block plain[proj::kMaxBlocks];
    int c_bf16[proj::kMaxBlocks];
    for (int b = 0; b < n_blocks; ++b) {
        const tfgk_proj_block_out &o = blocks[b];
        TFGK_CHECK_ARG(o.c_dtype == TFGK_DTYPE_F32 || o.c_dtype == TFGK_DTYPE_BF16, "gemm_proj: block %d has unknown dtype %d",
                       b, o.c_dtype);
        if (o.c_dtype == TFGK_DTYPE_BF16)
            TFGK_CHECK_ARG((reinterpret_cast<uintptr_t>(o.C) & 1u) == 0, "gemm_proj: block %d: bf16 output not 2-byte aligned", b);
        plain[b].B = o.B; plain[b].ldb = o.ldb; plain[b].ncols = o.ncols; plain[b].transB = o.transB;
        plain[b].bias = o.bias; plain[b].act = o.act; plain[b].C = static_cast<float *>(o.C); plain[b].ldc = o.ldc;
        c_bf16[b] = o.c_dtype == TFGK_DTYPE_BF16;
    }
    if (n_parts != 1) return set_error(TFGK_ERR_UNSUPPORTED, "gemm_proj_mixed: only a single-part A is supported (n_parts=%d)", n_parts);
    return gemm_proj_impl(A_parts, n_parts, part_rows, lda, M, K, plain, c_bf16, nullptr, nullptr, n_blocks, first_part,
                          max_ctas, stream);
}

extern "C" int tfgk_gemm_proj_fp8(const float *const *A_parts, int32_t n_parts, int64_t part_rows, int64_t lda,
                                  int32_t M, int32_t K, const tfgk_proj_block_fp8 *blocks, int32_t n_blocks,
                                  int32_t first_part, int32_t max_ctas, void *stream) {
    TFGK_CHECK_ARG(A_parts != nullptr && blocks != nullptr, "gemm_proj: null argument");
    TFGK_CHECK_ARG(n_blocks >= 1 && n_blocks <= proj::kMaxBlocks, "gemm_proj: n_blocks=%d not in [1, %d]", n_blocks, proj::kMaxBlocks);
    tfgk_proj_block plain[proj::kMaxBlocks];
    int kind[proj::kMaxBlocks];
    int8_t *E[proj::kMaxBlocks];
    int64_t lde[proj::kMaxBlocks];
    for (int b = 0; b < n_blocks; ++b) {
        const tfgk_proj_block_fp8 &o = blocks[b];
        TFGK_CHECK_ARG(o.c_dtype == TFGK_DTYPE_F32 || o.c_dtype == TFGK_DTYPE_BF16 || o.c_dtype == TFGK_DTYPE_FP8_E4M3,
                       "gemm_proj: block %d has unknown dtype %d", b, o.c_dtype);
        if (o.c_dtype == TFGK_DTYPE_BF16)
            TFGK_CHECK_ARG((reinterpret_cast<uintptr_t>(o.C) & 1u) == 0, "gemm_proj: block %d: bf16 output not 2-byte aligned", b);
        if (o.c_dtype == TFGK_DTYPE_FP8_E4M3)
            TFGK_CHECK_ARG(o.E != nullptr && o.lde >= 1, "gemm_proj: block %d: fp8 output without exponents", b);
        plain[b].B = o.B; plain[b].ldb = o.ldb; plain[b].ncols = o.ncols; plain[b].transB = o.transB;
        plain[b].bias = o.bias; plain[b].act = o.act; plain[b].C = static_cast<float *>(o.C); plain[b].ldc = o.ldc;
        kind[b] = o.c_dtype == TFGK_DTYPE_FP8_E4M3 ? 2 : o.c_dtype == TFGK_DTYPE_BF16 ? 1 : 0;
        E[b] = o.E; lde[b] = o.lde;
    }
    if (n_parts != 1) return set_error(TFGK_ERR_UNSUPPORTED, "gemm_proj_fp8: only a single-part A is supported (n_parts=%d)", n_parts);
    return gemm_proj_impl(A_parts, n_parts, part_rows, lda, M, K, plain, kind, E, lde, n_blocks, first_part, max_ctas, stream);
}

extern "C" int tfgk_quantize_fp8(const float *src, int64_t lds, int32_t rows, int32_t cols, uint8_t *dst, int64_t ldd,
                                 int8_t *exps, int64_t lde, void *stream) {
    TFGK_CHECK_ARG(rows >= 0 && cols >= 0, "quantize_fp8: negative size (rows=%d, cols=%d)", rows, cols);
    if (rows == 0 || cols == 0) return TFGK_OK;
    TFGK_CHECK_ARG(src != nullptr && dst != nullptr && exps != nullptr, "quantize_fp8: null pointer");
    TFGK_CHECK_ARG(lds >= cols && ldd >= cols && lde >= (cols + 127) / 128, "quantize_fp8: leading dimension too small");
    const int64_t warps = (int64_t)rows * ((cols + 127) / 128);
    const int64_t blocks = ceil_div64(warps, 8);
    const unsigned grid = (unsigned)(blocks < 8 * sm_count() ? blocks : 8 * sm_count());
    proj::quantize_fp8_kernel<<<grid, 256, 0, as_stream(stream)>>>(src, lds, rows, cols, dst, ldd, exps, lde);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

extern "C" int tfgk_round_bf16(const float *src, int64_t lds, int32_t rows, int32_t cols, uint16_t *dst, int64_t ldd,
                               void *stream) {
    TFGK_CHECK_ARG(rows >= 0 && cols >= 0, "round_bf16: negative size (rows=%d, cols=%d)", rows, cols);
    if (rows == 0 || cols == 0) return TFGK_OK;
    TFGK_CHECK_ARG(src != nullptr && dst != nullptr, "round_bf16: null pointer");
    TFGK_CHECK_ARG(lds >= cols && ldd >= cols, "round_bf16: leading dimension < cols");
    const int64_t n = (int64_t)rows * cols;
    const unsigned grid = (unsigned)(ceil_div64(n, 256) < 4 * sm_count() ? ceil_div64(n, 256) : 4 * sm_count());
    proj::round_bf16_kernel<<<grid, 256, 0, as_stream(stream)>>>(src, lds, rows, cols, reinterpret_cast<__nv_bfloat16 *>(dst),
                                                                 ldd);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}
