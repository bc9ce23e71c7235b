// Integer edge preprocessing, destination-sorted CSR build (stable LSD radix sort), GCN normalisation helpers.
// Everything here is HBM-bound integer/byte work: coalesced streaming loads, shared-memory staging for the
// radix ranks, no tensor cores.  Results are bit-exact with the numpy oracle (oracle/tfg_oracle.py).
#include "common.cuh"
#include "scan.cuh"
#include <cuda_fp16.h>
#include <string.h>
#include <algorithm>

namespace tfgk {

static thread_local char g_error[512] = "";

char *error_buffer() { return g_error; }

int set_error(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
    return code;
}

// ------------------------------------------------------------------------------------------------------------
// small elementwise kernels
// ------------------------------------------------------------------------------------------------------------

__global__ void self_loops_kernel(const int32_t *__restrict__ ei, int64_t E, int32_t N, int32_t *__restrict__ out) {
    // out is [2, E+N] row-major; ei is [2, E] row-major.
    const int64_t Ep = E + N;
    const int64_t total = 2 * Ep;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i >= Ep ? 1 : 0;
        const int64_t j = i - r * Ep;
        out[i] = j < E ? ei[r * E + j] : (int32_t)(j - E);
    }
}

__global__ void self_loop_weights_kernel(const float *__restrict__ w, int64_t E, int32_t N, float fill,
                                         float *__restrict__ out) {
    const int64_t total = E + N;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = i < E ? (w ? w[i] : 1.0f) : fill;
}

__global__ void count_kernel(const int32_t *__restrict__ ids, int64_t E, int32_t N, int32_t *__restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = ids[i];
        if (r >= 0 && r < N) atomicAdd(&out[r], 1);   // integer atomics: order-independent, deterministic
    }
}

__global__ void validate_kernel(const int32_t *__restrict__ ids, int64_t E, int32_t N, int32_t *__restrict__ bad) {
    int local = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = ids[i];
        local |= (r < 0 || r >= N);
    }
    if (__any_sync(0xffffffffu, local) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
}

__global__ void gather_i32_kernel(const int32_t *__restrict__ src, const int32_t *__restrict__ perm, int64_t E,
                                  int32_t *__restrict__ dst) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = src[perm[i]];
}

__global__ void permute_f32_kernel(const float *__restrict__ src, const int32_t *__restrict__ perm, int64_t E,
                                   int32_t width, float *__restrict__ dst, bool inverse) {
    const int64_t total = E * width;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = i / width;
        const int32_t j = (int32_t)(i - e * width);
        const int64_t p = perm[e];
        if (inverse) dst[p * width + j] = src[i];
        else         dst[i] = src[p * width + j];
    }
}

// ---- row gather from a feature table in host memory (tfgk_gather_rows_mapped_f32) -----------------------------------
// One warp per output row, grid-strided.  A read crosses the host link (microseconds, not HBM's hundreds of
// nanoseconds), so every SM holds gather warps and each lane issues up to kGatherUnroll loads before it stores.  On an
// H100 the rate of 400-byte rows was the same with 1, 2 and 8 blocks of 8 warps per SM, so the grid stops at 2 per SM and
// leaves the rest of each SM to kernels on other streams.  An id outside [0, n_rows) gives a NaN row and no read.
constexpr int kGatherThreads = 256;
constexpr int kGatherBlocksPerSm = 2;
constexpr int kGatherUnroll = 4;

template <typename V>
__device__ __forceinline__ V nan_vec();
template <> __device__ __forceinline__ float nan_vec<float>() { return __int_as_float(0x7fc00000); }
template <> __device__ __forceinline__ float4 nan_vec<float4>() {
    const float q = __int_as_float(0x7fc00000);
    return make_float4(q, q, q, q);
}

// V = float4: F, ld and ldo (and ldc when kCached) counted in floats are multiples of 4 and every base is 16-byte aligned.
// kCached (tfgk_gather_rows_cached_f32): slot[r] >= 0 says row r is also cache[slot[r], :F] in device memory, which is
// read instead of the host row; the map is read once per output row, by every lane of its warp from one address.
template <typename V, bool kCached>
__device__ __forceinline__ void gather_rows_mapped_body(const float *__restrict__ table, int64_t ld, int64_t n_rows,
                                                        int32_t F, const float *__restrict__ cache, int64_t ldc,
                                                        const int32_t *__restrict__ slot,
                                                        const int32_t *__restrict__ index, int64_t n,
                                                        float *__restrict__ out, int64_t ldo) {
    constexpr int kW = sizeof(V) / sizeof(float);
    const int lane = threadIdx.x & 31;
    const int32_t nv = F / kW;                                   // vectors per row
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int32_t r = index[i];
        V *dst = reinterpret_cast<V *>(out + i * ldo);
        if (r < 0 || (int64_t)r >= n_rows) {
            for (int32_t c = lane; c < nv; c += 32) dst[c] = nan_vec<V>();
            continue;
        }
        const V *src = reinterpret_cast<const V *>(table + (int64_t)r * ld);
        if constexpr (kCached) {
            const int32_t s = __ldg(slot + r);
            if (s >= 0) src = reinterpret_cast<const V *>(cache + (int64_t)s * ldc);
        }
        for (int32_t c0 = lane; c0 < nv; c0 += 32 * kGatherUnroll) {
            V v[kGatherUnroll];
#pragma unroll
            for (int u = 0; u < kGatherUnroll; ++u)
                if (c0 + 32 * u < nv) v[u] = src[c0 + 32 * u];
#pragma unroll
            for (int u = 0; u < kGatherUnroll; ++u)
                if (c0 + 32 * u < nv) dst[c0 + 32 * u] = v[u];
        }
    }
}

__global__ void __launch_bounds__(kGatherThreads) gather_rows_mapped_vec4_kernel(
        const float *__restrict__ table, int64_t ld, int64_t n_rows, int32_t F, const int32_t *__restrict__ index,
        int64_t n, float *__restrict__ out, int64_t ldo) {
    gather_rows_mapped_body<float4, false>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo);
}

__global__ void __launch_bounds__(kGatherThreads) gather_rows_mapped_f32_kernel(
        const float *__restrict__ table, int64_t ld, int64_t n_rows, int32_t F, const int32_t *__restrict__ index,
        int64_t n, float *__restrict__ out, int64_t ldo) {
    gather_rows_mapped_body<float, false>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo);
}

__global__ void __launch_bounds__(kGatherThreads) gather_rows_cached_vec4_kernel(
        const float *__restrict__ table, int64_t ld, int64_t n_rows, int32_t F, const float *__restrict__ cache,
        int64_t ldc, const int32_t *__restrict__ slot, const int32_t *__restrict__ index, int64_t n,
        float *__restrict__ out, int64_t ldo) {
    gather_rows_mapped_body<float4, true>(table, ld, n_rows, F, cache, ldc, slot, index, n, out, ldo);
}

__global__ void __launch_bounds__(kGatherThreads) gather_rows_cached_f32_kernel(
        const float *__restrict__ table, int64_t ld, int64_t n_rows, int32_t F, const float *__restrict__ cache,
        int64_t ldc, const int32_t *__restrict__ slot, const int32_t *__restrict__ index, int64_t n,
        float *__restrict__ out, int64_t ldo) {
    gather_rows_mapped_body<float, true>(table, ld, n_rows, F, cache, ldc, slot, index, n, out, ldo);
}

// ---- the same gather from a 16-bit table (tfgk_gather_rows_mapped_16, tfgk_gather_rows_cached_16) ------------------
// Elements are bf16 or fp16 bit patterns; kVec of them (8, 4, 2 or 1: 16, 8, 4 or 2 bytes) travel in one load, and the
// launcher takes the widest kVec that F, the strides and the base pointers allow.  Each element is widened to float32
// exactly (bf16: a 16-bit shift; fp16: the hardware conversion), so out is the float32 table's gather bit for bit.
// kCopy (mapped entry only) stores the 16-bit patterns unchanged instead, and a 16-bit NaN for a bad id.
template <int kVec> struct Bits16;
template <> struct Bits16<8> { using T = uint4; };
template <> struct Bits16<4> { using T = uint2; };
template <> struct Bits16<2> { using T = uint32_t; };
template <> struct Bits16<1> { using T = uint16_t; };

template <bool kHalf>
__device__ __forceinline__ float widen16(uint32_t h) {
    if constexpr (kHalf) return __half2float(__ushort_as_half((unsigned short)h));
    else return __uint_as_float(h << 16);
}

// element j of a kVec-wide load (little-endian: element 0 is the low half of the first word)
template <int kVec>
__device__ __forceinline__ uint32_t elem16(const typename Bits16<kVec>::T &v, int j) {
    if constexpr (kVec == 1) {
        return v;
    } else {
        const uint32_t *w = reinterpret_cast<const uint32_t *>(&v);
        return (w[j >> 1] >> (16 * (j & 1))) & 0xffffu;
    }
}

template <int kVec>
__device__ __forceinline__ typename Bits16<kVec>::T splat16(uint32_t h) {
    using L = typename Bits16<kVec>::T;
    if constexpr (kVec == 1) {
        return (L)h;
    } else {
        L v;
        uint32_t *w = reinterpret_cast<uint32_t *>(&v);
#pragma unroll
        for (int k = 0; k < kVec / 2; ++k) w[k] = h | (h << 16);
        return v;
    }
}

// kVec float32 values at dst, in float4 / float2 / float stores (dst is aligned to min(16, 4 kVec) bytes)
template <int kVec>
__device__ __forceinline__ void store_f32(float *dst, const float (&f)[kVec]) {
    if constexpr (kVec >= 4) {
#pragma unroll
        for (int k = 0; k < kVec / 4; ++k)
            reinterpret_cast<float4 *>(dst)[k] = make_float4(f[4 * k], f[4 * k + 1], f[4 * k + 2], f[4 * k + 3]);
    } else if constexpr (kVec == 2) {
        *reinterpret_cast<float2 *>(dst) = make_float2(f[0], f[1]);
    } else {
        dst[0] = f[0];
    }
}

template <int kVec, bool kHalf, bool kCached, bool kCopy>
__global__ void __launch_bounds__(kGatherThreads) gather_rows_16_kernel(
        const uint16_t *__restrict__ table, int64_t ld, int64_t n_rows, int32_t F, const uint16_t *__restrict__ cache,
        int64_t ldc, const int32_t *__restrict__ slot, const int32_t *__restrict__ index, int64_t n,
        void *__restrict__ out, int64_t ldo) {
    using L = typename Bits16<kVec>::T;
    const int lane = threadIdx.x & 31;
    const int32_t nv = F / kVec;                                 // loads per row
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
        const int32_t r = index[i];
        L *dst16 = reinterpret_cast<L *>(static_cast<uint16_t *>(out) + i * ldo);
        float *dst32 = static_cast<float *>(out) + i * ldo;
        if (r < 0 || (int64_t)r >= n_rows) {
            if constexpr (kCopy) {
                for (int32_t c = lane; c < nv; c += 32) dst16[c] = splat16<kVec>(kHalf ? 0x7e00u : 0x7fc0u);
            } else {
                float q[kVec];
#pragma unroll
                for (int j = 0; j < kVec; ++j) q[j] = __int_as_float(0x7fc00000);
                for (int32_t c = lane; c < nv; c += 32) store_f32<kVec>(dst32 + (int64_t)c * kVec, q);
            }
            continue;
        }
        const L *src = reinterpret_cast<const L *>(table + (int64_t)r * ld);
        if constexpr (kCached) {
            const int32_t s = __ldg(slot + r);
            if (s >= 0) src = reinterpret_cast<const L *>(cache + (int64_t)s * ldc);
        }
        for (int32_t c0 = lane; c0 < nv; c0 += 32 * kGatherUnroll) {
            L v[kGatherUnroll];
#pragma unroll
            for (int u = 0; u < kGatherUnroll; ++u)
                if (c0 + 32 * u < nv) v[u] = src[c0 + 32 * u];
#pragma unroll
            for (int u = 0; u < kGatherUnroll; ++u) {
                const int32_t c = c0 + 32 * u;
                if (c >= nv) continue;
                if constexpr (kCopy) {
                    dst16[c] = v[u];
                } else {
                    float f[kVec];
#pragma unroll
                    for (int j = 0; j < kVec; ++j) f[j] = widen16<kHalf>(elem16<kVec>(v[u], j));
                    store_f32<kVec>(dst32 + (int64_t)c * kVec, f);
                }
            }
        }
    }
}

// Whether kVec 16-bit elements per load fit: F and every stride a multiple of kVec, the 16-bit bases aligned to 2 kVec
// bytes, and the output's rows and base aligned to its store width (2 kVec bytes when copying, min(16, 4 kVec) when
// widening to float32, which is stored in float4 pieces).
static bool gather16_fits(int kVec, int32_t F, int64_t ld, const void *table, int64_t ldc, const void *cache,
                          int64_t ldo, const void *out, int out_bytes) {
    const uintptr_t in_align = 2u * kVec;
    const uintptr_t out_align = out_bytes == 2 ? in_align : (uintptr_t)std::min(16, 4 * kVec);
    return F % kVec == 0 && ld % kVec == 0 && (reinterpret_cast<uintptr_t>(table) & (in_align - 1)) == 0 &&
           (cache == nullptr || (ldc % kVec == 0 && (reinterpret_cast<uintptr_t>(cache) & (in_align - 1)) == 0)) &&
           ((uint64_t)ldo * out_bytes) % out_align == 0 && (reinterpret_cast<uintptr_t>(out) & (out_align - 1)) == 0;
}

template <bool kHalf, bool kCached, bool kCopy>
static void launch_gather16(const uint16_t *table, int64_t ld, int64_t n_rows, int32_t F, const uint16_t *cache,
                            int64_t ldc, const int32_t *slot, const int32_t *index, int64_t n, void *out, int64_t ldo,
                            cudaStream_t st) {
    const int64_t warps_per_block = kGatherThreads / 32;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(n, warps_per_block),
                                                        (int64_t)sm_count() * kGatherBlocksPerSm);
    const int out_bytes = kCopy ? 2 : 4;
    if (gather16_fits(8, F, ld, table, ldc, cache, ldo, out, out_bytes))
        gather_rows_16_kernel<8, kHalf, kCached, kCopy><<<blocks, kGatherThreads, 0, st>>>(table, ld, n_rows, F, cache,
                                                                                          ldc, slot, index, n, out, ldo);
    else if (gather16_fits(4, F, ld, table, ldc, cache, ldo, out, out_bytes))
        gather_rows_16_kernel<4, kHalf, kCached, kCopy><<<blocks, kGatherThreads, 0, st>>>(table, ld, n_rows, F, cache,
                                                                                          ldc, slot, index, n, out, ldo);
    else if (gather16_fits(2, F, ld, table, ldc, cache, ldo, out, out_bytes))
        gather_rows_16_kernel<2, kHalf, kCached, kCopy><<<blocks, kGatherThreads, 0, st>>>(table, ld, n_rows, F, cache,
                                                                                          ldc, slot, index, n, out, ldo);
    else
        gather_rows_16_kernel<1, kHalf, kCached, kCopy><<<blocks, kGatherThreads, 0, st>>>(table, ld, n_rows, F, cache,
                                                                                          ldc, slot, index, n, out, ldo);
}

__global__ void csr_rowsum_kernel(const int64_t *__restrict__ rowptr, const float *__restrict__ w, int32_t N,
                                  float *__restrict__ out) {
    // one thread per row, strictly left-to-right: reproduces unsorted_segment_sum's fp32 rounding sequence
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    float acc = 0.0f;
    for (int64_t e = rowptr[r]; e < rowptr[r + 1]; ++e) acc = __fadd_rn(acc, w[e]);
    out[r] = acc;
}

__global__ void deg_inv_kernel(const float *__restrict__ deg, int32_t N, int power, float *__restrict__ out) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const float d = deg[r];
    // pow(d, -0.5) / pow(d, -1) correctly rounded; inf and nan -> 0 (gcn.py:23-29)
    float v = power == TFGK_POW_INV_SQRT ? __frsqrt_rn(d) : __frcp_rn(d);
    if (isinf(v) || isnan(v)) v = 0.0f;
    out[r] = v;
}

__global__ void scale_edges_kernel(const int32_t *__restrict__ row, const int32_t *__restrict__ col,
                                   const float *__restrict__ w, int64_t E, const float *__restrict__ dl,
                                   const float *__restrict__ dr, float *__restrict__ out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        float v = w ? w[i] : 1.0f;
        if (dl) v = __fmul_rn(dl[row[i]], v);
        if (dr) v = __fmul_rn(v, dr[col[i]]);
        out[i] = v;
    }
}

// ------------------------------------------------------------------------------------------------------------
// stable LSD radix sort of (row -> edge position), 8 bits per pass
// ------------------------------------------------------------------------------------------------------------

constexpr int kRsThreads = 256;
constexpr int kRsWarps = kRsThreads / 32;
constexpr int kRsItems = 16;                       // rounds per warp
constexpr int kRsTile = kRsThreads * kRsItems;     // 4096 keys per block
constexpr int kRadix = 256;

__global__ void __launch_bounds__(kRsThreads) rs_hist_kernel(const int32_t *__restrict__ keys, int64_t E, int shift,
                                                             uint32_t *__restrict__ hist, int nblk) {
    __shared__ uint32_t sh[kRadix];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kRsTile;
#pragma unroll 4
    for (int i = threadIdx.x; i < kRsTile; i += kRsThreads) {
        const int64_t idx = base + i;
        if (idx < E) atomicAdd(&sh[(keys[idx] >> shift) & (kRadix - 1)], 1u);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * nblk + blockIdx.x] = sh[threadIdx.x];   // digit-major for the global scan
}

__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const int32_t *__restrict__ kin,
                                                                const int32_t *__restrict__ vin, int64_t E, int shift,
                                                                const uint32_t *__restrict__ hist_scanned, int nblk,
                                                                int32_t *__restrict__ kout, int32_t *__restrict__ vout) {
    __shared__ uint32_t warp_cnt[kRsWarps][kRadix];
    __shared__ uint32_t digit_base[kRadix];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int w = 0; w < kRsWarps; ++w) warp_cnt[w][threadIdx.x] = 0;
    digit_base[threadIdx.x] = hist_scanned[(int64_t)threadIdx.x * nblk + blockIdx.x];
    __syncthreads();

    // warp w owns the contiguous sub-tile [w*32*kRsItems, (w+1)*32*kRsItems); round i covers 32 consecutive keys.
    const int64_t base = (int64_t)blockIdx.x * kRsTile + (int64_t)warp * (32 * kRsItems);
    int32_t key[kRsItems];
    uint32_t rank[kRsItems];
#pragma unroll
    for (int i = 0; i < kRsItems; ++i) {
        const int64_t idx = base + i * 32 + lane;
        const bool valid = idx < E;
        key[i] = valid ? kin[idx] : 0;
        const uint32_t d = (uint32_t)(key[i] >> shift) & (kRadix - 1);
        // invalid tail lanes form their own group and never touch the counters
        const uint32_t peers = __match_any_sync(0xffffffffu, valid ? d : 0x100u);
        const int leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if (lane == leader && valid) {
            old = warp_cnt[warp][d];
            warp_cnt[warp][d] = old + __popc(peers);
        }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[i] = old + __popc(peers & ((1u << lane) - 1u));   // same-digit keys earlier in (round, lane) order
        __syncwarp();
    }
    __syncthreads();
    {   // exclusive prefix over warps, per digit (thread t = digit t)
        uint32_t run = 0;
#pragma unroll
        for (int w = 0; w < kRsWarps; ++w) {
            const uint32_t c = warp_cnt[w][threadIdx.x];
            warp_cnt[w][threadIdx.x] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kRsItems; ++i) {
        const int64_t idx = base + i * 32 + lane;
        if (idx < E) {
            const uint32_t d = (uint32_t)(key[i] >> shift) & (kRadix - 1);
            const uint32_t dst = digit_base[d] + warp_cnt[warp][d] + rank[i];
            if (kout) kout[dst] = key[i];
            vout[dst] = vin ? vin[idx] : (int32_t)idx;
        }
    }
}


// Stable LSD radix sort of int32 keys in [0, max_key] carrying the original positions; the sorted positions land in
// `perm_out`.  keys_a/keys_b/vals_b/hist/sums are scratch (E ints each for the first three).
static int stable_sort_positions(const int32_t *keys, int64_t E, int64_t max_key_exclusive, int32_t *perm_out,
                                 int32_t *keys_a, int32_t *keys_b, int32_t *vals_b, uint32_t *hist, void *sums, int nblk,
                                 cudaStream_t st) {
    int bits = 1;
    while (bits < 31 && (1ll << bits) < max_key_exclusive) ++bits;
    const int passes = (bits + 7) / 8;
    const int32_t *kin = keys;
    const int32_t *vin = nullptr;   // implicit iota
    for (int p = 1; p <= passes; ++p) {
        const bool to_x = ((passes - p) % 2) == 0;        // X = (keys_a, perm_out), Y = (keys_b, vals_b)
        int32_t *kout = to_x ? keys_a : keys_b;
        int32_t *vout = to_x ? perm_out : vals_b;
        const int shift = (p - 1) * 8;
        rs_hist_kernel<<<nblk, kRsThreads, 0, st>>>(kin, E, shift, hist, nblk);
        TFGK_LAUNCH_CHECK();
        const int64_t n_hist = (int64_t)kRadix * nblk;
        const int rc = exclusive_scan<uint32_t, uint32_t>(hist, n_hist, n_hist, hist, reinterpret_cast<uint32_t *>(sums), st);
        if (rc != TFGK_OK) return rc;
        rs_scatter_kernel<<<nblk, kRsThreads, 0, st>>>(kin, vin, E, shift, hist, nblk, p == passes ? nullptr : kout, vout);
        TFGK_LAUNCH_CHECK();
        kin = kout;
        vin = vout;
    }
    return TFGK_OK;
}

// order-preserving 32-bit key of a float (IEEE trick: flip all bits of negatives, the sign bit of non-negatives);
// -0.0 is folded into +0.0 first so that numerically equal scores tie.  descending = complement.
__global__ void sort_keys_f32_kernel(const float *__restrict__ score, int64_t n, int descending, int32_t *__restrict__ keys) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint32_t u = __float_as_uint(score[i] + 0.0f);
        u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
        keys[i] = (int32_t)(descending ? ~u : u);
    }
}

// ---- duplicate-edge detection (utils/graph_utils.py:67-125: hash = n*row+col, tf.unique first-occurrence order) ----------
__global__ void gather2_i32_kernel(const int32_t *__restrict__ a, const int32_t *__restrict__ b,
                                   const int32_t *__restrict__ perm, int64_t E, int32_t *__restrict__ a_out,
                                   int32_t *__restrict__ b_out) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t p = perm[i];
        if (a_out) a_out[i] = a[p];
        if (b_out) b_out[i] = b[p];
    }
}

// in (row, col)-sorted order: flag the first edge of every group of equal (row, col)
__global__ void group_flag_kernel(const int32_t *__restrict__ sr, const int32_t *__restrict__ sc, int64_t E,
                                  int32_t *__restrict__ flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = (i == 0 || sr[i] != sr[i - 1] || sc[i] != sc[i - 1]) ? 1 : 0;
}

// group g (sorted order) starts where flag == 1; its first occurrence in the input is the position stored there
__global__ void group_first_kernel(const int32_t *__restrict__ flag, const int32_t *__restrict__ gid_excl,
                                   const int32_t *__restrict__ pos_sorted, int64_t E, int32_t *__restrict__ first_pos) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x)
        if (flag[i]) first_pos[gid_excl[i]] = pos_sorted[i];      // stable sort: the group's smallest input position
}

// rank_of_group[order[j]] = j ; then per edge: unique_of_edge[pos_sorted[i]] = rank_of_group[group(i)], and the unique edge
// list in first-occurrence order
__global__ void invert_perm_kernel(const int32_t *__restrict__ order, int64_t n, int32_t *__restrict__ rank) {
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
        rank[order[j]] = (int32_t)j;
}

__global__ void unique_emit_kernel(const int32_t *__restrict__ flag, const int32_t *__restrict__ gid_excl,
                                   const int32_t *__restrict__ rank, const int32_t *__restrict__ pos_sorted,
                                   const int32_t *__restrict__ sr, const int32_t *__restrict__ sc, int64_t E, int64_t cap,
                                   int32_t *__restrict__ unique_index, int32_t *__restrict__ unique_of_edge) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < E; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t g = flag[i] ? gid_excl[i] : gid_excl[i] - 1;    // exclusive scan of the flags -> group id
        const int32_t u = rank[g];
        unique_of_edge[pos_sorted[i]] = u;
        if (flag[i]) { unique_index[u] = sr[i]; unique_index[cap + u] = sc[i]; }
    }
}

// convert_edge_to_directed (utils/graph_utils.py:181-190): mirrored copies of the non-self-loop upper edges, in order
__global__ void nonloop_flag_kernel(const int32_t *__restrict__ idx, int64_t U, int64_t ld, int32_t *__restrict__ flag) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < U; i += (int64_t)gridDim.x * blockDim.x)
        flag[i] = idx[i] != idx[ld + i] ? 1 : 0;
}

__global__ void directed_emit_kernel(const int32_t *__restrict__ idx, int64_t U, int64_t ld, const int32_t *__restrict__ flag,
                                     const int32_t *__restrict__ off, int64_t out_ld, int32_t *__restrict__ out,
                                     int32_t *__restrict__ lower_src) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < U; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = idx[i], c = idx[ld + i];
        out[i] = r;
        out[out_ld + i] = c;
        if (flag[i]) {
            const int64_t j = U + off[i];
            out[j] = c;
            out[out_ld + j] = r;
            lower_src[off[i]] = (int32_t)i;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// work plan: runs of <= rows_per_task light rows, hub rows cut into `chunk`-edge slices
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool plan_is_hub(const int64_t *rowptr, int32_t r, int32_t hub_threshold) {
    return rowptr[r + 1] - rowptr[r] > hub_threshold;
}

__global__ void plan_count_kernel(const int64_t *__restrict__ rowptr, int32_t N, int32_t hub_threshold, int32_t chunk,
                                  int32_t rpt, int32_t *__restrict__ cnt_tasks, int32_t *__restrict__ cnt_hubs,
                                  int32_t *__restrict__ cnt_slots) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const int64_t deg = rowptr[r + 1] - rowptr[r];
    const bool hub = deg > hub_threshold;
    int32_t tasks = 0, slots = 0;
    if (hub) {
        slots = (int32_t)((deg + chunk - 1) / chunk);
        tasks = slots;
    } else if (r % rpt == 0 || plan_is_hub(rowptr, r - 1, hub_threshold)) {
        tasks = 1;          // this row starts a run of light rows
    }
    cnt_tasks[r] = tasks;
    cnt_hubs[r] = hub ? 1 : 0;
    cnt_slots[r] = slots;
}

__global__ void plan_fill_kernel(const int64_t *__restrict__ rowptr, int32_t N, int32_t hub_threshold, int32_t chunk,
                                 int32_t rpt, const int32_t *__restrict__ off_tasks, const int32_t *__restrict__ off_hubs,
                                 const int32_t *__restrict__ off_slots, int32_t *__restrict__ task_row,
                                 int32_t *__restrict__ task_nrows, int64_t *__restrict__ task_e0,
                                 int64_t *__restrict__ task_e1, int32_t *__restrict__ task_slot,
                                 int32_t *__restrict__ hub_row, int32_t *__restrict__ hub_slot0,
                                 int32_t *__restrict__ hub_nslots) {
    const int32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    const int64_t start = rowptr[r], end = rowptr[r + 1];
    const int64_t deg = end - start;
    if (deg > hub_threshold) {
        const int32_t slots = (int32_t)((deg + chunk - 1) / chunk);
        const int32_t h = off_hubs[r], s0 = off_slots[r], t0 = off_tasks[r];
        hub_row[h] = r; hub_slot0[h] = s0; hub_nslots[h] = slots;
        for (int32_t j = 0; j < slots; ++j) {
            task_row[t0 + j] = r; task_nrows[t0 + j] = 1;
            task_e0[t0 + j] = start + (int64_t)j * chunk;
            task_e1[t0 + j] = min(end, start + (int64_t)(j + 1) * chunk);
            task_slot[t0 + j] = s0 + j;
        }
    } else if (r % rpt == 0 || plan_is_hub(rowptr, r - 1, hub_threshold)) {
        int32_t r2 = r + 1;
        while (r2 < N && r2 % rpt != 0 && !plan_is_hub(rowptr, r2, hub_threshold)) ++r2;
        const int32_t t = off_tasks[r];
        task_row[t] = r; task_nrows[t] = r2 - r; task_e0[t] = start; task_e1[t] = rowptr[r2]; task_slot[t] = -1;
    }
}

// ---- building a CSR from an edge list in host memory (utils.HostNeighborSampler) -----------------------------------
// Every kernel here streams the mapped edge list in order: thread t of a block reads the 4 consecutive ids at
// 4 (g * blockDim + t), one 16-byte load when the array is 16-byte aligned, so a warp reads 512 contiguous bytes.
constexpr int kMapThreads = 256;
constexpr int kMapTile = 4 * kMapThreads;            // edges per tile of the row selection

// ids[e0 .. e0 + 4) into v; ids past n read as -1.  vec: ids is 16-byte aligned (e0 is a multiple of 4).
__device__ __forceinline__ void load_ids4(const int32_t *__restrict__ ids, int64_t e0, int64_t n, bool vec, int32_t v[4]) {
    if (vec && e0 + 4 <= n) {
        const int4 q = *reinterpret_cast<const int4 *>(ids + e0);
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        return;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = e0 + j < n ? ids[e0 + j] : -1;
}

// range[0..4) = {min row, max row, min col, max col}, folded with atomics into INT32_MAX / INT32_MIN seeds
__global__ void mapped_range_init_kernel(int32_t *range) {
    range[0] = range[2] = INT32_MAX;
    range[1] = range[3] = INT32_MIN;
}

__global__ void __launch_bounds__(kMapThreads) mapped_id_range_kernel(const int32_t *__restrict__ row,
                                                                      const int32_t *__restrict__ col, int64_t E,
                                                                      bool vec_row, bool vec_col, int32_t *range) {
    int32_t lo[2] = {INT32_MAX, INT32_MAX}, hi[2] = {INT32_MIN, INT32_MIN};
    const int64_t n4 = (E + 3) / 4;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n4; g += (int64_t)gridDim.x * blockDim.x) {
        int32_t v[4];
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            load_ids4(a ? col : row, 4 * g, E, a ? vec_col : vec_row, v);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (4 * g + j < E) { lo[a] = min(lo[a], v[j]); hi[a] = max(hi[a], v[j]); }
        }
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            lo[a] = min(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], off));
            hi[a] = max(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], off));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(range + 2 * a, lo[a]);
            atomicMax(range + 2 * a + 1, hi[a]);
        }
    }
}

// counts[r] += 1 per edge of row r (int64 counts, so a row of 2^31 edges or more is counted, then refused by the caller)
__global__ void __launch_bounds__(kMapThreads) mapped_row_count_kernel(const int32_t *__restrict__ row, int64_t E,
                                                                       bool vec, int32_t n_rows,
                                                                       unsigned long long *__restrict__ counts) {
    const int64_t n4 = (E + 3) / 4;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n4; g += (int64_t)gridDim.x * blockDim.x) {
        int32_t v[4];
        load_ids4(row, 4 * g, E, vec, v);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (v[j] >= 0 && v[j] < n_rows) atomicAdd(counts + v[j], 1ull);
    }
}

// the edges of tile blockIdx.x with r0 <= row < r1
__global__ void __launch_bounds__(kMapThreads) mapped_select_count_kernel(const int32_t *__restrict__ row, int64_t E,
                                                                          bool vec, int32_t r0, int32_t r1,
                                                                          int64_t *__restrict__ tile_count) {
    __shared__ int warp_sum[kMapThreads / 32];
    int32_t v[4];
    load_ids4(row, (int64_t)blockIdx.x * kMapTile + 4 * threadIdx.x, E, vec, v);
    int c = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) c += (v[j] >= r0 && v[j] < r1);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int total = 0;
        for (int w = 0; w < kMapThreads / 32; ++w) total += warp_sum[w];
        tile_count[blockIdx.x] = total;
    }
}

// Stable compaction of the tile's selected edges to tile_off[tile] + (selected edges before them in the tile): the
// offset within a tile is an int, the tile's offset an int64.  Writes row - r0, col and w (when w is not null); nothing
// at or past cap.
__global__ void __launch_bounds__(kMapThreads) mapped_select_emit_kernel(
        const int32_t *__restrict__ row, const int32_t *__restrict__ col, const float *__restrict__ w, int64_t E,
        bool vec, int32_t r0, int32_t r1, const int64_t *__restrict__ tile_off, int64_t cap,
        int32_t *__restrict__ out_row, int32_t *__restrict__ out_col, float *__restrict__ out_w) {
    __shared__ int warp_sum[kMapThreads / 32];
    const int64_t e0 = (int64_t)blockIdx.x * kMapTile + 4 * threadIdx.x;
    int32_t v[4];
    load_ids4(row, e0, E, vec, v);
    int c = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) c += (v[j] >= r0 && v[j] < r1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = c;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    int before = incl - c;
    for (int q = 0; q < warp; ++q) before += warp_sum[q];
    int64_t p = tile_off[blockIdx.x] + before;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (v[j] >= r0 && v[j] < r1) {
            if (p < cap) {
                out_row[p] = v[j] - r0;
                out_col[p] = col[e0 + j];
                if (w) out_w[p] = w[e0 + j];
            }
            ++p;
        }
    }
}

struct CsrWorkspace {
    size_t off_flag, off_keys_a, off_keys_b, off_vals_b, off_hist, off_sums, off_counts, total;
    int nblk;
    CsrWorkspace(int64_t E, int32_t N) {
        nblk = (int)ceil_div64(E > 0 ? E : 1, kRsTile);
        const int64_t n_hist = (int64_t)kRadix * nblk;
        const int64_t n_sums = ceil_div64((n_hist > (int64_t)N + 1 ? n_hist : (int64_t)N + 1), kScanTile) + 1;
        size_t o = 0;
        off_flag = o;   o += align_up(sizeof(int32_t));
        off_keys_a = o; o += align_up((size_t)E * 4);
        off_keys_b = o; o += align_up((size_t)E * 4);
        off_vals_b = o; o += align_up((size_t)E * 4);
        off_hist = o;   o += align_up((size_t)n_hist * 4);
        off_sums = o;   o += align_up((size_t)n_sums * 8);
        off_counts = o; o += align_up(((size_t)N + 1) * 4);
        total = o;
    }
};

}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_version(void) { return TFGK_ABI_VERSION; }

const char *tfgk_last_error(void) { return error_buffer(); }

int tfgk_device_info(int *sm_count, int *cc_major, int *cc_minor) {
    int dev = 0;
    TFGK_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    TFGK_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return TFGK_OK;
}

int tfgk_self_loops_i32(const int32_t *edge_index, int64_t E, int32_t N, int32_t *out, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && N >= 0, "self_loops: negative size (E=%lld, N=%d)", (long long)E, N);
    TFGK_CHECK_ARG(E + N < (1ll << 31), "self_loops: E + N must be < 2^31");
    if (E + N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(out != nullptr && (E == 0 || edge_index != nullptr), "self_loops: null pointer");
    self_loops_kernel<<<grid_for(2 * (E + N)), 256, 0, as_stream(stream)>>>(edge_index, E, N, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_self_loop_weights_f32(const float *w, int64_t E, int32_t N, float fill, float *out, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && N >= 0, "self_loop_weights: negative size");
    if (E + N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(out != nullptr, "self_loop_weights: null output");
    self_loop_weights_kernel<<<grid_for(E + N), 256, 0, as_stream(stream)>>>(w, E, N, fill, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_segment_count_i32(const int32_t *ids, int64_t E, int32_t N, int32_t *out, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && N >= 0, "segment_count: negative size");
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(out != nullptr && (E == 0 || ids != nullptr), "segment_count: null pointer");
    TFGK_CUDA(cudaMemsetAsync(out, 0, (size_t)N * 4, as_stream(stream)));
    if (E > 0) {
        count_kernel<<<grid_for(E), 256, 0, as_stream(stream)>>>(ids, E, N, out);
        TFGK_LAUNCH_CHECK();
    }
    return TFGK_OK;
}

int tfgk_csr_workspace_bytes(int64_t E, int32_t N, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr, "csr_workspace_bytes: null output");
    TFGK_CHECK_ARG(E >= 0 && N >= 0 && E < (1ll << 31), "csr_workspace_bytes: need 0 <= E < 2^31, N >= 0");
    *out_bytes = CsrWorkspace(E, N).total;
    return TFGK_OK;
}

static int csr_build(const int32_t *row, const int32_t *col, int64_t E, int32_t N_rows, int32_t N_cols,
                     int64_t *rowptr, int32_t *col_sorted, int32_t *perm, void *workspace, size_t workspace_bytes,
                     bool check_ids, cudaStream_t st) {
    TFGK_CHECK_ARG(E >= 0 && E < (1ll << 31), "csr_build: need 0 <= E < 2^31 (got %lld)", (long long)E);
    TFGK_CHECK_ARG(N_rows >= 0 && N_cols >= 0, "csr_build: negative node count");
    TFGK_CHECK_ARG(rowptr != nullptr, "csr_build: null rowptr");
    if (E == 0) {
        TFGK_CUDA(cudaMemsetAsync(rowptr, 0, ((size_t)N_rows + 1) * 8, st));
        return TFGK_OK;
    }
    TFGK_CHECK_ARG(row && col && col_sorted && perm, "csr_build: null pointer");
    const CsrWorkspace L(E, N_rows);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "csr_build: workspace too small (%zu < %zu bytes)", workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    int32_t *flag = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int32_t *keys_a = reinterpret_cast<int32_t *>(ws + L.off_keys_a);
    int32_t *keys_b = reinterpret_cast<int32_t *>(ws + L.off_keys_b);
    int32_t *vals_b = reinterpret_cast<int32_t *>(ws + L.off_vals_b);
    uint32_t *hist = reinterpret_cast<uint32_t *>(ws + L.off_hist);
    void *sums = ws + L.off_sums;
    int32_t *counts = reinterpret_cast<int32_t *>(ws + L.off_counts);

    // 1. validate ids (TF-CPU's gather / segment ops raise on out-of-range ids)
    if (check_ids) {
        TFGK_CUDA(cudaMemsetAsync(flag, 0, 4, st));
        validate_kernel<<<grid_for(E), 256, 0, st>>>(row, E, N_rows, flag);
        TFGK_LAUNCH_CHECK();
        validate_kernel<<<grid_for(E), 256, 0, st>>>(col, E, N_cols, flag);
        TFGK_LAUNCH_CHECK();
        int32_t bad = 0;
        TFGK_CUDA(cudaMemcpyAsync(&bad, flag, 4, cudaMemcpyDeviceToHost, st));
        TFGK_CUDA(cudaStreamSynchronize(st));
        if (bad) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "csr_build: edge_index holds node ids outside [0, N)");
    }

    // 2. rowptr = exclusive scan of the per-row edge counts
    TFGK_CUDA(cudaMemsetAsync(counts, 0, ((size_t)N_rows + 1) * 4, st));
    count_kernel<<<grid_for(E), 256, 0, st>>>(row, E, N_rows, counts);
    TFGK_LAUNCH_CHECK();
    int rc = exclusive_scan<int32_t, int64_t>(counts, N_rows, (int64_t)N_rows + 1, rowptr,
                                              reinterpret_cast<int64_t *>(sums), st);
    if (rc != TFGK_OK) return rc;

    // 3. stable LSD radix sort of (row, position); the last pass lands in `perm`
    rc = stable_sort_positions(row, E, N_rows, perm, keys_a, keys_b, vals_b, hist, sums, L.nblk, st);
    if (rc != TFGK_OK) return rc;
    // 4. col_sorted = col[perm]
    gather_i32_kernel<<<grid_for(E), 256, 0, st>>>(col, perm, E, col_sorted);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_csr_build(const int32_t *row, const int32_t *col, int64_t E, int32_t N_rows, int32_t N_cols,
                   int64_t *rowptr, int32_t *col_sorted, int32_t *perm,
                   void *workspace, size_t workspace_bytes, void *stream) {
    return csr_build(row, col, E, N_rows, N_cols, rowptr, col_sorted, perm, workspace, workspace_bytes, true,
                     as_stream(stream));
}

int tfgk_csr_build_in_range(const int32_t *row, const int32_t *col, int64_t E, int32_t N_rows, int32_t N_cols,
                            int64_t *rowptr, int32_t *col_sorted, int32_t *perm,
                            void *workspace, size_t workspace_bytes, void *stream) {
    return csr_build(row, col, E, N_rows, N_cols, rowptr, col_sorted, perm, workspace, workspace_bytes, false,
                     as_stream(stream));
}

int tfgk_sort_keys_f32(const float *score, int64_t n, int descending, int32_t *keys, void *stream) {
    TFGK_CHECK_ARG(n >= 0, "sort_keys: negative size");
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(score && keys, "sort_keys: null pointer");
    sort_keys_f32_kernel<<<grid_for(n), 256, 0, as_stream(stream)>>>(score, n, descending, keys);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_argsort_workspace_bytes(int64_t n, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n >= 0 && n < (1ll << 31), "argsort_workspace_bytes: bad argument");
    *out_bytes = CsrWorkspace(n, 0).total;
    return TFGK_OK;
}

int tfgk_stable_argsort_u32(const int32_t *keys, int64_t n, int key_bits, int32_t *perm_out,
                            void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(n >= 0 && n < (1ll << 31), "stable_argsort: need 0 <= n < 2^31");
    TFGK_CHECK_ARG(key_bits >= 1 && key_bits <= 32, "stable_argsort: key_bits must be in [1, 32]");
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(keys && perm_out, "stable_argsort: null pointer");
    const CsrWorkspace L(n, 0);
    if (workspace == nullptr || workspace_bytes < L.total)
        return set_error(TFGK_ERR_WORKSPACE, "stable_argsort: workspace too small (%zu < %zu bytes)", workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    // every pass looks at one byte of the bit pattern, so 4 passes order all 32 bits as an unsigned number
    return stable_sort_positions(keys, n, 1ll << (key_bits > 31 ? 31 : key_bits), perm_out,
                                 reinterpret_cast<int32_t *>(ws + L.off_keys_a), reinterpret_cast<int32_t *>(ws + L.off_keys_b),
                                 reinterpret_cast<int32_t *>(ws + L.off_vals_b), reinterpret_cast<uint32_t *>(ws + L.off_hist),
                                 ws + L.off_sums, L.nblk, as_stream(stream));
}

int tfgk_edge_unique_workspace_bytes(int64_t E, int32_t N, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr, "edge_unique_workspace_bytes: null output");
    TFGK_CHECK_ARG(E >= 0 && N >= 0 && E < (1ll << 31), "edge_unique_workspace_bytes: need 0 <= E < 2^31, N >= 0");
    *out_bytes = CsrWorkspace(E, N).total + 9 * align_up((size_t)(E + 1) * 4);
    return TFGK_OK;
}

int tfgk_edge_unique(const int32_t *row, const int32_t *col, int64_t E, int32_t N, int32_t *unique_index,
                     int32_t *unique_of_edge, int32_t *n_unique_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && E < (1ll << 31) && N >= 0, "edge_unique: need 0 <= E < 2^31, N >= 0");
    TFGK_CHECK_ARG(n_unique_host != nullptr, "edge_unique: null count");
    *n_unique_host = 0;
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(row && col && unique_index && unique_of_edge, "edge_unique: null pointer");
    size_t need = 0;
    tfgk_edge_unique_workspace_bytes(E, N, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "edge_unique: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    const CsrWorkspace L(E, N);
    char *ws = static_cast<char *>(workspace);
    int32_t *flagv = reinterpret_cast<int32_t *>(ws + L.off_flag);
    int32_t *keys_a = reinterpret_cast<int32_t *>(ws + L.off_keys_a), *keys_b = reinterpret_cast<int32_t *>(ws + L.off_keys_b);
    int32_t *vals_b = reinterpret_cast<int32_t *>(ws + L.off_vals_b);
    uint32_t *hist = reinterpret_cast<uint32_t *>(ws + L.off_hist);
    void *sums = ws + L.off_sums;
    const size_t arr = align_up((size_t)(E + 1) * 4);
    char *extra = ws + L.total;
    int32_t *perm1 = reinterpret_cast<int32_t *>(extra), *rows1 = reinterpret_cast<int32_t *>(extra + arr);
    int32_t *perm2 = reinterpret_cast<int32_t *>(extra + 2 * arr), *pos = reinterpret_cast<int32_t *>(extra + 3 * arr);
    int32_t *sr = reinterpret_cast<int32_t *>(extra + 4 * arr), *sc = reinterpret_cast<int32_t *>(extra + 5 * arr);
    int32_t *flag = reinterpret_cast<int32_t *>(extra + 6 * arr), *gid = reinterpret_cast<int32_t *>(extra + 7 * arr);
    int32_t *first_pos = reinterpret_cast<int32_t *>(extra + 8 * arr);

    TFGK_CUDA(cudaMemsetAsync(flagv, 0, 4, st));
    validate_kernel<<<grid_for(E), 256, 0, st>>>(row, E, N, flagv);
    TFGK_LAUNCH_CHECK();
    validate_kernel<<<grid_for(E), 256, 0, st>>>(col, E, N, flagv);
    TFGK_LAUNCH_CHECK();
    int32_t bad = 0;
    TFGK_CUDA(cudaMemcpyAsync(&bad, flagv, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (bad) return set_error(TFGK_ERR_INDEX_OUT_OF_RANGE, "edge_unique: edge_index holds node ids outside [0, N)");

    // sort by (row, col) = by the reference's hash n*row+col: stable by col, then stable by row
    int rc = stable_sort_positions(col, E, N, perm1, keys_a, keys_b, vals_b, hist, sums, L.nblk, st);
    if (rc != TFGK_OK) return rc;
    gather2_i32_kernel<<<grid_for(E), 256, 0, st>>>(row, nullptr, perm1, E, rows1, nullptr);
    TFGK_LAUNCH_CHECK();
    rc = stable_sort_positions(rows1, E, N, perm2, keys_a, keys_b, vals_b, hist, sums, L.nblk, st);
    if (rc != TFGK_OK) return rc;
    gather2_i32_kernel<<<grid_for(E), 256, 0, st>>>(perm1, nullptr, perm2, E, pos, nullptr);       // input position of sorted slot i
    TFGK_LAUNCH_CHECK();
    gather2_i32_kernel<<<grid_for(E), 256, 0, st>>>(row, col, pos, E, sr, sc);
    TFGK_LAUNCH_CHECK();
    group_flag_kernel<<<grid_for(E), 256, 0, st>>>(sr, sc, E, flag);
    TFGK_LAUNCH_CHECK();
    rc = exclusive_scan<int32_t, int32_t>(flag, E, E + 1, gid, reinterpret_cast<int32_t *>(sums), st);
    if (rc != TFGK_OK) return rc;
    int32_t n_unique = 0;
    TFGK_CUDA(cudaMemcpyAsync(&n_unique, gid + E, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    *n_unique_host = n_unique;
    group_first_kernel<<<grid_for(E), 256, 0, st>>>(flag, gid, pos, E, first_pos);
    TFGK_LAUNCH_CHECK();
    // rank the groups by their first occurrence (tf.unique order): sort the groups by first_pos (keys < E)
    int32_t *order = perm1, *rank = rows1;       // scratch reuse: perm1 / rows1 are dead now
    const int nblk_u = (int)ceil_div64(n_unique, kRsTile);
    rc = stable_sort_positions(first_pos, n_unique, E, order, keys_a, keys_b, vals_b, hist, sums, nblk_u, st);
    if (rc != TFGK_OK) return rc;
    invert_perm_kernel<<<grid_for(n_unique), 256, 0, st>>>(order, n_unique, rank);
    TFGK_LAUNCH_CHECK();
    unique_emit_kernel<<<grid_for(E), 256, 0, st>>>(flag, gid, rank, pos, sr, sc, E, E, unique_index, unique_of_edge);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_directed_workspace_bytes(int64_t U, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && U >= 0 && U < (1ll << 30), "directed_workspace_bytes: bad argument");
    *out_bytes = 2 * align_up((size_t)(U + 1) * 4) + align_up((size_t)(ceil_div64(U + 1, kScanTile) + 1) * 8) + 256;
    return TFGK_OK;
}

int tfgk_directed_edges(const int32_t *upper_index, int64_t U, int64_t ld, int32_t *out, int64_t out_ld,
                        int32_t *lower_src, int32_t *n_lower_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(U >= 0 && U < (1ll << 30) && ld >= U && out_ld >= 2 * U, "directed_edges: bad size");
    TFGK_CHECK_ARG(n_lower_host != nullptr, "directed_edges: null count");
    *n_lower_host = 0;
    if (U == 0) return TFGK_OK;
    TFGK_CHECK_ARG(upper_index && out && lower_src, "directed_edges: null pointer");
    size_t need = 0;
    tfgk_directed_workspace_bytes(U, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "directed_edges: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    const size_t arr = align_up((size_t)(U + 1) * 4);
    int32_t *flag = reinterpret_cast<int32_t *>(ws), *off = reinterpret_cast<int32_t *>(ws + arr);
    int32_t *sums = reinterpret_cast<int32_t *>(ws + 2 * arr);
    nonloop_flag_kernel<<<grid_for(U), 256, 0, st>>>(upper_index, U, ld, flag);
    TFGK_LAUNCH_CHECK();
    const int rc = exclusive_scan<int32_t, int32_t>(flag, U, U + 1, off, sums, st);
    if (rc != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(n_lower_host, off + U, 4, cudaMemcpyDeviceToHost, st));
    directed_emit_kernel<<<grid_for(U), 256, 0, st>>>(upper_index, U, ld, flag, off, out_ld, out, lower_src);
    TFGK_LAUNCH_CHECK();
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

int tfgk_plan_capacity(int64_t E, int32_t N, int32_t hub_threshold, int32_t chunk, int32_t rows_per_task,
                       int64_t *max_tasks, int64_t *max_hubs) {
    TFGK_CHECK_ARG(E >= 0 && N >= 0 && hub_threshold >= 1 && chunk >= 1 && rows_per_task >= 1 && rows_per_task <= 32,
                   "plan_capacity: bad argument");
    TFGK_CHECK_ARG(max_tasks && max_hubs, "plan_capacity: null output");
    const int64_t hubs = E / ((int64_t)hub_threshold + 1) + 1;
    *max_hubs = hubs;
    // runs: one per rows_per_task block plus one after every hub row; slices: ceil(deg/chunk) <= deg/chunk + 1 per hub
    *max_tasks = ceil_div64(N, rows_per_task) + hubs + (E / chunk + hubs) + 2;
    return TFGK_OK;
}

int tfgk_plan_workspace_bytes(int32_t N, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes && N >= 0, "plan_workspace_bytes: bad argument");
    const size_t arr = align_up(((size_t)N + 1) * 4);
    *out_bytes = 6 * arr + align_up((size_t)(ceil_div64((int64_t)N + 1, kScanTile) + 1) * 8) + 256;
    return TFGK_OK;
}

int tfgk_plan_build(const int64_t *rowptr, int32_t N, int32_t hub_threshold, int32_t chunk, int32_t rows_per_task,
                    int32_t *task_row, int32_t *task_nrows, int64_t *task_e0, int64_t *task_e1, int32_t *task_slot,
                    int32_t *hub_row, int32_t *hub_slot0, int32_t *hub_nslots, int64_t cap_tasks, int64_t cap_hubs,
                    int32_t *counts_host, void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(N >= 0 && hub_threshold >= 1 && chunk >= 1 && rows_per_task >= 1 && rows_per_task <= 32,
                   "plan_build: bad argument");
    TFGK_CHECK_ARG(counts_host != nullptr, "plan_build: null counts");
    counts_host[0] = counts_host[1] = counts_host[2] = 0;
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && task_row && task_nrows && task_e0 && task_e1 && task_slot && hub_row && hub_slot0 && hub_nslots,
                   "plan_build: null pointer");
    size_t need = 0;
    tfgk_plan_workspace_bytes(N, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "plan_build: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    const size_t arr = align_up(((size_t)N + 1) * 4);
    int32_t *cnt_t = reinterpret_cast<int32_t *>(ws), *cnt_h = reinterpret_cast<int32_t *>(ws + arr),
            *cnt_s = reinterpret_cast<int32_t *>(ws + 2 * arr);
    int32_t *off_t = reinterpret_cast<int32_t *>(ws + 3 * arr), *off_h = reinterpret_cast<int32_t *>(ws + 4 * arr),
            *off_s = reinterpret_cast<int32_t *>(ws + 5 * arr);
    int32_t *sums = reinterpret_cast<int32_t *>(ws + 6 * arr);
    const unsigned blocks = (unsigned)ceil_div64(N, 256);
    plan_count_kernel<<<blocks, 256, 0, st>>>(rowptr, N, hub_threshold, chunk, rows_per_task, cnt_t, cnt_h, cnt_s);
    TFGK_LAUNCH_CHECK();
    int rc;
    if ((rc = exclusive_scan<int32_t, int32_t>(cnt_t, N, (int64_t)N + 1, off_t, sums, st)) != TFGK_OK) return rc;
    if ((rc = exclusive_scan<int32_t, int32_t>(cnt_h, N, (int64_t)N + 1, off_h, sums, st)) != TFGK_OK) return rc;
    if ((rc = exclusive_scan<int32_t, int32_t>(cnt_s, N, (int64_t)N + 1, off_s, sums, st)) != TFGK_OK) return rc;
    TFGK_CUDA(cudaMemcpyAsync(&counts_host[0], off_t + N, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(&counts_host[1], off_h + N, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaMemcpyAsync(&counts_host[2], off_s + N, 4, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    if (counts_host[0] > cap_tasks || counts_host[1] > cap_hubs)
        return set_error(TFGK_ERR_WORKSPACE, "plan_build: capacity too small (tasks %d > %lld or hubs %d > %lld)",
                         counts_host[0], (long long)cap_tasks, counts_host[1], (long long)cap_hubs);
    plan_fill_kernel<<<blocks, 256, 0, st>>>(rowptr, N, hub_threshold, chunk, rows_per_task, off_t, off_h, off_s, task_row,
                                             task_nrows, task_e0, task_e1, task_slot, hub_row, hub_slot0, hub_nslots);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_permute_f32(const float *src, const int32_t *perm, int64_t E, int32_t width, float *dst, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && width >= 1, "permute: bad size");
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(src && perm && dst, "permute: null pointer");
    permute_f32_kernel<<<grid_for(E * width), 256, 0, as_stream(stream)>>>(src, perm, E, width, dst, false);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_unpermute_f32(const float *src, const int32_t *perm, int64_t E, int32_t width, float *dst, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && width >= 1, "unpermute: bad size");
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(src && perm && dst, "unpermute: null pointer");
    permute_f32_kernel<<<grid_for(E * width), 256, 0, as_stream(stream)>>>(src, perm, E, width, dst, true);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

// a failed registration call leaves its error as the runtime's last error, which the next launch check would report:
// clear it and return it with the call's name
static int host_error(cudaError_t err, const char *what) {
    cudaGetLastError();
    return set_error(TFGK_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(err));
}

int tfgk_host_register(void *ptr, size_t bytes, void **dev_ptr) {
    TFGK_CHECK_ARG(ptr != nullptr && dev_ptr != nullptr, "host_register: null pointer");
    TFGK_CHECK_ARG(bytes > 0, "host_register: empty range");
    *dev_ptr = nullptr;
    cudaError_t err = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
    if (err != cudaSuccess) return host_error(err, "cudaHostRegister");
    void *dev = nullptr;
    err = cudaHostGetDevicePointer(&dev, ptr, 0);
    if (err != cudaSuccess) {
        cudaHostUnregister(ptr);
        return host_error(err, "cudaHostGetDevicePointer");
    }
    *dev_ptr = dev;
    return TFGK_OK;
}

int tfgk_host_unregister(void *ptr) {
    TFGK_CHECK_ARG(ptr != nullptr, "host_unregister: null pointer");
    // a gather still in flight on any stream would read the range after it is released
    cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) return host_error(err, "cudaDeviceSynchronize");
    err = cudaHostUnregister(ptr);
    if (err != cudaSuccess) return host_error(err, "cudaHostUnregister");
    return TFGK_OK;
}

int tfgk_gather_rows_mapped_f32(const float *table, int64_t ld, int64_t n_rows, int32_t F, const int32_t *index,
                                int64_t n, float *out, int64_t ldo, void *stream) {
    TFGK_CHECK_ARG(n >= 0 && n_rows >= 0 && F >= 1, "gather_rows_mapped: bad size (n=%lld, n_rows=%lld, F=%d)",
                   (long long)n, (long long)n_rows, F);
    TFGK_CHECK_ARG(ld >= F && ldo >= F, "gather_rows_mapped: need ld >= F and ldo >= F (ld=%lld, ldo=%lld, F=%d)",
                   (long long)ld, (long long)ldo, F);
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(index && out && (table || n_rows == 0), "gather_rows_mapped: null pointer");
    const int64_t warps_per_block = kGatherThreads / 32;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(n, warps_per_block),
                                                        (int64_t)sm_count() * kGatherBlocksPerSm);
    const bool vec = F % 4 == 0 && ld % 4 == 0 && ldo % 4 == 0 && aligned16(table) && aligned16(out);
    if (vec)
        gather_rows_mapped_vec4_kernel<<<blocks, kGatherThreads, 0, as_stream(stream)>>>(table, ld, n_rows, F, index, n,
                                                                                        out, ldo);
    else
        gather_rows_mapped_f32_kernel<<<blocks, kGatherThreads, 0, as_stream(stream)>>>(table, ld, n_rows, F, index, n,
                                                                                       out, ldo);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_gather_rows_cached_f32(const float *table, int64_t ld, int64_t n_rows, int32_t F, const float *cache,
                                int64_t ldc, const int32_t *slot, const int32_t *index, int64_t n, float *out,
                                int64_t ldo, void *stream) {
    TFGK_CHECK_ARG(n >= 0 && n_rows >= 0 && F >= 1, "gather_rows_cached: bad size (n=%lld, n_rows=%lld, F=%d)",
                   (long long)n, (long long)n_rows, F);
    TFGK_CHECK_ARG(ld >= F && ldc >= F && ldo >= F,
                   "gather_rows_cached: need ld, ldc and ldo >= F (ld=%lld, ldc=%lld, ldo=%lld, F=%d)", (long long)ld,
                   (long long)ldc, (long long)ldo, F);
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(index && out && cache && slot && (table || n_rows == 0), "gather_rows_cached: null pointer");
    const int64_t warps_per_block = kGatherThreads / 32;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(n, warps_per_block),
                                                        (int64_t)sm_count() * kGatherBlocksPerSm);
    const bool vec = F % 4 == 0 && ld % 4 == 0 && ldc % 4 == 0 && ldo % 4 == 0 && aligned16(table) &&
                     aligned16(cache) && aligned16(out);
    if (vec)
        gather_rows_cached_vec4_kernel<<<blocks, kGatherThreads, 0, as_stream(stream)>>>(table, ld, n_rows, F, cache,
                                                                                        ldc, slot, index, n, out, ldo);
    else
        gather_rows_cached_f32_kernel<<<blocks, kGatherThreads, 0, as_stream(stream)>>>(table, ld, n_rows, F, cache,
                                                                                       ldc, slot, index, n, out, ldo);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_gather_rows_mapped_16(const uint16_t *table, int32_t dtype, int64_t ld, int64_t n_rows, int32_t F,
                               const int32_t *index, int64_t n, void *out, int32_t out_dtype, int64_t ldo,
                               void *stream) {
    TFGK_CHECK_ARG(dtype == TFGK_DTYPE_BF16 || dtype == TFGK_DTYPE_F16,
                   "gather_rows_mapped_16: dtype must be TFGK_DTYPE_BF16 or TFGK_DTYPE_F16 (got %d)", dtype);
    TFGK_CHECK_ARG(out_dtype == TFGK_DTYPE_F32 || out_dtype == dtype,
                   "gather_rows_mapped_16: out_dtype must be TFGK_DTYPE_F32 or the table's dtype %d (got %d)", dtype,
                   out_dtype);
    TFGK_CHECK_ARG(n >= 0 && n_rows >= 0 && F >= 1, "gather_rows_mapped_16: bad size (n=%lld, n_rows=%lld, F=%d)",
                   (long long)n, (long long)n_rows, F);
    TFGK_CHECK_ARG(ld >= F && ldo >= F, "gather_rows_mapped_16: need ld >= F and ldo >= F (ld=%lld, ldo=%lld, F=%d)",
                   (long long)ld, (long long)ldo, F);
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(index && out && (table || n_rows == 0), "gather_rows_mapped_16: null pointer");
    const bool half = dtype == TFGK_DTYPE_F16, copy = out_dtype == dtype;
    cudaStream_t st = as_stream(stream);
    if (half && copy)
        launch_gather16<true, false, true>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo, st);
    else if (half)
        launch_gather16<true, false, false>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo, st);
    else if (copy)
        launch_gather16<false, false, true>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo, st);
    else
        launch_gather16<false, false, false>(table, ld, n_rows, F, nullptr, 0, nullptr, index, n, out, ldo, st);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_gather_rows_cached_16(const uint16_t *table, int32_t dtype, int64_t ld, int64_t n_rows, int32_t F,
                               const uint16_t *cache, int64_t ldc, const int32_t *slot, const int32_t *index,
                               int64_t n, float *out, int64_t ldo, void *stream) {
    TFGK_CHECK_ARG(dtype == TFGK_DTYPE_BF16 || dtype == TFGK_DTYPE_F16,
                   "gather_rows_cached_16: dtype must be TFGK_DTYPE_BF16 or TFGK_DTYPE_F16 (got %d)", dtype);
    TFGK_CHECK_ARG(n >= 0 && n_rows >= 0 && F >= 1, "gather_rows_cached_16: bad size (n=%lld, n_rows=%lld, F=%d)",
                   (long long)n, (long long)n_rows, F);
    TFGK_CHECK_ARG(ld >= F && ldc >= F && ldo >= F,
                   "gather_rows_cached_16: need ld, ldc and ldo >= F (ld=%lld, ldc=%lld, ldo=%lld, F=%d)",
                   (long long)ld, (long long)ldc, (long long)ldo, F);
    if (n == 0) return TFGK_OK;
    TFGK_CHECK_ARG(index && out && cache && slot && (table || n_rows == 0), "gather_rows_cached_16: null pointer");
    cudaStream_t st = as_stream(stream);
    if (dtype == TFGK_DTYPE_F16)
        launch_gather16<true, true, false>(table, ld, n_rows, F, cache, ldc, slot, index, n, out, ldo, st);
    else
        launch_gather16<false, true, false>(table, ld, n_rows, F, cache, ldc, slot, index, n, out, ldo, st);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

static unsigned mapped_grid(int64_t E) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(ceil_div64(E, 4), kMapThreads),
                                                            (int64_t)sm_count() * 8));
}

int tfgk_mapped_id_range_i32(const int32_t *row, const int32_t *col, int64_t E, int32_t *range_host, void *workspace,
                             size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(E > 0 && range_host != nullptr, "mapped_id_range: bad argument (E=%lld)", (long long)E);
    TFGK_CHECK_ARG(row && col, "mapped_id_range: null edge list");
    if (workspace == nullptr || workspace_bytes < 16)
        return set_error(TFGK_ERR_WORKSPACE, "mapped_id_range: workspace too small (%zu < 16 bytes)", workspace_bytes);
    cudaStream_t st = as_stream(stream);
    int32_t *range = static_cast<int32_t *>(workspace);
    mapped_range_init_kernel<<<1, 1, 0, st>>>(range);
    TFGK_LAUNCH_CHECK();
    mapped_id_range_kernel<<<mapped_grid(E), kMapThreads, 0, st>>>(row, col, E, aligned16(row), aligned16(col), range);
    TFGK_LAUNCH_CHECK();
    TFGK_CUDA(cudaMemcpyAsync(range_host, range, 16, cudaMemcpyDeviceToHost, st));
    TFGK_CUDA(cudaStreamSynchronize(st));
    return TFGK_OK;
}

int tfgk_mapped_rowptr_workspace_bytes(int32_t n_rows, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && n_rows >= 0, "mapped_rowptr_workspace_bytes: bad argument");
    *out_bytes = scan_scratch_bytes((int64_t)n_rows + 1);
    return TFGK_OK;
}

int tfgk_mapped_rowptr_i32(const int32_t *row, int64_t E, int32_t n_rows, int64_t *rowptr, void *workspace,
                           size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && n_rows >= 0, "mapped_rowptr: bad size (E=%lld, n_rows=%d)", (long long)E, n_rows);
    TFGK_CHECK_ARG(rowptr != nullptr && (E == 0 || row != nullptr), "mapped_rowptr: null pointer");
    size_t need = 0;
    tfgk_mapped_rowptr_workspace_bytes(n_rows, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "mapped_rowptr: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
    cudaStream_t st = as_stream(stream);
    TFGK_CUDA(cudaMemsetAsync(rowptr, 0, ((size_t)n_rows + 1) * 8, st));
    if (E > 0 && n_rows > 0) {
        mapped_row_count_kernel<<<mapped_grid(E), kMapThreads, 0, st>>>(row, E, aligned16(row), n_rows,
                                                                       reinterpret_cast<unsigned long long *>(rowptr));
        TFGK_LAUNCH_CHECK();
    }
    // in place: each scan thread reads its counts before it writes their offsets
    return exclusive_scan<int64_t, int64_t>(rowptr, n_rows, (int64_t)n_rows + 1, rowptr,
                                            static_cast<int64_t *>(workspace), st);
}

int tfgk_mapped_select_rows_workspace_bytes(int64_t E, size_t *out_bytes) {
    TFGK_CHECK_ARG(out_bytes != nullptr && E >= 0, "mapped_select_rows_workspace_bytes: bad argument");
    const int64_t tiles = ceil_div64(E, kMapTile);
    *out_bytes = align_up((size_t)(tiles + 1) * 8) + scan_scratch_bytes(tiles + 1);
    return TFGK_OK;
}

int tfgk_mapped_select_rows_i32(const int32_t *row, const int32_t *col, const float *w, int64_t E, int32_t r0,
                                int32_t r1, int32_t *out_row, int32_t *out_col, float *out_w, int64_t cap,
                                void *workspace, size_t workspace_bytes, void *stream) {
    TFGK_CHECK_ARG(E >= 0 && r0 >= 0 && r1 >= r0 && cap >= 0 && cap < (1ll << 31),
                   "mapped_select_rows: bad size (E=%lld, rows [%d, %d), cap=%lld)", (long long)E, r0, r1, (long long)cap);
    if (E == 0 || cap == 0 || r1 == r0) return TFGK_OK;
    TFGK_CHECK_ARG(row && col && out_row && out_col && (!w || out_w), "mapped_select_rows: null pointer");
    size_t need = 0;
    tfgk_mapped_select_rows_workspace_bytes(E, &need);
    if (workspace == nullptr || workspace_bytes < need)
        return set_error(TFGK_ERR_WORKSPACE, "mapped_select_rows: workspace too small (%zu < %zu bytes)", workspace_bytes,
                         need);
    const int64_t tiles = ceil_div64(E, kMapTile);
    TFGK_CHECK_ARG(tiles < (1ll << 31), "mapped_select_rows: %lld edges are too many tiles", (long long)E);
    cudaStream_t st = as_stream(stream);
    char *ws = static_cast<char *>(workspace);
    int64_t *tile_off = reinterpret_cast<int64_t *>(ws);
    int64_t *sums = reinterpret_cast<int64_t *>(ws + align_up((size_t)(tiles + 1) * 8));
    const bool vec = aligned16(row);
    mapped_select_count_kernel<<<(unsigned)tiles, kMapThreads, 0, st>>>(row, E, vec, r0, r1, tile_off);
    TFGK_LAUNCH_CHECK();
    int rc = exclusive_scan<int64_t, int64_t>(tile_off, tiles, tiles, tile_off, sums, st);
    if (rc != TFGK_OK) return rc;
    mapped_select_emit_kernel<<<(unsigned)tiles, kMapThreads, 0, st>>>(row, col, w, E, vec, r0, r1, tile_off, cap, out_row,
                                                                       out_col, out_w);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_csr_rowsum_f32(const int64_t *rowptr, const float *w_csr, int32_t N, float *out, void *stream) {
    TFGK_CHECK_ARG(N >= 0, "csr_rowsum: negative N");
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && out, "csr_rowsum: null pointer");
    csr_rowsum_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, as_stream(stream)>>>(rowptr, w_csr, N, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_deg_inv_f32(const float *deg, int32_t N, int power, float *out, void *stream) {
    TFGK_CHECK_ARG(N >= 0, "deg_inv: negative N");
    TFGK_CHECK_ARG(power == TFGK_POW_INV_SQRT || power == TFGK_POW_INV, "deg_inv: unknown power %d", power);
    if (N == 0) return TFGK_OK;
    TFGK_CHECK_ARG(deg && out, "deg_inv: null pointer");
    deg_inv_kernel<<<(unsigned)ceil_div64(N, 256), 256, 0, as_stream(stream)>>>(deg, N, power, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

int tfgk_scale_edges_f32(const int32_t *row, const int32_t *col, const float *w, int64_t E,
                         const float *dl, const float *dr, float *out, void *stream) {
    TFGK_CHECK_ARG(E >= 0, "scale_edges: negative E");
    if (E == 0) return TFGK_OK;
    TFGK_CHECK_ARG(out && (!dl || row) && (!dr || col), "scale_edges: null pointer");
    scale_edges_kernel<<<grid_for(E), 256, 0, as_stream(stream)>>>(row, col, w, E, dl, dr, out);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // extern "C"
