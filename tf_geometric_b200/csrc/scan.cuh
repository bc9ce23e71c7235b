// Device-wide exclusive scan shared by the index kernels (tile scan -> scan of tile sums -> add) plus the small
// launch helpers they use.  Header-only: every translation unit that includes it gets its own instantiations.
#pragma once
#include "common.cuh"

namespace tfgk {

// ------------------------------------------------------------------------------------------------------------
// exclusive scan (tile scan -> scan of tile sums -> add), used for the radix histograms and rowptr
// ------------------------------------------------------------------------------------------------------------

constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;
constexpr int kScanTile = kScanThreads * kScanItems;

// kCountNonZero: scan (in[i] != 0) instead of in[i], so that a flag of any non-zero value counts once
template <typename TIn, typename TOut, bool kCountNonZero = false>
__global__ void __launch_bounds__(kScanThreads) scan_tile_kernel(const TIn *in, int64_t n_in, int64_t n_out,
                                                                 TOut *out, TOut *__restrict__ tile_sums) {
    // thread t owns items [t*kScanItems, (t+1)*kScanItems) of the tile (blocked arrangement)
    __shared__ TOut warp_tot[kScanThreads / 32];
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    TOut v[kScanItems];
    TOut sum = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        const int64_t idx = base + i;
        const TOut x = idx < n_in ? (kCountNonZero ? (TOut)(in[idx] != 0) : (TOut)in[idx]) : (TOut)0;
        v[i] = sum;      // exclusive within the thread
        sum += x;
    }
    // inclusive warp scan of the thread sums
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    TOut incl = sum;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const TOut y = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += y;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    TOut warp_off = 0;
    for (int w = 0; w < warp; ++w) warp_off += warp_tot[w];
    const TOut thread_off = warp_off + incl - sum;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        const int64_t idx = base + i;
        if (idx < n_out) out[idx] = v[i] + thread_off;
    }
    if (threadIdx.x == kScanThreads - 1) tile_sums[blockIdx.x] = thread_off + sum;
}

template <typename TOut>
__global__ void __launch_bounds__(1024) scan_sums_kernel(TOut *__restrict__ tile_sums, int64_t n_tiles) {
    // single block: exclusive scan of the tile sums in chunks of 1024 with a running carry
    __shared__ TOut warp_tot[32];
    __shared__ TOut carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t base = 0; base < n_tiles; base += 1024) {
        const int64_t idx = base + threadIdx.x;
        const TOut x = idx < n_tiles ? tile_sums[idx] : (TOut)0;
        TOut incl = x;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const TOut y = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off) incl += y;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        TOut warp_off = 0;
        for (int w = 0; w < warp; ++w) warp_off += warp_tot[w];
        const TOut carry = carry_s;
        if (idx < n_tiles) tile_sums[idx] = carry + warp_off + incl - x;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + warp_off + incl;
        __syncthreads();
    }
}

template <typename TOut>
__global__ void __launch_bounds__(kScanThreads) scan_add_kernel(TOut *__restrict__ out, int64_t n_out,
                                                                const TOut *__restrict__ tile_sums) {
    const TOut off = tile_sums[blockIdx.x];
    const int64_t base = (int64_t)blockIdx.x * kScanTile;
    for (int i = threadIdx.x; i < kScanTile; i += kScanThreads) {
        const int64_t idx = base + i;
        if (idx < n_out) out[idx] += off;
    }
}

// out[0..n_out) = exclusive scan of in[0..n_in) (elements beyond n_in count as 0; n_out may be n_in + 1);
// with kCountNonZero, of (in[i] != 0): out[i] is then the number of non-zero entries before i
template <typename TIn, typename TOut, bool kCountNonZero = false>
static int exclusive_scan(const TIn *in, int64_t n_in, int64_t n_out, TOut *out, TOut *tile_sums, cudaStream_t st) {
    const int64_t n_tiles = ceil_div64(n_out, kScanTile);
    if (n_tiles == 0) return TFGK_OK;
    scan_tile_kernel<TIn, TOut, kCountNonZero><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(in, n_in, n_out, out, tile_sums);
    TFGK_LAUNCH_CHECK();
    if (n_tiles > 1) {
        scan_sums_kernel<TOut><<<1, 1024, 0, st>>>(tile_sums, n_tiles);
        TFGK_LAUNCH_CHECK();
        scan_add_kernel<TOut><<<(unsigned)n_tiles, kScanThreads, 0, st>>>(out, n_out, tile_sums);
        TFGK_LAUNCH_CHECK();
    }
    return TFGK_OK;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

static inline unsigned grid_for(int64_t n, int threads = 256) {
    int64_t b = ceil_div64(n, threads);
    if (b < 1) b = 1;
    if (b > sm_count() * 32) b = sm_count() * 32;   // grid-stride loops: 32 CTAs of 256 threads per SM is plenty
    return (unsigned)b;
}

// bytes of tile-sum scratch exclusive_scan needs for n_out outputs (as TOut = 8 bytes, the larger case)
static inline size_t scan_scratch_bytes(int64_t n_out) { return align_up((size_t)(ceil_div64(n_out, kScanTile) + 1) * 8); }

}  // namespace tfgk
