// Shared helpers for the tfgk kernels (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <float.h>
#include <atomic>
#include <mutex>
#include "tfgk.h"

namespace tfgk {

constexpr int kWarp = 32;

// thread-local error message, returned by tfgk_last_error()
char *error_buffer();
int set_error(int code, const char *fmt, ...);

inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

#define TFGK_CHECK_ARG(cond, ...)                                              \
    do {                                                                       \
        if (!(cond)) return ::tfgk::set_error(TFGK_ERR_INVALID_ARGUMENT, __VA_ARGS__); \
    } while (0)

#define TFGK_CUDA(expr)                                                        \
    do {                                                                       \
        cudaError_t err__ = (expr);                                            \
        if (err__ != cudaSuccess)                                              \
            return ::tfgk::set_error(TFGK_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, \
                                     cudaGetErrorString(err__), __FILE__, __LINE__); \
    } while (0)

#define TFGK_LAUNCH_CHECK() TFGK_CUDA(cudaGetLastError())

inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// copies a work plan's tasks, hub slices and scratch into a kernel parameter struct (SpmmParams, GatParams, MaxParams)
template <typename Params>
inline void use_plan(Params &p, const tfgk_plan *plan) {
    p.n_tasks = plan->n_tasks; p.task_row = plan->task_row; p.task_nrows = plan->task_nrows;
    p.task_e0 = plan->task_e0; p.task_e1 = plan->task_e1; p.task_slot = plan->task_slot;
    p.n_hubs = plan->n_hubs; p.hub_row = plan->hub_row; p.hub_slot0 = plan->hub_slot0; p.hub_nslots = plan->hub_nslots;
    p.scratch = plan->scratch;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize once per (kernel, device) instead of on every launch (the attribute call costs
// microseconds - invisible next to a 10 ms aggregation, visible on Cora-sized graphs where a forward is a few launches).
// Only ever raises the limit; safe from several host threads (a repeated set is harmless).
template <typename Kernel>
inline cudaError_t ensure_dynamic_smem(Kernel kernel, size_t bytes) {
    struct Entry { const void *fn; int dev; size_t bytes; };
    static Entry table[256];
    static int used = 0;
    static std::mutex guard;                  // launches may come from several host threads
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) return err;
    std::lock_guard<std::mutex> lock(guard);
    const void *fn = reinterpret_cast<const void *>(kernel);
    const int n = used < 256 ? used : 256;
    for (int i = 0; i < n; ++i)
        if (table[i].fn == fn && table[i].dev == dev && table[i].bytes >= bytes) return cudaSuccess;
    err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (err == cudaSuccess && used < 256) {
        table[used].fn = fn; table[used].dev = dev; table[used].bytes = bytes;
        ++used;
    }
    return err;
}

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe), queried once per device.  It sizes the
// grid-stride grids, the split-K and column-sum decisions and the copy kernel's default grid.
inline int sm_count() {
    static std::atomic<int> cache[64];       // zero-initialised: static storage
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = -1;
    int n = dev >= 0 ? cache[dev].load(std::memory_order_relaxed) : 0;
    if (n == 0) {
        if (dev < 0 || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            return 132;                      // no device to ask: the launch that follows reports the error
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline bool is_pow2(int x) { return x > 0 && (x & (x - 1)) == 0; }

// (H, dqk) of the GAT training path without the [E, H] coefficient table.  The forward that keeps (max, denominator)
// per (row, head) (tfgk_gat_fused_stats_f32) exists only to feed the backward that recomputes the coefficients
// (tfgk_gat_bwd_*_f32), so both take exactly these shapes: dqk / 4 lanes per head, A = H * dqk <= 128 (one float4 per
// lane), H <= 8 (the backward packs [m | den | delta] per row in 8-float slots).  Any other shape keeps the table.
inline bool gat_recompute_shape(int H, int dqk) {
    return is_pow2(H) && H <= 8 && dqk % 4 == 0 && is_pow2(dqk / 4) && H * dqk <= 128;
}

// activation applied in every fused epilogue
__device__ __forceinline__ float apply_act(float v, int act) {
    return act == TFGK_ACT_RELU ? fmaxf(v, 0.0f) : v;
}

// streaming (read-once) loads: keep them out of L1 so gathered feature rows own the cache
__device__ __forceinline__ int ld_stream_i32(const int *p) {
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_stream_f32(const float *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// bf16 message rows are stored as their 16-bit patterns (uint16_t); widening to fp32 is exact (the pattern is the upper
// half of the fp32 one), so a kernel that widens each element and then runs the fp32 arithmetic computes exactly what the
// fp32 kernel computes over the widened table.
__device__ __forceinline__ float bf16_to_f32(uint32_t bits) { return __uint_as_float(bits << 16); }

// four consecutive row elements at `p` (shared or global memory), widened to fp32: one 16-byte load for fp32 rows, one
// 8-byte load for bf16 rows (p aligned accordingly)
template <typename T> __device__ __forceinline__ float4 load_row4(const uint8_t *p);
template <> __device__ __forceinline__ float4 load_row4<float>(const uint8_t *p) {
    return *reinterpret_cast<const float4 *>(p);
}
template <> __device__ __forceinline__ float4 load_row4<uint16_t>(const uint8_t *p) {
    const uint2 t = *reinterpret_cast<const uint2 *>(p);
    return make_float4(__uint_as_float(t.x << 16), __uint_as_float(t.x & 0xFFFF0000u), __uint_as_float(t.y << 16),
                       __uint_as_float(t.y & 0xFFFF0000u));
}

inline bool aligned8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

// ---- fp8 message rows (OCP e4m3fn with one power-of-two exponent k per row and group of 128 columns, tfgk.h) ----------
// Dequantised value x^ = float(q) * 2^k: e4m3 -> f16 -> f32 is exact, and so is the product for every k in [-126, 127],
// so a kernel that widens each element this way and then runs the fp32 arithmetic computes exactly what the fp32 kernel
// computes over the dequantised table.

// 2^e for e in [-127, 127] (2^-127 is the one subnormal)
__device__ __forceinline__ float pow2i(int e) {
    return e >= -126 ? __int_as_float((e + 127) << 23) : __int_as_float(0x00400000);
}
__device__ __forceinline__ float f16_bits_to_f32(unsigned short h) {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
}
// two e4m3 bytes (low byte first) -> f16x2 (low half first), exact
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(unsigned short b) {
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(b));
    return r;
}
__device__ __forceinline__ float e4m3_to_f32(uint32_t byte) {
    return f16_bits_to_f32((unsigned short)(e4m3x2_to_f16x2((unsigned short)(byte & 0xFFu)) & 0xFFFFu));
}
// four e4m3 elements from one 4-byte load, widened (not yet scaled by 2^k)
template <> __device__ __forceinline__ float4 load_row4<uint8_t>(const uint8_t *p) {
    const uint32_t t = *reinterpret_cast<const uint32_t *>(p);
    const uint32_t lo = e4m3x2_to_f16x2((unsigned short)(t & 0xFFFFu)), hi = e4m3x2_to_f16x2((unsigned short)(t >> 16));
    return make_float4(f16_bits_to_f32((unsigned short)(lo & 0xFFFFu)), f16_bits_to_f32((unsigned short)(lo >> 16)),
                       f16_bits_to_f32((unsigned short)(hi & 0xFFFFu)), f16_bits_to_f32((unsigned short)(hi >> 16)));
}
__device__ __forceinline__ float4 scale4(float4 v, float s) {
    return make_float4(__fmul_rn(v.x, s), __fmul_rn(v.y, s), __fmul_rn(v.z, s), __fmul_rn(v.w, s));
}
// running maximum of |v| over the finite entries of a group
__device__ __forceinline__ float fp8_amax(float m, float v) {
    const float a = fabsf(v);
    return a <= FLT_MAX ? fmaxf(m, a) : m;
}
// the smallest k with amax * 2^-k <= 448, clamped to [-126, 127]; 0 for amax == 0 (a group without finite entries).
// amax = f 2^e with f in [1, 2): k = e - 8 when f <= 1.75 (448 = 1.75 2^8), else e - 7; subnormal amax clamps to -126
__device__ __forceinline__ int fp8_exponent(float amax) {
    if (amax == 0.0f) return 0;
    const uint32_t b = __float_as_uint(amax);
    const int field = (int)(b >> 23);
    if (field == 0) return -126;
    const int k = field - 127 - 8 + ((b & 0x7FFFFFu) > 0x600000u ? 1 : 0);
    return k < -126 ? -126 : (k > 127 ? 127 : k);
}
// x0, x1 -> two e4m3 bytes (x0 in the low byte): RNE of x * inv (inv = 2^-k, the product is exact or far below the
// smallest e4m3 subnormal); +-inf and NaN become NaN with their sign (0x7F / 0xFF), as e4m3fn has no infinities
__device__ __forceinline__ uint32_t fp8_pack2(float x0, float x1, float inv) {
    unsigned short r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__fmul_rn(x1, inv)), "f"(__fmul_rn(x0, inv)));
    uint32_t b0 = r & 0xFFu, b1 = (uint32_t)r >> 8;
    if (!(fabsf(x0) <= FLT_MAX)) b0 = 0x7Fu | ((__float_as_uint(x0) >> 24) & 0x80u);
    if (!(fabsf(x1) <= FLT_MAX)) b1 = 0x7Fu | ((__float_as_uint(x1) >> 24) & 0x80u);
    return b0 | (b1 << 8);
}

}  // namespace tfgk
