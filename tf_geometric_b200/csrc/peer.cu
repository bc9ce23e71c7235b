// K5 plumbing: IPC-exportable device buffers and a device-side barrier over NVLink peer mappings (include/tfgk.h).
// The data path itself is in gemm_proj.cu (cp.async straight from the owning rank's memory).
#include "common.cuh"

namespace tfgk {

struct FlagTable { uint32_t *flags[8]; };

__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

__global__ void peer_barrier_kernel(const FlagTable tab, int rank, int world, uint32_t value, uint64_t timeout_ns) {
    const int j = threadIdx.x;
    if (j >= world) return;
    // everything this stream did before the barrier (the copy into the published slot) is complete at kernel start;
    // the fence orders it before the flag for observers on other GPUs
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(tab.flags[j] + rank), "r"(value) : "memory");
    const uint32_t *mine = tab.flags[rank] + j;
    const uint64_t t0 = global_timer_ns();
    for (;;) {
        uint32_t seen;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(mine) : "memory");
        if ((int32_t)(seen - value) >= 0) break;
        if (global_timer_ns() - t0 > timeout_ns) __trap();      // a missing peer becomes a launch failure, not a hang
        __nanosleep(200);
    }
}

// Pull a contiguous block of rows out of another rank's published buffer: every lane moves 16 bytes per load, a warp 512
// contiguous bytes, eight loads in flight per thread - NVLink wants large contiguous requests and ~2 MB in flight per GPU
// (latency ~2 us).  A handful of CTAs is enough, so the kernel runs next to the projection GEMM that consumes the previous block.
__global__ void __launch_bounds__(256) peer_pull_kernel(const uint4 *__restrict__ src, uint4 *__restrict__ dst, int64_t n_vec) {
    constexpr int kUnroll = 8;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + (kUnroll - 1) * stride < n_vec; i += kUnroll * stride) {
        uint4 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) v[u] = src[i + u * stride];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) dst[i + u * stride] = v[u];
    }
    for (; i < n_vec; i += stride) dst[i] = src[i];
}

}  // namespace tfgk

using namespace tfgk;

extern "C" int tfgk_peer_pull(const void *src, void *dst, int64_t bytes, int32_t max_ctas, void *stream) {
    TFGK_CHECK_ARG(bytes >= 0, "peer_pull: negative size");
    if (bytes == 0) return TFGK_OK;
    TFGK_CHECK_ARG(src != nullptr && dst != nullptr && bytes % 16 == 0 && aligned16(src) && aligned16(dst),
                   "peer_pull: buffers must be 16-byte aligned and a multiple of 16 bytes");
    if (max_ctas < 0) {
        // copy engine: it leaves every SM to the projection GEMM that runs beside it
        TFGK_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToDevice, as_stream(stream)));
        return TFGK_OK;
    }
    const int64_t n_vec = bytes / 16;
    int64_t blocks = ceil_div64(n_vec, 256 * 8);
    const int cap = max_ctas > 0 ? max_ctas : sm_count();
    if (blocks > cap) blocks = cap;
    peer_pull_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(static_cast<const uint4 *>(src), static_cast<uint4 *>(dst), n_vec);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

extern "C" int tfgk_peer_alloc(size_t bytes, void **ptr) {
    TFGK_CHECK_ARG(ptr != nullptr && bytes > 0, "peer_alloc: bad argument");
    TFGK_CUDA(cudaMalloc(ptr, bytes));
    TFGK_CUDA(cudaMemset(*ptr, 0, bytes));
    TFGK_CUDA(cudaDeviceSynchronize());
    return TFGK_OK;
}

extern "C" int tfgk_peer_free(void *ptr) {
    if (ptr != nullptr) TFGK_CUDA(cudaFree(ptr));
    return TFGK_OK;
}

extern "C" int tfgk_peer_export(void *ptr, void *handle_out) {
    TFGK_CHECK_ARG(ptr != nullptr && handle_out != nullptr, "peer_export: null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == TFGK_PEER_HANDLE_BYTES, "IPC handle size");
    cudaIpcMemHandle_t h;
    TFGK_CUDA(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle_out, &h, sizeof(h));
    return TFGK_OK;
}

extern "C" int tfgk_peer_open(const void *handle, void **ptr) {
    TFGK_CHECK_ARG(ptr != nullptr && handle != nullptr, "peer_open: null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    TFGK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return TFGK_OK;
}

extern "C" int tfgk_peer_close(void *ptr) {
    if (ptr != nullptr) TFGK_CUDA(cudaIpcCloseMemHandle(ptr));
    return TFGK_OK;
}

extern "C" int tfgk_peer_barrier(uint32_t *const *flags, int32_t rank, int32_t world, uint32_t value, int32_t timeout_ms,
                                 void *stream) {
    TFGK_CHECK_ARG(flags != nullptr && world >= 1 && world <= 8 && rank >= 0 && rank < world, "peer_barrier: bad argument");
    FlagTable tab;
    for (int i = 0; i < 8; ++i) tab.flags[i] = flags[i < world ? i : 0];
    for (int i = 0; i < world; ++i) TFGK_CHECK_ARG(tab.flags[i] != nullptr, "peer_barrier: null flag array for rank %d", i);
    const uint64_t timeout_ns = (uint64_t)(timeout_ms > 0 ? timeout_ms : 20000) * 1000000ull;
    peer_barrier_kernel<<<1, 32, 0, as_stream(stream)>>>(tab, rank, world, value, timeout_ns);
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}
