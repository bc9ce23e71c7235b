// Counter-based random numbers for the training-mode kernels (dropout masks, neighbour sampling).
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), restated from the paper:
// no state is kept anywhere - element i of stream `seed` is a pure function of (seed, i), so the backward pass and the
// test-side CPU restatement regenerate the very same mask instead of storing it.
#pragma once
#include <stdint.h>

namespace tfgk {

struct Philox4 {
    uint32_t v[4];
};

__host__ __device__ __forceinline__ void philox_mulhilo(uint32_t a, uint32_t b, uint32_t &hi, uint32_t &lo) {
    const uint64_t p = (uint64_t)a * (uint64_t)b;
    hi = (uint32_t)(p >> 32);
    lo = (uint32_t)p;
}

// counter = (c0, c1, c2, c3), key = (k0, k1); ten rounds, Weyl key schedule
__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                           uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int round = 0; round < 10; ++round) {
        uint32_t hi0, lo0, hi1, lo1;
        philox_mulhilo(0xD2511F53u, c0, hi0, lo0);
        philox_mulhilo(0xCD9E8D57u, c2, hi1, lo1);
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    Philox4 r;
    r.v[0] = c0; r.v[1] = c1; r.v[2] = c2; r.v[3] = c3;
    return r;
}

// One 32-bit draw for element `idx` of (seed, stream): counter = (idx >> 2 as 64 bit, stream, 0), lane idx & 3.
__host__ __device__ __forceinline__ uint32_t random_u32(uint64_t seed, uint32_t stream, uint64_t idx) {
    const uint64_t blk = idx >> 2;
    const Philox4 r = philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), stream, 0u, (uint32_t)seed, (uint32_t)(seed >> 32));
    return r.v[idx & 3];
}

// uniform in [0, 1) with 24 random bits (every value is exactly representable in fp32)
__host__ __device__ __forceinline__ float random_uniform(uint64_t seed, uint32_t stream, uint64_t idx) {
    return (float)(random_u32(seed, stream, idx) >> 8) * (1.0f / 16777216.0f);
}

// integer in [0, n) by multiply-shift
__host__ __device__ __forceinline__ uint32_t random_below(uint64_t seed, uint32_t stream, uint64_t idx, uint32_t n) {
    return (uint32_t)(((uint64_t)random_u32(seed, stream, idx) * (uint64_t)n) >> 32);
}

// 64-bit integer in [0, n): u = random_u32(2 idx) | random_u32(2 idx + 1) << 32 (two lanes of one Philox block),
// k = high 64 bits of u * n
__host__ __device__ __forceinline__ uint64_t random_below64(uint64_t seed, uint32_t stream, uint64_t idx, uint64_t n) {
    const uint64_t blk = idx >> 1;
    const Philox4 r = philox4x32_10((uint32_t)blk, (uint32_t)(blk >> 32), stream, 0u, (uint32_t)seed, (uint32_t)(seed >> 32));
    const int l = (int)(idx & 1) * 2;
    const uint64_t u = (uint64_t)r.v[l] | ((uint64_t)r.v[l + 1] << 32);
#ifdef __CUDA_ARCH__
    return __umul64hi(u, n);
#else
    return (uint64_t)(((unsigned __int128)u * n) >> 64);
#endif
}

// splitmix64's output function (Steele, Lea and Flood, "Fast splittable pseudorandom number generators", OOPSLA'14):
// the same mix as tf_geometric_b200/_rng.py applies to its keys
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// key of draw `slot` of a captured region whose device-resident base is `base` (include/tfgk.h, "device keys")
__host__ __device__ __forceinline__ uint64_t device_key(uint64_t base, uint64_t slot) {
    return splitmix64(base + 0x9E3779B97F4A7C15ull * (slot + 1));
}

}  // namespace tfgk
