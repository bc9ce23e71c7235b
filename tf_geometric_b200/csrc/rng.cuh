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

// ---- weighted draws (include/tfgk.h, "weighted block sampler") ----------------------------------------------------
// Every double operation below is rounded on its own (__dmul_rn and friends on the device, plain SSE2 arithmetic on the
// host), so that no contraction into an FMA can change a bit and numpy float64 restates the routine exactly.
__host__ __device__ __forceinline__ double rn_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ double rn_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ __forceinline__ double rn_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double rn_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ __forceinline__ uint64_t dbits(double x) {
    union { double d; uint64_t u; } c;
    c.d = x;
    return c.u;
}
__host__ __device__ __forceinline__ double dfrom(uint64_t u) {
    union { double d; uint64_t u; } c;
    c.u = u;
    return c.d;
}

// ln(u) for a positive normal double u, not the device libm: u = 2^e m with m in [sqrt(2)/2, sqrt(2)] by exact exponent
// extraction, f = m - 1 (exact), s = f / (2 + f) and ln(m) = f - f^2/2 + s (f^2/2 + R(s^2)), with the degree-14 minimax
// polynomial R and the split ln 2 of the classic fdlibm log (Sun Microsystems, 1993).  Within 2 ulp of math.log on (0, 1]
// (tests/test_weighted_sampling_host.py).
__host__ __device__ __forceinline__ double log_rn(double u) {
    const double Lg1 = dfrom(0x3FE5555555555593ull), Lg2 = dfrom(0x3FD999999997FA04ull),
                 Lg3 = dfrom(0x3FD2492494229359ull), Lg4 = dfrom(0x3FCC71C51D8E78AFull),
                 Lg5 = dfrom(0x3FC7466496CB03DEull), Lg6 = dfrom(0x3FC39A09D078C69Full),
                 Lg7 = dfrom(0x3FC2F112DF3E5244ull);
    const double ln2_hi = dfrom(0x3FE62E42FEE00000ull), ln2_lo = dfrom(0x3DEA39EF35793C76ull);
    const uint64_t b = dbits(u);
    int e = (int)(b >> 52) - 1023;
    uint64_t mb = (b & 0x000FFFFFFFFFFFFFull) | 0x3FF0000000000000ull;
    if (mb > 0x3FF6A09E667F3BCDull) {                // m > sqrt(2): halve it (exact) and carry the factor into e
        mb -= 1ull << 52;
        e += 1;
    }
    const double f = rn_sub(dfrom(mb), 1.0);
    const double s = rn_div(f, rn_add(2.0, f));
    const double z = rn_mul(s, s), w = rn_mul(z, z);
    const double t1 = rn_mul(w, rn_add(Lg2, rn_mul(w, rn_add(Lg4, rn_mul(w, Lg6)))));
    const double t2 = rn_mul(z, rn_add(Lg1, rn_mul(w, rn_add(Lg3, rn_mul(w, rn_add(Lg5, rn_mul(w, Lg7)))))));
    const double R = rn_add(t2, t1);
    const double hfsq = rn_mul(0.5, rn_mul(f, f));
    const double dk = (double)e;
    return rn_sub(rn_mul(dk, ln2_hi),
                  rn_sub(rn_sub(hfsq, rn_add(rn_mul(s, rn_add(hfsq, R)), rn_mul(dk, ln2_lo))), f));
}

// The Efraimidis-Spirakis key of entry v (virtual position) of global row r, draw j, weight w > 0: one Philox block
// with counter (v, r, stream, j), u = ((lanes 0 | 1 << 32) >> 11) + 1) 2^-53 in (0, 1], E = -ln(u) / w in double.
// Returned as the bits of E with the sign cleared (E = -0.0 at u = 1): non-negative doubles order as their bits.
__host__ __device__ __forceinline__ uint64_t weighted_key(uint64_t seed, uint32_t stream, uint32_t v, uint32_t r,
                                                          uint32_t j, float w) {
    const Philox4 x = philox4x32_10(v, r, stream, j, (uint32_t)seed, (uint32_t)(seed >> 32));
    const uint64_t u64 = (uint64_t)x.v[0] | ((uint64_t)x.v[1] << 32);
    const double u = rn_mul((double)((u64 >> 11) + 1), 1.1102230246251565e-16);      // 2^-53
    return dbits(rn_div(-log_rn(u), (double)w)) & 0x7FFFFFFFFFFFFFFFull;
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
