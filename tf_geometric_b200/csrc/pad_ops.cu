// K9: the padded row gather of lstm_graph_sage (nn/conv/graph_sage.py:319-337) and convert_x_to_3d
// (utils/graph_utils.py:215-249), and the backward of the latter.
//
// Both reference functions build out[r, j] = the j-th row of group r in stable input order, zero-padded to K, by
// scattering an index matrix and gathering from a copy of x with one zero row appended.  Here the groups are the rows of
// a CSR (stable by construction), so the j-th member of row r is slot rowptr[r] + j and no index matrix is needed.
//
// Work split: every CSR row produces exactly K output rows (padded or not), so the work per row is uniform; one group of
// G lanes owns one CSR row at a time (grid-stride) and walks its K output rows U at a time: U src ids are loaded, then U
// X rows are in flight, then U output rows are stored.  Lanes of a group split the D columns into vectors of VEC floats.
// Nothing is reduced: a pure copy, bit-exact, every output row written once.
//
// The unpad kernel is the transpose of the same walk for src = perm: slot p of row r sends G[r, j] (or zeros when the
// row was truncated, j >= K) to out[perm[p]], so every input row receives exactly one write and no atomics are needed.
#include "common.cuh"

namespace tfgk {
namespace {

constexpr int kPadThreads = 256;
constexpr int kPadUnroll = 4;

template <int VEC>
__device__ __forceinline__ void copy_vec(const float *__restrict__ s, float *__restrict__ d) {
    if constexpr (VEC == 4) {
        *reinterpret_cast<float4 *>(d) = __ldg(reinterpret_cast<const float4 *>(s));
    } else {
        *d = __ldg(s);
    }
}

template <int VEC>
__device__ __forceinline__ void fill_vec(float *__restrict__ d, float v) {
    if constexpr (VEC == 4) {
        *reinterpret_cast<float4 *>(d) = make_float4(v, v, v, v);
    } else {
        *d = v;
    }
}

template <int VEC, int G>
__global__ void __launch_bounds__(kPadThreads) pad_rows_kernel(
    const int64_t *__restrict__ rowptr, const int32_t *__restrict__ src, int32_t R, int32_t K, int step_major,
    const float *__restrict__ X, int64_t ldx, int32_t NX, int32_t D, float *__restrict__ out,
    int32_t *__restrict__ slot_out) {
    constexpr int U = kPadUnroll;
    const int gl = threadIdx.x & (G - 1);
    const int64_t group = ((int64_t)blockIdx.x * kPadThreads + threadIdx.x) / G;
    const int64_t n_groups = ((int64_t)gridDim.x * kPadThreads) / G;
    const int64_t D64 = D;
    for (int64_t r = group; r < R; r += n_groups) {
        const int64_t p0 = rowptr[r];
        const int64_t deg = rowptr[r + 1] - p0;
        const int32_t kept = (int32_t)(deg < K ? deg : K);
        if (slot_out != nullptr) {
            for (int64_t j = gl; j < deg; j += G)
                slot_out[p0 + j] = j < K ? (int32_t)(step_major ? j * R + r : r * K + j) : -1;
        }
        for (int32_t j0 = 0; j0 < K; j0 += U) {
            const float *px[U];
            float *po[U];
            int state[U];                          // 0: skip (j >= K), 1: copy, 2: zeros, 3: NaN (bad src id)
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t j = j0 + u;
                po[u] = out + (step_major ? j * R + r : r * K + j) * D64;
                px[u] = X;
                state[u] = j < K ? 2 : 0;
                if (j < kept) {
                    const int32_t s = __ldg(src + p0 + j);
                    if (s >= 0 && s < NX) {
                        px[u] = X + (int64_t)s * ldx;
                        state[u] = 1;
                    } else {
                        state[u] = 3;
                    }
                }
            }
            for (int c = gl * VEC; c < D; c += G * VEC) {
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (state[u] == 1) copy_vec<VEC>(px[u] + c, po[u] + c);
                    else if (state[u] == 2) fill_vec<VEC>(po[u] + c, 0.0f);
                    else if (state[u] == 3) fill_vec<VEC>(po[u] + c, __int_as_float(0x7fc00000));
                }
            }
        }
    }
}

template <int VEC, int G>
__global__ void __launch_bounds__(kPadThreads) unpad_rows_kernel(
    const int64_t *__restrict__ rowptr, const int32_t *__restrict__ perm, int32_t R, int32_t K,
    const float *__restrict__ Gm, int32_t D, float *__restrict__ out, int64_t n_out) {
    constexpr int U = kPadUnroll;
    const int gl = threadIdx.x & (G - 1);
    const int64_t group = ((int64_t)blockIdx.x * kPadThreads + threadIdx.x) / G;
    const int64_t n_groups = ((int64_t)gridDim.x * kPadThreads) / G;
    const int64_t D64 = D;
    for (int64_t r = group; r < R; r += n_groups) {
        const int64_t p0 = rowptr[r];
        const int64_t deg = rowptr[r + 1] - p0;
        for (int64_t j0 = 0; j0 < deg; j0 += U) {
            const float *pg[U];
            float *po[U];
            int state[U];                          // 0: skip, 1: copy, 2: zeros (truncated slot)
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t j = j0 + u;
                pg[u] = Gm + ((int64_t)r * K + j) * D64;
                po[u] = out;
                state[u] = 0;
                if (j < deg) {
                    const int32_t d = __ldg(perm + p0 + j);
                    if (d >= 0 && d < n_out) {
                        po[u] = out + (int64_t)d * D64;
                        state[u] = j < K ? 1 : 2;
                    }
                }
            }
            for (int c = gl * VEC; c < D; c += G * VEC) {
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    if (state[u] == 1) copy_vec<VEC>(pg[u] + c, po[u] + c);
                    else if (state[u] == 2) fill_vec<VEC>(po[u] + c, 0.0f);
                }
            }
        }
    }
}

// lanes per group: the smallest power of two covering the row's vectors, at most a warp
inline int group_lanes(int32_t vectors) {
    int g = 1;
    while (g < 32 && g < vectors) g <<= 1;
    return g;
}

inline unsigned pad_grid(int64_t R, int G) {
    const int64_t want = ceil_div64(R * G, kPadThreads);
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)(want < 1 ? 1 : (want < cap ? want : cap));
}

template <int VEC>
int launch_pad(const int64_t *rowptr, const int32_t *src, int32_t R, int32_t K, int step_major, const float *X,
               int64_t ldx, int32_t NX, int32_t D, float *out, int32_t *slot_out, cudaStream_t st) {
    const int G = group_lanes(D / VEC);
    const unsigned blocks = pad_grid(R, G);
#define TFGK_PAD(GL) \
    pad_rows_kernel<VEC, GL><<<blocks, kPadThreads, 0, st>>>(rowptr, src, R, K, step_major, X, ldx, NX, D, out, slot_out)
    switch (G) {
        case 1: TFGK_PAD(1); break;
        case 2: TFGK_PAD(2); break;
        case 4: TFGK_PAD(4); break;
        case 8: TFGK_PAD(8); break;
        case 16: TFGK_PAD(16); break;
        default: TFGK_PAD(32); break;
    }
#undef TFGK_PAD
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

template <int VEC>
int launch_unpad(const int64_t *rowptr, const int32_t *perm, int32_t R, int32_t K, const float *Gm, int32_t D, float *out,
                 int64_t n_out, cudaStream_t st) {
    const int G = group_lanes(D / VEC);
    const unsigned blocks = pad_grid(R, G);
#define TFGK_UNPAD(GL) unpad_rows_kernel<VEC, GL><<<blocks, kPadThreads, 0, st>>>(rowptr, perm, R, K, Gm, D, out, n_out)
    switch (G) {
        case 1: TFGK_UNPAD(1); break;
        case 2: TFGK_UNPAD(2); break;
        case 4: TFGK_UNPAD(4); break;
        case 8: TFGK_UNPAD(8); break;
        case 16: TFGK_UNPAD(16); break;
        default: TFGK_UNPAD(32); break;
    }
#undef TFGK_UNPAD
    TFGK_LAUNCH_CHECK();
    return TFGK_OK;
}

}  // namespace
}  // namespace tfgk

using namespace tfgk;

extern "C" {

int tfgk_pad_rows_f32(const int64_t *rowptr, const int32_t *src, int32_t R, int32_t K, int layout, const float *X,
                      int64_t ldx, int32_t NX, int32_t D, float *out, int32_t *slot_out, void *stream) {
    TFGK_CHECK_ARG(R >= 0 && K >= 0 && D >= 0 && NX >= 0, "pad_rows: negative R, K, D or NX");
    TFGK_CHECK_ARG(layout == TFGK_PAD_ROW_MAJOR || layout == TFGK_PAD_STEP_MAJOR, "pad_rows: unknown layout %d", layout);
    TFGK_CHECK_ARG(slot_out == nullptr || (int64_t)K * R < (1ll << 31),
                   "pad_rows: K * R = %lld does not fit the int32 slot index", (long long)K * R);
    if (R == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && src, "pad_rows: null rowptr or src");
    TFGK_CHECK_ARG((int64_t)K * D == 0 || out, "pad_rows: null out");
    TFGK_CHECK_ARG(D == 0 || NX == 0 || (X && ldx >= D), "pad_rows: bad X (ldx %lld, D %d)", (long long)ldx, D);
    cudaStream_t st = as_stream(stream);
    const int step = layout == TFGK_PAD_STEP_MAJOR;
    if (D % 4 == 0 && ldx % 4 == 0 && aligned16(X) && aligned16(out))
        return launch_pad<4>(rowptr, src, R, K, step, X, ldx, NX, D, out, slot_out, st);
    return launch_pad<1>(rowptr, src, R, K, step, X, ldx, NX, D, out, slot_out, st);
}

int tfgk_unpad_rows_f32(const int64_t *rowptr, const int32_t *perm, int32_t R, int32_t K, const float *G, int32_t D,
                        float *out, int64_t n_out, void *stream) {
    TFGK_CHECK_ARG(R >= 0 && K >= 0 && D >= 0 && n_out >= 0, "unpad_rows: negative R, K, D or n_out");
    if (R == 0 || D == 0 || n_out == 0) return TFGK_OK;
    TFGK_CHECK_ARG(rowptr && perm && out && (K == 0 || G), "unpad_rows: null rowptr, perm, G or out");
    cudaStream_t st = as_stream(stream);
    if (D % 4 == 0 && (K == 0 || aligned16(G)) && aligned16(out))
        return launch_unpad<4>(rowptr, perm, R, K, G, D, out, n_out, st);
    return launch_unpad<1>(rowptr, perm, R, K, G, D, out, n_out, st);
}

}  // extern "C"
