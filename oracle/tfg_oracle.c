/*
 * CPU ORACLE (plain C) - TEST INFRASTRUCTURE ONLY, never linked into or called by tf_geometric_b200/.
 *
 * The same restatement as oracle/tfg_oracle.py for the arithmetic core of the hot path, fast enough to check the
 * CUDA kernels at BASELINE.json's full sizes.  Loops run in EDGE ORDER with float32 accumulators and separately
 * rounded multiply/add (compile with -ffp-contract=off), i.e. exactly TensorFlow-CPU's
 * tf.math.unsorted_segment_{sum,mean,max} applied to gcn_mapper's products.
 * Parity status: "unpinned" for TensorFlow/tf_sparse kernel internals (see the header of tfg_oracle.py);
 * tests/test_oracle.py checks this file bit-for-bit against the numpy restatement.
 *
 * References (relative to tf_geometric/ of the reference, CrawlScript/tf_geometric):
 *   nn/kernel/map_reduce.py:15-16,27-28,38-42,45-73   nn/kernel/segment.py:26-33   nn/conv/gcn.py:221-222
 *   nn/conv/gat.py:73-114
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* out[N,D] = reduce_{e} (w[e] * h[col[e],:]) scattered by row[e]; reduce: 0 sum, 1 mean, 2 max. COO, edge order. */
int tfgo_aggregate_f32(const int32_t *row, const int32_t *col, const float *w, int64_t E, const float *h, int32_t N,
                       int32_t D, int reduce, float *out) {
    const int64_t total = (int64_t)N * D;
    if (reduce == 2) {
        for (int64_t i = 0; i < total; ++i) out[i] = -FLT_MAX;
    } else {
        memset(out, 0, (size_t)total * sizeof(float));
    }
    int32_t *cnt = NULL;
    if (reduce == 1) {
        cnt = (int32_t *)calloc((size_t)(N > 0 ? N : 1), sizeof(int32_t));
        if (!cnt) return 1;
    }
    for (int64_t e = 0; e < E; ++e) {
        const int32_t r = row[e], c = col[e];
        if (r < 0) continue;                        /* unsorted_segment_* drop negative ids */
        if (r >= N || c < 0) { free(cnt); return 2; }
        const float we = w ? w[e] : 1.0f;
        const float *src = h + (int64_t)c * D;
        float *dst = out + (int64_t)r * D;
        if (reduce == 2) {
            for (int32_t j = 0; j < D; ++j) { const float m = src[j] * we; if (m > dst[j]) dst[j] = m; }
        } else {
            for (int32_t j = 0; j < D; ++j) { const float m = src[j] * we; dst[j] = dst[j] + m; }
        }
        if (cnt) cnt[r] += 1;
    }
    if (reduce == 1) {
        for (int32_t r = 0; r < N; ++r) {
            const float c = (float)(cnt[r] > 1 ? cnt[r] : 1);
            float *dst = out + (int64_t)r * D;
            for (int32_t j = 0; j < D; ++j) dst[j] = dst[j] / c;
        }
        free(cnt);
    }
    return 0;
}

/* segment.py:26-33 on H interleaved columns: data/out [E,H], ids [E]. */
int tfgo_segment_softmax_f32(const float *data, const int32_t *ids, int64_t E, int32_t H, int32_t n_seg, float *out) {
    const int64_t total = (int64_t)n_seg * H;
    float *mx = (float *)malloc((size_t)(total > 0 ? total : 1) * sizeof(float));
    float *den = (float *)calloc((size_t)(total > 0 ? total : 1), sizeof(float));
    if (!mx || !den) { free(mx); free(den); return 1; }
    for (int64_t i = 0; i < total; ++i) mx[i] = -FLT_MAX;
    for (int64_t e = 0; e < E; ++e)
        for (int32_t h = 0; h < H; ++h) {
            const float v = data[e * H + h];
            float *m = &mx[(int64_t)ids[e] * H + h];
            if (v > *m) *m = v;
        }
    for (int64_t e = 0; e < E; ++e)
        for (int32_t h = 0; h < H; ++h) {
            const float p = expf(data[e * H + h] - mx[(int64_t)ids[e] * H + h]);
            out[e * H + h] = p;
            den[(int64_t)ids[e] * H + h] += p;
        }
    for (int64_t e = 0; e < E; ++e)
        for (int32_t h = 0; h < H; ++h) out[e * H + h] = out[e * H + h] / (den[(int64_t)ids[e] * H + h] + 1e-8f);
    free(mx); free(den);
    return 0;
}

/* gat.py:73-114 core given the projected Q,K [N,H*dqk] and V [N,H*dv]; edges ALREADY contain the self loops.
 * att_out (nullable) [E,H].  split=1: out [N,H*dv]; split=0: out [N,dv] = mean over heads. */
int tfgo_gat_core_f32(const int32_t *row, const int32_t *col, int64_t E, const float *Q, const float *K, const float *V,
                      int32_t N, int32_t H, int32_t dqk, int32_t dv, int split, float *att_out, float *out) {
    const int32_t A = H * dqk, VW = H * dv;
    float *score = (float *)malloc((size_t)(E > 0 ? E : 1) * H * sizeof(float));
    float *att = att_out ? att_out : (float *)malloc((size_t)(E > 0 ? E : 1) * H * sizeof(float));
    float *acc = (float *)calloc((size_t)(N > 0 ? N : 1) * VW, sizeof(float));
    if (!score || !att || !acc) return 1;
    const float scale = sqrtf((float)dqk);
    for (int64_t e = 0; e < E; ++e)
        for (int32_t h = 0; h < H; ++h) {
            const float *q = Q + (int64_t)row[e] * A + h * dqk, *k = K + (int64_t)col[e] * A + h * dqk;
            float s = 0.0f;
            for (int32_t j = 0; j < dqk; ++j) s = s + q[j] * k[j];
            score[e * H + h] = s / scale;
        }
    int rc = tfgo_segment_softmax_f32(score, row, E, H, N, att);
    if (rc == 0) {
        for (int64_t e = 0; e < E; ++e) {
            const float *v = V + (int64_t)col[e] * VW;
            float *dst = acc + (int64_t)row[e] * VW;
            for (int32_t h = 0; h < H; ++h) {
                const float a = att[e * H + h];
                for (int32_t j = 0; j < dv; ++j) { const float m = v[h * dv + j] * a; dst[h * dv + j] = dst[h * dv + j] + m; }
            }
        }
        if (split) {
            memcpy(out, acc, (size_t)N * VW * sizeof(float));
        } else {
            for (int32_t r = 0; r < N; ++r)
                for (int32_t j = 0; j < dv; ++j) {
                    float t = acc[(int64_t)r * VW + j];
                    for (int32_t h = 1; h < H; ++h) t = t + acc[(int64_t)r * VW + h * dv + j];
                    out[(int64_t)r * dv + j] = t / (float)H;
                }
        }
    }
    free(score); if (!att_out) free(att); free(acc);
    return rc;
}

/* stable sort by row -> rowptr / col_sorted / perm (integer oracle of the CSR build) */
int tfgo_csr_build(const int32_t *row, const int32_t *col, int64_t E, int32_t N, int64_t *rowptr, int32_t *col_sorted,
                   int32_t *perm) {
    memset(rowptr, 0, ((size_t)N + 1) * sizeof(int64_t));
    for (int64_t e = 0; e < E; ++e) { if (row[e] < 0 || row[e] >= N) return 2; rowptr[row[e] + 1] += 1; }
    for (int32_t r = 0; r < N; ++r) rowptr[r + 1] += rowptr[r];
    int64_t *cursor = (int64_t *)malloc(((size_t)N + 1) * sizeof(int64_t));
    if (!cursor) return 1;
    memcpy(cursor, rowptr, ((size_t)N + 1) * sizeof(int64_t));
    for (int64_t e = 0; e < E; ++e) { const int64_t p = cursor[row[e]]++; col_sorted[p] = col[e]; perm[p] = (int32_t)e; }
    free(cursor);
    return 0;
}
