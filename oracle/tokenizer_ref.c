/* ORACLE (test infrastructure, NOT product code).
 *
 * Plain-C restatement of the reference tokenizer arithmetic.  Only tests/, smoke() and bench.py's
 * cpu_baseline / --impl reference leg may load this library.
 *
 *  oracle_fps_f32        literal simulation of
 *                        third_party/torkit3d/torkit3d/csrc/cuda/sample_farthest_points_kernel.cu:8-104
 *                        (per-thread strided scan :45-73, shared-memory tree :82-95, block size from
 *                        csrc/include/utils.h:13-19 capped at 512 with a floor of 32, :132-161).
 *                        Squared distance is fmaf(dz,dz,fmaf(dy,dy,dx*dx)) with d = p_j - p_sel, the
 *                        contraction nvcc emits for the loop at :51-55 (SASS-verified).
 *  oracle_fps_closed_f32 the closed form of the same tie-break: among the
 *                        points holding the maximum min-distance pick the lexicographic minimum of
 *                        (bitrev(j mod T), j div T); repeat the previous index when the maximum is 0.
 *  oracle_knn_f32        exact brute-force K nearest (direct-difference squared distance, ties broken
 *                        by lower index), the set semantics of pc_sam/model/common.py:27-56.
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC (see oracle/build_oracle.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int block_size_for(int64_t n) {
    /* utils.h:13-19 getBlockSize(n, 512); the launch switch falls to 32 for anything below 64. */
    int64_t bs = 1;
    while (bs < n && bs < 512) bs *= 2;
    if (bs < 64) bs = 32;
    return (int)bs;
}

static inline float sqdist(const float* p, const float* q) {
    float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
    return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

int oracle_fps_f32(const float* points, int64_t B, int64_t N, int64_t G, int64_t* index) {
    if (G <= 0 || N < G) return -1;
    const int T = block_size_for(N);
    float* min_dist = (float*)malloc(sizeof(float) * (size_t)N);
    float* sd = (float*)malloc(sizeof(float) * (size_t)T);
    int* si = (int*)malloc(sizeof(int) * (size_t)T);
    for (int64_t b = 0; b < B; ++b) {
        const float* pts = points + b * N * 3;
        int64_t* out = index + b * G;
        for (int64_t j = 0; j < N; ++j) min_dist[j] = -1.0f;
        int selected = 0;
        out[0] = 0;
        for (int64_t i = 1; i < G; ++i) {
            const float* ps = pts + (int64_t)selected * 3;
            for (int t = 0; t < T; ++t) {
                float max_dist = 0.0f;
                int max_idx = selected;
                for (int64_t j = t; j < N; j += T) {
                    float dist = sqdist(pts + j * 3, ps);
                    float mdj = min_dist[j];
                    if (mdj > dist || mdj < 0.0f) {
                        min_dist[j] = dist;
                        mdj = dist;
                    }
                    if (mdj > max_dist) {
                        max_dist = mdj;
                        max_idx = (int)j;
                    }
                }
                sd[t] = max_dist;
                si[t] = max_idx;
            }
            for (int s = T / 2; s > 0; s >>= 1)
                for (int t = 0; t < s; ++t)
                    if (sd[t] < sd[t + s]) {
                        sd[t] = sd[t + s];
                        si[t] = si[t + s];
                    }
            selected = si[0];
            out[i] = selected;
        }
    }
    free(min_dist);
    free(sd);
    free(si);
    return 0;
}

static inline uint32_t bitrev(uint32_t v, int bits) {
    uint32_t r = 0;
    for (int i = 0; i < bits; ++i) r |= ((v >> i) & 1u) << (bits - 1 - i);
    return r;
}

int oracle_fps_closed_f32(const float* points, int64_t B, int64_t N, int64_t G, int64_t* index) {
    if (G <= 0 || N < G) return -1;
    const int T = block_size_for(N);
    int lg = 0;
    while ((1 << lg) < T) ++lg;
    float* min_dist = (float*)malloc(sizeof(float) * (size_t)N);
    for (int64_t b = 0; b < B; ++b) {
        const float* pts = points + b * N * 3;
        int64_t* out = index + b * G;
        for (int64_t j = 0; j < N; ++j) min_dist[j] = INFINITY;
        int64_t selected = 0;
        out[0] = 0;
        for (int64_t i = 1; i < G; ++i) {
            const float* ps = pts + selected * 3;
            float best = 0.0f;
            uint64_t best_key = ~0ull;
            int64_t best_j = selected;
            for (int64_t j = 0; j < N; ++j) {
                float d = sqdist(pts + j * 3, ps);
                if (d < min_dist[j]) min_dist[j] = d;
                float m = min_dist[j];
                uint64_t key = ((uint64_t)bitrev((uint32_t)(j % T), lg) << 40) | (uint64_t)(j / T);
                if (m > best || (m == best && m > 0.0f && key < best_key)) {
                    best = m;
                    best_key = key;
                    best_j = j;
                }
            }
            selected = best_j;
            out[i] = selected;
        }
    }
    free(min_dist);
    return 0;
}

/* K nearest keys for every query; out_idx [B,Q,K] sorted by (distance, index) ascending. */
int oracle_knn_f32(const float* query, const float* key, int64_t B, int64_t Q, int64_t N, int64_t K,
                   int64_t* out_idx, float* out_d2) {
    if (K <= 0 || K > N) return -1;
    float* bd = (float*)malloc(sizeof(float) * (size_t)K);
    int64_t* bi = (int64_t*)malloc(sizeof(int64_t) * (size_t)K);
    for (int64_t b = 0; b < B; ++b)
        for (int64_t q = 0; q < Q; ++q) {
            const float* pq = query + (b * Q + q) * 3;
            int64_t cnt = 0;
            for (int64_t j = 0; j < N; ++j) {
                float d = sqdist(key + (b * N + j) * 3, pq);
                if (cnt == K && !(d < bd[K - 1])) continue;
                int64_t pos = cnt < K ? cnt : K - 1;
                while (pos > 0 && bd[pos - 1] > d) {
                    bd[pos] = bd[pos - 1];
                    bi[pos] = bi[pos - 1];
                    --pos;
                }
                bd[pos] = d;
                bi[pos] = j;
                if (cnt < K) ++cnt;
            }
            memcpy(out_idx + (b * Q + q) * K, bi, sizeof(int64_t) * (size_t)K);
            if (out_d2) memcpy(out_d2 + (b * Q + q) * K, bd, sizeof(float) * (size_t)K);
        }
    free(bd);
    free(bi);
    return 0;
}
