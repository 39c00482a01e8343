// kNN grouping and 3-NN interpolation weights for sm_90a.
//
// Replaces pc_sam/model/common.py: knn_points (:27-56, torch.cdist + torch.topk), the gathers of
// KNNGrouper.forward / group_with_centers_and_knn (:99-123, :126-187) and compute_interp_weights
// (:238-255).  The reference materialises the [B,G,N] distance matrix (64 MiB per cloud at
// G=512,N=32768); here nothing but xyz is read and only the K winners are written.
//
// psam_knn_f32: one CTA per group of 1 / 2 / 4 query centres (see knn_kernel): sample bound -> one branch-free sweep of all
// keys recording hit bits in registers -> exact re-test of the hits -> exact K-th by radix select, ties by lower key
// index, output sorted by (distance, index) so the result is deterministic.
// Distances are the direct-difference form fmaf(dz,dz,fmaf(dy,dy,dx*dx)) (exact for coincident points).
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {

constexpr int KNN_THREADS = 256;
constexpr int KNN_MAX_CAP = 16384;     // candidate list capacity limit
constexpr int KNN_MAX_SAMPLE = 16384;  // sample size limit (bounds the cost of phase A)

__device__ __forceinline__ float sqdist3(float x, float y, float z, float cx, float cy, float cz) {
    const float dx = x - cx, dy = y - cy, dz = z - cz;
    return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

// Block-wide sum of per-thread counts through one shared counter slot (one __syncthreads).
__device__ __forceinline__ int block_count(int c, int* slot) {
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(slot, c);
    __syncthreads();
    return *slot;
}

__device__ __forceinline__ void zero_counters(int* cnt) {
    __syncthreads();
    if (threadIdx.x < 64) cnt[threadIdx.x] = 0;
    __syncthreads();
}

// Radix select: bit pattern of the k-th smallest (1-indexed) of vals[0..n), non-negative floats compared as unsigned.
// Three histogram passes over the digits [30:20], [19:10], [9:0] (2048 / 1024 / 1024 bins in shared memory) replace the 31
// counting passes of the bitwise bisection; each pass: histogram of the elements that match the prefix decided so far,
// block-wide scan of the bins, the thread whose bin range crosses k publishes the digit.  `hist` holds KNN_HIST ints.
constexpr int KNN_HIST = 2048;

__device__ uint32_t kth_smallest_radix(const float* vals, int n, int k, int* hist) {
    __shared__ int s_warp_tot[KNN_THREADS / 32];
    __shared__ int s_digit, s_krem;
    uint32_t prefix = 0, mask = 0;
    int kk = k;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = pass == 0 ? 20 : (pass == 1 ? 10 : 0);
        const int nb = pass == 0 ? 2048 : 1024;
        __syncthreads();
        for (int i = tid; i < nb; i += KNN_THREADS) hist[i] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += KNN_THREADS) {
            const uint32_t u = __float_as_uint(vals[i]);
            if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & (uint32_t)(nb - 1)], 1);
        }
        __syncthreads();
        // each thread owns nb/256 consecutive bins
        const int per = nb / KNN_THREADS;
        int local = 0;
        for (int t = 0; t < per; ++t) local += hist[tid * per + t];
        int incl = local;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_warp_tot[warp] = incl;
        __syncthreads();
        int before = incl - local;
        for (int w = 0; w < warp; ++w) before += s_warp_tot[w];
        if (before < kk && kk <= before + local) {  // exactly one thread: the k-th element falls into one of its bins
            int run = before;
            for (int t = 0; t < per; ++t) {
                const int h = hist[tid * per + t];
                if (kk <= run + h) {
                    s_digit = tid * per + t;
                    s_krem = kk - run;
                    break;
                }
                run += h;
            }
        }
        __syncthreads();
        prefix |= (uint32_t)s_digit << shift;
        mask |= (uint32_t)(nb - 1) << shift;
        kk = s_krem;
    }
    __syncthreads();
    return prefix;
}

// Upper bound of the k-th smallest of vals[0..n) from ONE histogram pass over the digit [30:20] (exponent + 3 mantissa bits):
// the upper edge of the bin that holds the k-th element.  At most 12.5 % above the k-th value - good enough for the
// candidate filter of phase A (a looser tau only admits a few more candidates), at a third of the passes and barriers of
// the exact select.
__device__ uint32_t kth_upper_bound_from_hist(const int* hist, int k) {
    __shared__ int s_warp_tot2[KNN_THREADS / 32];
    __shared__ int s_digit2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int nb = 2048, per = nb / KNN_THREADS;
    __syncthreads();  // histogram complete; previous use of the static slots finished
    int local = 0;
#pragma unroll
    for (int t = 0; t < per; ++t) local += hist[tid * per + t];
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp_tot2[warp] = incl;
    __syncthreads();
    int before = incl - local;
    for (int w = 0; w < warp; ++w) before += s_warp_tot2[w];
    if (before < k && k <= before + local) {  // exactly one thread
        int run = before;
        for (int t = 0; t < per; ++t) {
            run += hist[tid * per + t];
            if (k <= run) {
                s_digit2 = tid * per + t;
                break;
            }
        }
    }
    __syncthreads();
    const uint32_t edge = ((uint32_t)s_digit2 << 20) | 0xFFFFFu;
    return edge < 0x7F800000u ? edge : 0x7F7FFFFFu;  // never a NaN / inf pattern: the sweep compares tau as a float
}

// One CTA serves C consecutive query centres of one cloud.
//   A. per centre: squared distances to a strided SAMPLE of the keys -> exact K-th smallest of the sample (radix select)
//      = tau_c, an upper bound of the true K-th distance.
//   B. ONE sweep over all keys for the C centres together (each 128-bit key load feeds 4 x C pair tests).  The test is a
//      3-FMA filter |p|^2 + |c|^2 - 2 p.c, biased low by 2e-6 (|p|^2 + |c|^2) so that it can only over-accept; hits are only
//      recorded as one bit per (point, centre) in registers - no branch, no shared-memory traffic in the hot loop
//      (round 1 branched into a shared-memory append for every point: 45 of its 61 thread-instructions per pair).
//      After each super-tile of 32 quads per thread the set bits are revisited: exact direct-difference distance
//      (bit-identical to the oracle), exact test against tau_c, append to the centre's candidate list.
//   C. per centre: exact K-th among the candidates, ties at the K-th distance by lower key index, output sorted by
//      (distance, index).  Candidate overflow (adversarial duplicates) falls back to exact bisection over all keys.
template <int C>
struct KnnSmem {
    float* s_sample;  // [sample_cap] (>= 2K); reused as the final list of each centre
    float* c_d2;      // [C][cap]
    int* c_idx;       // [C][cap]
    int* cnt;         // [64]
    int* hist;        // [KNN_HIST]
};

constexpr int KNN_TILE_QUADS = 32;  // quads (4 keys) per thread and super-tile: 4 x 32 hit bits = 4 registers per centre

template <int C>
__global__ void __launch_bounds__(KNN_THREADS)
knn_kernel(const float* __restrict__ query, const float* __restrict__ key, int Q, int N, int K, int sample_stride,
           int sample_cap, int cap, long long* __restrict__ idx_out, float* __restrict__ d2_out) {
    pdl_prologue();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* s_sample = reinterpret_cast<float*>(smem_raw);       // [sample_cap = 2K]: the final list of the centre being finished
    float* c_d2_all = s_sample + sample_cap;                    // [C][cap]
    int* c_idx_all = reinterpret_cast<int*>(c_d2_all + (size_t)C * cap);  // [C][cap]
    int* cnt = c_idx_all + (size_t)C * cap;                     // [64]
    int* hist = cnt + 64;                                       // [C][KNN_HIST]: per-centre sample histograms (phase A); [0] reused by the selects
    __shared__ int s_ncand[C], s_overflow[C], s_nsel;
    __shared__ uint32_t s_tau[C];
    __shared__ int s_wcnt[KNN_THREADS / 32];

    const int b = blockIdx.y, q0 = blockIdx.x * C, tid = threadIdx.x, lane = tid & 31;
    key += (size_t)b * N * 3;
    float cx[C], cy[C], cz[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int q = min(q0 + c, Q - 1);  // a ragged last group recomputes the last centre (results not stored twice)
        const float* pq = query + ((size_t)b * Q + q) * 3;
        cx[c] = pq[0], cy[c] = pq[1], cz[c] = pq[2];
    }
    if (tid < C) s_ncand[tid] = 0, s_overflow[tid] = 0;
    if (tid == 0) s_nsel = 0;
    zero_counters(cnt);

    // ---- A. sample bound per centre ------------------------------------------------------------
    // the strided sample is loaded ONCE for the C centres, eight points per thread at a time with all 24 loads in flight; its
    // squared distances go straight into one 2048-bin histogram per centre (top 11 bits) - the sample itself is never stored
    const int ns = (N + sample_stride - 1) / sample_stride;
    for (int i = tid; i < C * KNN_HIST; i += KNN_THREADS) hist[i] = 0;
    __syncthreads();
    for (int i0 = 0; i0 < ns; i0 += 8 * KNN_THREADS) {
        float sx[8], sy[8], sz[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * KNN_THREADS + tid;
            const size_t j = (size_t)min(i, ns - 1) * sample_stride;
            sx[u] = key[j * 3], sy[u] = key[j * 3 + 1], sz[u] = key[j * 3 + 2];
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * KNN_THREADS + tid;
#pragma unroll
            for (int c = 0; c < C; ++c) {
                if (i < ns) atomicAdd(&hist[c * KNN_HIST + (__float_as_uint(sqdist3(sx[u], sy[u], sz[u], cx[c], cy[c], cz[c])) >> 20)], 1);
            }
        }
    }
#pragma unroll 1
    for (int c = 0; c < C; ++c) {
        const uint32_t t = kth_upper_bound_from_hist(hist + c * KNN_HIST, K);
        if (tid == 0) s_tau[c] = t;
    }
    __syncthreads();
    uint32_t tau[C];
#pragma unroll
    for (int c = 0; c < C; ++c) tau[c] = s_tau[c];

    auto append = [&](int c, float d, int j) {
        const int pos = atomicAdd(&s_ncand[c], 1);
        if (pos < cap) {
            c_d2_all[(size_t)c * cap + pos] = d;
            c_idx_all[(size_t)c * cap + pos] = j;
        } else {
            s_overflow[c] = 1;
        }
    };

    // ---- B. the sweep ----------------------------------------------------------------------------
    int n_vec = 0;
    if ((N & 3) == 0 && (reinterpret_cast<uintptr_t>(key) & 15) == 0) {
        n_vec = N;
        const float4* key4 = reinterpret_cast<const float4*>(key);
        const int nquad = N >> 2;
        constexpr float SHRINK = 1.0f - 2e-6f;  // the filter may only over-accept: bias the positive part low
        float m2x[C], m2y[C], m2z[C], cn[C], tauf[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            m2x[c] = -2.0f * cx[c], m2y[c] = -2.0f * cy[c], m2z[c] = -2.0f * cz[c];
            cn[c] = fmaf(cz[c], cz[c], fmaf(cy[c], cy[c], cx[c] * cx[c])) * SHRINK;
            tauf[c] = __uint_as_float(tau[c]);
        }
        for (int qt = 0; qt < nquad; qt += KNN_TILE_QUADS * KNN_THREADS) {
            uint32_t bits[C][4];
#pragma unroll
            for (int c = 0; c < C; ++c) bits[c][0] = bits[c][1] = bits[c][2] = bits[c][3] = 0u;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
#pragma unroll
                for (int i8 = 0; i8 < 8; ++i8) {
                    const int qd = qt + (w * 8 + i8) * KNN_THREADS + tid;
                    if (qd < nquad) {
                        const float4 a = key4[(size_t)qd * 3], bq = key4[(size_t)qd * 3 + 1], cq = key4[(size_t)qd * 3 + 2];
                        const float px[4] = {a.x, a.w, bq.z, cq.y}, py[4] = {a.y, bq.x, bq.w, cq.z}, pz[4] = {a.z, bq.y, cq.x, cq.w};
                        float pn[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) pn[u] = fmaf(pz[u], pz[u], fmaf(py[u], py[u], px[u] * px[u])) * SHRINK;
#pragma unroll
                        for (int c = 0; c < C; ++c) {
                            uint32_t m = 0u;
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const float f = fmaf(px[u], m2x[c], fmaf(py[u], m2y[c], fmaf(pz[u], m2z[c], pn[u] + cn[c])));
                                m |= (f <= tauf[c]) ? (1u << u) : 0u;
                            }
                            bits[c][w] |= m << (i8 * 4);
                        }
                    }
                }
            }
            // revisit the recorded hits: exact distance, exact test, append
#pragma unroll
            for (int c = 0; c < C; ++c) {
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    uint32_t m = bits[c][w];
                    while (m) {
                        const int bpos = __ffs(m) - 1;
                        m &= m - 1u;
                        const int it = w * 8 + (bpos >> 2);
                        const int j = (qt + it * KNN_THREADS + tid) * 4 + (bpos & 3);
                        const float d = sqdist3(key[(size_t)j * 3], key[(size_t)j * 3 + 1], key[(size_t)j * 3 + 2], cx[c], cy[c], cz[c]);
                        if (__float_as_uint(d) <= tau[c]) append(c, d, j);
                    }
                }
            }
        }
    }
    for (int j0 = n_vec; j0 < N; j0 += KNN_THREADS) {  // unaligned / ragged clouds: plain point-wise sweep
        const int j = j0 + tid;
        if (j < N) {
            const float x = key[(size_t)j * 3], y = key[(size_t)j * 3 + 1], z = key[(size_t)j * 3 + 2];
#pragma unroll
            for (int c = 0; c < C; ++c) {
                const float d = sqdist3(x, y, z, cx[c], cy[c], cz[c]);
                if (__float_as_uint(d) <= tau[c]) append(c, d, j);
            }
        }
    }
    __syncthreads();

    // ---- per centre: overflow fallback, then C ------------------------------------------------------
#pragma unroll 1
    for (int c = 0; c < C; ++c) {
        if (q0 + c >= Q) break;  // uniform
        const int q = q0 + c;
        float* c_d2 = c_d2_all + (size_t)c * cap;
        int* c_idx = c_idx_all + (size_t)c * cap;
        const float ccx = cx[c], ccy = cy[c], ccz = cz[c];
        int ncand = min(s_ncand[c], cap);
        if (s_overflow[c]) {
            // ---- fallback: exact bisection over the whole key set (distances recomputed per pass) ----
            zero_counters(cnt);
            uint32_t res = 0;
            for (int bit = 30; bit >= 0; --bit) {
                const uint32_t cand = res | (1u << bit);
                int n = 0;
                for (int j = tid; j < N; j += KNN_THREADS)
                    n += (__float_as_uint(sqdist3(key[(size_t)j * 3], key[(size_t)j * 3 + 1], key[(size_t)j * 3 + 2], ccx, ccy, ccz)) < cand);
                if (block_count(n, &cnt[bit]) < K) res = cand;
            }
            __syncthreads();
            if (tid == 0) s_ncand[c] = 0;
            __syncthreads();
            const uint32_t tx = res;  // the exact K-th distance
            // strictly-below first (fewer than K of them), then ties in ascending key index until full
            for (int pass = 0; pass < 2; ++pass) {
                for (int j0 = 0; j0 < N; j0 += KNN_THREADS) {
                    const int j = j0 + tid;
                    float d = 0.f;
                    bool hit = false;
                    if (j < N) {
                        d = sqdist3(key[(size_t)j * 3], key[(size_t)j * 3 + 1], key[(size_t)j * 3 + 2], ccx, ccy, ccz);
                        const uint32_t u = __float_as_uint(d);
                        hit = pass == 0 ? (u < tx) : (u == tx);
                    }
                    const uint32_t m = __ballot_sync(0xffffffffu, hit);
                    if (lane == 0) s_wcnt[tid >> 5] = __popc(m);
                    __syncthreads();
                    int base = s_ncand[c];
                    for (int w = 0; w < (tid >> 5); ++w) base += s_wcnt[w];
                    if (hit) {
                        const int pos = base + __popc(m & ((1u << lane) - 1u));
                        if (pos < cap) {
                            c_d2[pos] = d;
                            c_idx[pos] = j;
                        }
                    }
                    __syncthreads();
                    if (tid == 0) {
                        int tot = 0;
                        for (int w = 0; w < KNN_THREADS / 32; ++w) tot += s_wcnt[w];
                        s_ncand[c] = min(s_ncand[c] + tot, cap);
                    }
                    __syncthreads();
                    if (s_ncand[c] >= cap) break;
                }
            }
            ncand = s_ncand[c];
        }

        // ---- C. exact K-th among candidates; ties at the K-th distance by lower key index -----------
        zero_counters(cnt);
        if (tid == 0) s_nsel = 0;
        const uint32_t kth = kth_smallest_radix(c_d2, ncand, K, hist);
        int c_lt = 0, c_le = 0;
        for (int i = tid; i < ncand; i += KNN_THREADS) {
            const uint32_t u = __float_as_uint(c_d2[i]);
            c_lt += (u < kth);
            c_le += (u <= kth);
        }
        c_lt = block_count(c_lt, &cnt[32]);
        c_le = block_count(c_le, &cnt[33]);
        uint32_t idx_thr = 0xFFFFFFFFu;  // keep ties with index <= idx_thr
        if (c_le > K) {
            const int need = K - c_lt;  // >= 1
            uint32_t res = 0;           // `need`-th smallest index among the ties
            for (int bit = 30; bit >= 0; --bit) {
                const uint32_t cand = res | (1u << bit);
                int n = 0;
                for (int i = tid; i < ncand; i += KNN_THREADS)
                    n += (__float_as_uint(c_d2[i]) == kth && (uint32_t)c_idx[i] < cand);
                if (block_count(n, &cnt[bit]) < need) res = cand;
            }
            idx_thr = res;
        }
        __syncthreads();
        // compact the K winners into the sample area (free after phase A), then order them by (d2, index)
        float* f_d2 = s_sample;
        int* f_idx = reinterpret_cast<int*>(s_sample + K);
        for (int i0 = 0; i0 < ncand; i0 += KNN_THREADS) {
            const int i = i0 + tid;
            bool hit = false;
            if (i < ncand) {
                const uint32_t u = __float_as_uint(c_d2[i]);
                hit = (u < kth) || (u == kth && (uint32_t)c_idx[i] <= idx_thr);
            }
            const uint32_t m = __ballot_sync(0xffffffffu, hit);
            if (m) {
                int base = 0;
                if (lane == 0) base = atomicAdd(&s_nsel, __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (hit) {
                    const int pos = base + __popc(m & ((1u << lane) - 1u));
                    if (pos < K) {
                        f_d2[pos] = c_d2[i];
                        f_idx[pos] = c_idx[i];
                    }
                }
            }
        }
        __syncthreads();
        // rank of every winner among the K by (d2, index): four lanes per winner, each over a quarter of the list
        for (int i0 = 0; i0 < K; i0 += KNN_THREADS / 4) {
            const int i = i0 + (tid >> 2), part = tid & 3;
            int rank = 0;
            uint32_t u = 0;
            int ji = 0;
            if (i < K) {
                u = __float_as_uint(f_d2[i]);
                ji = f_idx[i];
                for (int t = part; t < K; t += 4) {
                    const uint32_t ut = __float_as_uint(f_d2[t]);
                    rank += (ut < u) || (ut == u && f_idx[t] < ji);
                }
            }
            rank += __shfl_xor_sync(0xffffffffu, rank, 1);
            rank += __shfl_xor_sync(0xffffffffu, rank, 2);
            if (i < K && part == 0) {
                idx_out[((size_t)b * Q + q) * K + rank] = ji;
                if (d2_out) d2_out[((size_t)b * Q + q) * K + rank] = __uint_as_float(u);
            }
        }
        __syncthreads();  // f_d2 / f_idx (the sample area) are reused by the next centre
    }
}

// groups[b2, g, k, :] = [ (xyz[b, idx] - centers[b, g]) / radius , feats[b2, idx, 0:C] (, feats[b2, idx] - feats[b2, center_idx[b, g]]) ]
// (b = b2 / rep; the third part only with center_idx: centralize_features=True, common.py:116-118 / :181-185)
__global__ void group_gather_kernel(const float* __restrict__ xyz, const float* __restrict__ feats,
                                    const float* __restrict__ centers, const long long* __restrict__ knn_idx,
                                    const long long* __restrict__ center_idx, int B2,
                                    int rep, int N, int G, int K, int C, float inv_radius, float* __restrict__ out) {
    pdl_prologue();
    const long long total = (long long)B2 * G * K;
    const int CO = 3 + C + (center_idx ? C : 0);
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
        const int b2 = (int)(r / ((long long)G * K));
        const int g = (int)((r / K) % G);
        const int k = (int)(r % K);
        const int b = b2 / rep;
        const long long j = knn_idx[((size_t)b * G + g) * K + k];
        const float* p = xyz + ((size_t)b * N + j) * 3;
        const float* c = centers + ((size_t)b * G + g) * 3;
        float* o = out + (size_t)r * CO;
        o[0] = (p[0] - c[0]) * inv_radius;
        o[1] = (p[1] - c[1]) * inv_radius;
        o[2] = (p[2] - c[2]) * inv_radius;
        const float* f = feats + ((size_t)b2 * N + j) * C;
        for (int ch = 0; ch < C; ++ch) o[3 + ch] = f[ch];
        if (center_idx) {
            const float* fc = feats + ((size_t)b2 * N + center_idx[(size_t)b * G + g]) * C;
            for (int ch = 0; ch < C; ++ch) o[3 + C + ch] = f[ch] - fc[ch];
        }
    }
}

// 3 nearest centres per point + inverse-squared-distance weights (common.py:238-255).
// FOUR lanes per point: lane `part` scans the centres part, part + 4, ... keeping its three nearest, then two shuffle
// rounds merge the four sorted triples (order: distance, then centre index - what the ascending scan with a strict '<'
// produces).  One thread per point left 32768 / 32 = 1024 warps for 132 SMs (two per scheduler, a 512-long dependent
// chain each: 28 us); a quarter of the chain on four times the warps.
struct Near3 {
    float d0, d1, d2;
    int i0, i1, i2;
};

__device__ __forceinline__ bool near_less(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

__device__ __forceinline__ void near3_insert(Near3& t, float d, int g) {
    if (near_less(d, g, t.d2, t.i2)) {
        if (near_less(d, g, t.d1, t.i1)) {
            t.d2 = t.d1, t.i2 = t.i1;
            if (near_less(d, g, t.d0, t.i0)) {
                t.d1 = t.d0, t.i1 = t.i0;
                t.d0 = d, t.i0 = g;
            } else {
                t.d1 = d, t.i1 = g;
            }
        } else {
            t.d2 = d, t.i2 = g;
        }
    }
}

__global__ void __launch_bounds__(256)
knn3_interp_kernel(const float* __restrict__ xyz, const float* __restrict__ centers, int N, int G,
                   long long* __restrict__ idx_out, float* __restrict__ w_out) {
    pdl_prologue();
    extern __shared__ float s_c[];  // [G*3]
    const int b = blockIdx.y;
    centers += (size_t)b * G * 3;
    for (int i = threadIdx.x; i < G * 3; i += blockDim.x) s_c[i] = centers[i];
    __syncthreads();
    const int part = threadIdx.x & 3;
    const int n = blockIdx.x * (blockDim.x >> 2) + (threadIdx.x >> 2);
    const int nn = min(n, N - 1);  // all lanes stay in the shuffles; a ragged tail recomputes the last point
    const float* p = xyz + ((size_t)b * N + nn) * 3;
    const float x = p[0], y = p[1], z = p[2];
    Near3 t = {3.4e38f, 3.4e38f, 3.4e38f, 0x7fffffff, 0x7fffffff, 0x7fffffff};
    for (int g = part; g < G; g += 4) near3_insert(t, sqdist3(s_c[g * 3], s_c[g * 3 + 1], s_c[g * 3 + 2], x, y, z), g);
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        const float e0 = __shfl_xor_sync(0xffffffffu, t.d0, o), e1 = __shfl_xor_sync(0xffffffffu, t.d1, o),
                    e2 = __shfl_xor_sync(0xffffffffu, t.d2, o);
        const int j0 = __shfl_xor_sync(0xffffffffu, t.i0, o), j1 = __shfl_xor_sync(0xffffffffu, t.i1, o),
                  j2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
        near3_insert(t, e0, j0);
        near3_insert(t, e1, j1);
        near3_insert(t, e2, j2);
    }
    if (part != 0 || n >= N) return;
    // reference: dist = cdist (sqrt), then dist.square(), clamp(min=1e-8), reciprocal, normalise
    const float e0 = sqrtf(t.d0), e1 = sqrtf(t.d1), e2 = sqrtf(t.d2);
    const float v0 = 1.0f / fmaxf(e0 * e0, 1e-8f), v1 = 1.0f / fmaxf(e1 * e1, 1e-8f), v2 = 1.0f / fmaxf(e2 * e2, 1e-8f);
    const float sum = (v0 + v1) + v2;
    const size_t o = ((size_t)b * N + n) * 3;
    idx_out[o] = t.i0, idx_out[o + 1] = t.i1, idx_out[o + 2] = t.i2;
    w_out[o] = v0 / sum, w_out[o + 1] = v1 / sum, w_out[o + 2] = v2 / sum;
}


// Nearest-neighbour squared distance of every query to a key set (brute force, key tiles in smem).
// Replaces chamfer_distance_forward (torkit3d csrc/cuda/chamfer_distance_kernel.cu:10-89) as used by
// sample_furthest_points_from_border (pc_sam/model/common.py:466): dist1 and idx1 only.
__global__ void __launch_bounds__(256)
nn_distance_kernel(const float* __restrict__ q, const float* __restrict__ key, int n1, int n2, float* __restrict__ dist,
                   long long* __restrict__ idx) {
    pdl_prologue();
    __shared__ float s_k[256 * 3];
    const int i = blockIdx.x * 256 + threadIdx.x;
    float x = 0.f, y = 0.f, z = 0.f;
    if (i < n1) x = q[(size_t)i * 3], y = q[(size_t)i * 3 + 1], z = q[(size_t)i * 3 + 2];
    float best = 3.4e38f;
    int bi = -1;
    for (int j0 = 0; j0 < n2; j0 += 256) {
        const int j = j0 + threadIdx.x;
        if (j < n2) {
            s_k[threadIdx.x * 3] = key[(size_t)j * 3];
            s_k[threadIdx.x * 3 + 1] = key[(size_t)j * 3 + 1];
            s_k[threadIdx.x * 3 + 2] = key[(size_t)j * 3 + 2];
        }
        __syncthreads();
        const int lim = min(256, n2 - j0);
        for (int t = 0; t < lim; ++t) {
            const float d = sqdist3(s_k[t * 3], s_k[t * 3 + 1], s_k[t * 3 + 2], x, y, z);
            if (d < best) best = d, bi = j0 + t;
        }
        __syncthreads();
    }
    if (i < n1) {
        dist[i] = best;
        if (idx) idx[i] = bi;
    }
}


// ---------------------------------------------------------------------------------------------------------
// Batched ground-truth prompt sampler (pc_sam/model/common.py:371-474, the body of forward(is_eval=True) between two
// decoder passes).  The reference loops over (cloud, mask) in Python, compacts foreground / background points with
// boolean indexing, calls the chamfer kernel and compares results on the host (several synchronisations per mask).
// Here one launch handles every (cloud, mask, region): region membership is evaluated on the fly from the ground truth
// and the logits, the nearest-background distance of every foreground point is computed with the chamfer kernel's
// arithmetic (fma(dz,dz,fma(dy,dy,dx*dx)), d = background - foreground), and the farthest foreground point is kept by
// a 64-bit atomic max on (distance bits, ~index): ties resolve to the lowest index exactly like torch.argmax over the
// compacted array.  A second tiny kernel applies the reference's selection rules.  No host round trip.
//   region 0: false negatives  gt & ~pred      (mode 0, "error region" sampling: (gt & ~pred) | (~gt & pred))
//   region 1: false positives ~gt &  pred
//   region 2: the ground-truth mask itself (fallback when both error regions are empty)
__device__ __forceinline__ int border_region_label(int region, int mode, bool gt, bool pred) {
    if (mode == 0) return (gt != pred) ? 1 : 0;
    if (region == 0) return (gt && !pred) ? 1 : 0;
    if (region == 1) return (!gt && pred) ? 1 : 0;
    return gt ? 1 : 0;
}

// Pass 1: compact the foreground AND background point indices of every (cloud x mask, region) - order is irrelevant because
// min() is order independent and the arg-max key carries the original index.  Warp-aggregated append (one atomic per warp
// and list); the per-point minimum is initialised to +inf on the way.
__device__ __forceinline__ void warp_append(bool pred, int value, int* counter, int* list, unsigned* init_inf) {
    const int lane = threadIdx.x & 31;
    const unsigned m = __ballot_sync(0xffffffffu, pred);
    if (m == 0) return;
    const int leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(counter, __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (pred) {
        const int slot = base + __popc(m & ((1u << lane) - 1));
        list[slot] = value;
        if (init_inf) init_inf[slot] = 0x7f800000u;
    }
}

__global__ void __launch_bounds__(256)
border_compact_kernel(const unsigned char* __restrict__ gt, const float* __restrict__ logits,
                      const unsigned char* __restrict__ pred_mask, int N, int mode, int nreg, int* __restrict__ counts /* [BM][3][2] */,
                      int* __restrict__ fg_list, int* __restrict__ bg_list, unsigned* __restrict__ mind /* each [BM][nreg][N] */) {
    const int bm = blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    bool g = false, p = false;
    if (i < N) {
        g = gt[(size_t)bm * N + i] != 0;
        p = logits ? (logits[(size_t)bm * N + i] > 0.f) : (pred_mask ? pred_mask[(size_t)bm * N + i] != 0 : false);
    }
    for (int r = 0; r < nreg; ++r) {
        const int lab = border_region_label(r, mode, g, p);
        const size_t off = ((size_t)bm * nreg + r) * N;
        warp_append(i < N && lab == 1, i, counts + (bm * 3 + r) * 2, fg_list + off, mind + off);
        warp_append(i < N && lab == 0, i, counts + (bm * 3 + r) * 2 + 1, bg_list + off, nullptr);
    }
}

// Pass 2: block = 512 foreground points (2 per thread) x one chunk of BORDER_CHUNK background points, staged through
// shared memory as float4 (one LDS.128 feeds two distance evaluations).  |fg| x |bg| evaluations in total - the same
// work as the reference's compacted chamfer call - spread over enough blocks to fill the GPU for a single mask.
constexpr int BORDER_CHUNK = 2048;

__global__ void __launch_bounds__(256)
border_mindist_kernel(const float* __restrict__ coords, int M, int N, int nreg, const int* __restrict__ counts,
                      const int* __restrict__ fg_list, const int* __restrict__ bg_list, unsigned* __restrict__ mind) {
    __shared__ float4 s_b[256];
    const int br = blockIdx.z, bm = br / nreg, region = br - bm * nreg;
    const int nfg = counts[(bm * 3 + region) * 2], nbg = counts[(bm * 3 + region) * 2 + 1];
    const int f0 = blockIdx.x * 512, c0 = blockIdx.y * BORDER_CHUNK;
    if (f0 >= nfg || c0 >= nbg) return;
    const float* xyz = coords + (size_t)(bm / M) * N * 3;
    const size_t off = (size_t)br * N;
    const int s0 = f0 + threadIdx.x, s1 = s0 + 256;
    const int i0 = s0 < nfg ? fg_list[off + s0] : 0, i1 = s1 < nfg ? fg_list[off + s1] : 0;
    const float x0 = xyz[(size_t)i0 * 3], y0 = xyz[(size_t)i0 * 3 + 1], z0 = xyz[(size_t)i0 * 3 + 2];
    const float x1 = xyz[(size_t)i1 * 3], y1 = xyz[(size_t)i1 * 3 + 1], z1 = xyz[(size_t)i1 * 3 + 2];
    float m0 = __int_as_float(0x7f800000), m1 = m0;
    const int c1 = min(c0 + BORDER_CHUNK, nbg);
    for (int j0 = c0; j0 < c1; j0 += 256) {
        const int j = j0 + threadIdx.x;
        if (j < c1) {
            const int k = bg_list[off + j];
            s_b[threadIdx.x] = make_float4(xyz[(size_t)k * 3], xyz[(size_t)k * 3 + 1], xyz[(size_t)k * 3 + 2], 0.f);
        }
        __syncthreads();
        const int lim = min(256, c1 - j0);
#pragma unroll 4
        for (int t = 0; t < lim; ++t) {
            const float4 b = s_b[t];
            m0 = fminf(m0, sqdist3(b.x, b.y, b.z, x0, y0, z0));
            m1 = fminf(m1, sqdist3(b.x, b.y, b.z, x1, y1, z1));
        }
        __syncthreads();
    }
    if (s0 < nfg) atomicMin(mind + off + s0, __float_as_uint(m0));  // distances are >= 0: uint order == float order
    if (s1 < nfg) atomicMin(mind + off + s1, __float_as_uint(m1));
}

// Pass 3: one block per (cloud x mask): arg-max of the per-point minima in each region (ties -> lowest point index, like
// torch.argmax over the compacted array), then the reference's selection rules (common.py:411-431).
__global__ void __launch_bounds__(256)
border_select_kernel(const float* __restrict__ coords, const unsigned char* __restrict__ gt, const int* __restrict__ counts,
                     const int* __restrict__ fg_list, const unsigned* __restrict__ mind, int M, int N, int mode, int nreg,
                     float* __restrict__ out_xyz, unsigned char* __restrict__ out_label, int* __restrict__ status) {
    __shared__ unsigned long long s_best[8];
    __shared__ unsigned long long s_reg[3];
    const int bm = blockIdx.x;
    for (int r = 0; r < nreg; ++r) {
        const int nfg = counts[(bm * 3 + r) * 2], nbg = counts[(bm * 3 + r) * 2 + 1];
        const size_t off = ((size_t)bm * nreg + r) * N;
        unsigned long long key = 0ull;
        if (nbg > 0)
            for (int s_ = threadIdx.x; s_ < nfg; s_ += 256) {
                const unsigned long long k = ((unsigned long long)mind[off + s_] << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)fg_list[off + s_]);
                key = k > key ? k : key;
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
            key = other > key ? other : key;
        }
        if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = key;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; ++w) key = s_best[w] > key ? s_best[w] : key;
            s_reg[r] = key;
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const unsigned long long p = s_reg[0], n = nreg > 1 ? s_reg[1] : 0ull, g = nreg > 2 ? s_reg[2] : 0ull;
    const float pd = p ? __uint_as_float((unsigned)(p >> 32)) : -1.f;
    const float nd = n ? __uint_as_float((unsigned)(n >> 32)) : -1.f;
    unsigned long long pick;
    if (mode == 0) pick = p;                  // from_error_region: the single merged region
    else if (pd > nd) pick = p;               // common.py:417-419
    else if (nd == -1.f) pick = g;            // :420-428 both error regions empty -> sample inside the ground truth
    else pick = n;                            // :429-431
    if (!pick) {  // the reference fails here (torch.stack of None); reported through status
        out_xyz[bm * 3] = out_xyz[bm * 3 + 1] = out_xyz[bm * 3 + 2] = 0.f;
        out_label[bm] = 0;
        atomicExch(status, 1);
        return;
    }
    const unsigned idx = 0xFFFFFFFFu - (unsigned)(pick & 0xFFFFFFFFull);
    const float* xyz = coords + ((size_t)(bm / M) * N + idx) * 3;
    out_xyz[bm * 3] = xyz[0], out_xyz[bm * 3 + 1] = xyz[1], out_xyz[bm * 3 + 2] = xyz[2];
    out_label[bm] = gt[(size_t)bm * N + idx];
}

}  // namespace psam

// workspace layout: counts[BM][3][2] i32 | fg_list, bg_list [BM][3][N] i32 | mind[BM][3][N] u32
extern "C" size_t psam_border_prompt_workspace_bytes(int B, int M, int N) {
    const size_t bm = (size_t)B * M;
    return bm * 6 * 4 + bm * 3 * (size_t)N * 4 * 3;
}

extern "C" int psam_border_prompt_f32(const float* coords, const unsigned char* gt_masks, const float* pred_logits,
                                      const unsigned char* pred_masks, int B, int M, int N, int from_error_region,
                                      float* prompt_xyz_out, unsigned char* prompt_label_out, int* status, void* workspace,
                                      cudaStream_t stream) {
    using namespace psam;
    if (!coords || !gt_masks || !prompt_xyz_out || !prompt_label_out || !status || !workspace || B <= 0 || M <= 0 || N <= 0 ||
        (pred_logits && pred_masks) || ((uintptr_t)workspace & 3) != 0)
        return PSAM_ERR_ARG;
    if ((long long)B * M * 3 > 65535) return PSAM_ERR_UNSUPPORTED;
    const int BM = B * M;
    const int mode = from_error_region ? 0 : 1;
    const int nreg = mode == 0 ? 1 : 3;
    int* counts = static_cast<int*>(workspace);
    int* fg_list = counts + (size_t)BM * 6;
    int* bg_list = fg_list + (size_t)BM * 3 * N;
    unsigned* mind = reinterpret_cast<unsigned*>(bg_list + (size_t)BM * 3 * N);
    PSAM_CUDA_TRY(cudaMemsetAsync(counts, 0, (size_t)BM * 6 * 4, stream));
    border_compact_kernel<<<dim3(ceil_div(N, 256), BM), 256, 0, stream>>>(gt_masks, pred_logits, pred_masks, N, mode, nreg, counts, fg_list,
                                                                         bg_list, mind);
    PSAM_LAUNCH_CHECK();
    border_mindist_kernel<<<dim3(ceil_div(N, 512), ceil_div(N, BORDER_CHUNK), BM * nreg), 256, 0, stream>>>(coords, M, N, nreg, counts, fg_list,
                                                                                                          bg_list, mind);
    PSAM_LAUNCH_CHECK();
    border_select_kernel<<<BM, 256, 0, stream>>>(coords, gt_masks, counts, fg_list, mind, M, N, mode, nreg, prompt_xyz_out, prompt_label_out,
                                                 status);
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

namespace psam {
}  // namespace psam

extern "C" int psam_nn_distance_f32(const float* query, const float* key, int n1, int n2, float* dist_out,
                                    long long* idx_out, cudaStream_t stream) {
    using namespace psam;
    if (!query || !key || !dist_out || n1 <= 0 || n2 <= 0) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(nn_distance_kernel, dim3(ceil_div(n1, 256)), dim3(256), (size_t)(0), stream, query, key, n1, n2, dist_out, idx_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_knn_f32(const float* query, const float* key, int B, int Q, int N, int K, long long* idx_out,
                            float* d2_out, cudaStream_t stream) {
    using namespace psam;
    if (!query || !key || !idx_out || B <= 0 || Q <= 0 || N <= 0 || K <= 0 || K > N) return PSAM_ERR_ARG;
    if (K > 1024) return PSAM_ERR_UNSUPPORTED;
    // sample stride: expected candidate count ~ K*stride (<= 1024), sample size >= 4K and <= the smem limit
    int stride = 1;
    while ((long long)K * stride * 2 <= 1024 && (N + 2 * stride - 1) / (2 * stride) >= 4 * K) stride *= 2;
    while ((N + stride - 1) / stride > KNN_MAX_SAMPLE) stride *= 2;
    const int ns = (N + stride - 1) / stride;
    (void)ns;
    int sample_cap = (2 * K + 3) & ~3;  // scratch for the final (distance, index) list of one centre
    // candidate capacity per centre: the bound admits ~1.2 K stride keys (sampling std ~ K^-1/2); beyond it the exact fallback runs
    long long cap = (long long)2 * K * stride;
    if (cap < 1024) cap = 1024;
    if (cap > KNN_MAX_CAP) cap = KNN_MAX_CAP;
    if (cap > N) cap = (N + 3) & ~3;  // cannot hold more candidates than keys
    if (cap < K) return PSAM_ERR_UNSUPPORTED;
    // centres per CTA: as many as keep >= 1.5 CTAs per SM (the per-centre select phases are latency-bound: they need
    // co-resident CTAs to overlap) and fit two CTAs' shared memory on an SM
    auto smem_for = [&](int c) { return (size_t)sample_cap * 4 + (size_t)c * cap * 8 + (64 + (size_t)c * KNN_HIST) * 4; };
    int C = 4;
    while (C > 1 && ((long long)B * ((Q + C - 1) / C) < 222 || smem_for(C) > 100 * 1024)) C /= 2;
    const size_t smem = smem_for(C);
    const dim3 grid((unsigned)((Q + C - 1) / C), (unsigned)B);
#define PSAM_KNN_LAUNCH(CC)                                                                                                  \
    do {                                                                                                                     \
        PSAM_CUDA_TRY(cudaFuncSetAttribute(knn_kernel<CC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));         \
        PSAM_CUDA_TRY(psam::launch(knn_kernel<CC>, grid, dim3(KNN_THREADS), smem, stream, query, key, Q, N, K, stride,      \
                                   sample_cap, (int)cap, idx_out, d2_out));                                                 \
    } while (0)
    if (C == 4) PSAM_KNN_LAUNCH(4);
    else if (C == 2) PSAM_KNN_LAUNCH(2);
    else PSAM_KNN_LAUNCH(1);
#undef PSAM_KNN_LAUNCH
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_group_gather_f32(const float* xyz, const float* feats, const float* centers,
                                     const long long* knn_idx, const long long* center_idx, int B, int rep, int N, int G, int K,
                                     int C, float radius, float* groups_out, cudaStream_t stream) {
    using namespace psam;
    if (!xyz || !feats || !centers || !knn_idx || !groups_out || B <= 0 || rep <= 0 || C < 0) return PSAM_ERR_ARG;
    const long long total = (long long)B * rep * G * K;
    const int blocks = (int)min((long long)132 * 16, ceil_div_ll(total, 256));
    PSAM_CUDA_TRY(psam::launch(group_gather_kernel, dim3(blocks), dim3(256), (size_t)(0), stream, xyz, feats, centers, knn_idx, center_idx, B * rep, rep, N, G, K, C,
                                                    radius > 0.f ? 1.0f / radius : 1.0f, groups_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_knn3_interp_f32(const float* xyz, const float* centers, int B, int N, int G, long long* idx_out,
                                    float* w_out, cudaStream_t stream) {
    using namespace psam;
    if (!xyz || !centers || !idx_out || !w_out || B <= 0 || N <= 0 || G < 3) return PSAM_ERR_ARG;
    const size_t smem = (size_t)G * 3 * sizeof(float);
    if (smem > 200 * 1024) return PSAM_ERR_UNSUPPORTED;
    PSAM_CUDA_TRY(cudaFuncSetAttribute(knn3_interp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSAM_CUDA_TRY(psam::launch(knn3_interp_kernel, dim3(dim3(ceil_div(N, 64), B)), dim3(256), (size_t)(smem), stream, xyz, centers, N, G, idx_out, w_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
