// Automatic mask generation ("segment everything"): candidate extraction from multimask decoder logits and greedy
// mask-IoU NMS, all on the device.  The semantics are stated in include/psam_b200.h.  Every kernel takes a cloud
// dimension: the single-cloud entry points are the B = 1 case of the batched ones.
//
//   mask_candidates_kernel   one CTA per logit row: a single streaming pass (128-bit loads where aligned) produces the
//                            bit-packed mask, the three threshold counts, the stability score and the filtered score.
//   nms_order_kernel         one CTA per cloud: bitonic sort of the (score desc, slot asc) keys in shared memory, valid count.
//   nms_pairs_kernel         64 x 64 tiles of sorted positions (upper triangle) per cloud (grid.z): AND + popc over the
//                            bit-packed masks staged through shared memory, comparisons turned into 64-bit suppression
//                            words by ballots.
//   nms_scan_kernel          one CTA per cloud: greedy walk in blocks of 64; one warp resolves a block against its diagonal
//                            words, then every thread ORs the kept rows into the "removed" bitset.
//   mask_regions_kernel<S>   one CTA per (cloud, kept mask): lock-free union-find over the kNN graph, first on the points
//                            outside the mask (small holes are filled), then on the mask (small islands are removed); labels
//                            in shared memory (S = true, N <= 49152) or in a per-CTA slice of the workspace.
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace {

constexpr int kCandThreads = 256;
constexpr int kNmsMaxK = 16384;
constexpr int kTile = 64;       // sorted positions per tile side / per scan block
constexpr int kTileWords = 32;  // mask words staged per shared-memory round
constexpr int kScanThreads = 512;
constexpr int kNmsMaxClouds = 65535;  // grid.z of nms_pairs_kernel

__device__ __forceinline__ bool candidate_survives(float iou, float stab, int area, float iou_t, float stab_t, int min_area) {
    if (!(iou == iou)) return false;  // a NaN predicted IoU is never kept
    if (iou_t > 0.f && !(iou > iou_t)) return false;
    if (stab_t > 0.f && !(stab >= stab_t)) return false;
    return area >= min_area && area >= 1;
}

// VARLEN: rows have Ns logits of which cloud b's first lengths[b] (clamped to [0, Ns]) are points; only those are counted and
// packed (later bits are 0), and the slots of prompts past min(P, lengths[b]) (slot / C) score -inf.  Otherwise N = Ns.
template <bool VEC, bool VARLEN>
__global__ void __launch_bounds__(kCandThreads) mask_candidates_kernel(const float* __restrict__ logits,
                                                                       const float* __restrict__ iou_preds, int Ns,
                                                                       float thr, float thr_hi, float thr_lo, float iou_t,
                                                                       float stab_t, int min_area, long long base,
                                                                       int rows_per_cloud, long long cloud_stride, int W,
                                                                       const int* __restrict__ lengths, int P, int C,
                                                                       uint32_t* __restrict__ bits, int* __restrict__ area_out,
                                                                       float* __restrict__ stab_out, float* __restrict__ score_out) {
    psam::pdl_prologue();
    constexpr int U = 4;  // warp iterations whose loads are issued together
    const int row = blockIdx.x;
    const float* rp = logits + (size_t)row * Ns;
    const int cloud = row / rows_per_cloud;  // rows of cloud b are b * rows_per_cloud .. (b + 1) * rows_per_cloud
    const long long slot = cloud * cloud_stride + base + (row - cloud * rows_per_cloud);
    const int N = VARLEN ? min(max(lengths[cloud], 0), Ns) : Ns;
    uint32_t* bp = bits + (size_t)slot * W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int n_area = 0, n_hi = 0, n_lo = 0;
    if (VEC) {
        // a warp iteration covers 128 points = 4 words; lane l holds points 4l..4l+3 of it
        const float4* rp4 = reinterpret_cast<const float4*>(rp);
        const int n4 = VARLEN ? (N + 3) >> 2 : N >> 2;  // VEC needs Ns % 4 == 0, so a cloud's last quad is inside its row
        const int iters = (W + 3) >> 2;
        for (int it0 = warp * U; it0 < iters; it0 += nw * U) {
            float4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int q = (it0 + u) * 32 + lane;
                v[u] = q < n4 ? __ldcs(rp4 + q) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int it = it0 + u;
                if (it >= iters) break;  // warp-uniform
                const bool in = it * 32 + lane < n4;
                const float x[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
                uint32_t nib = 0;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    if (in && (!VARLEN || (it * 32 + lane) * 4 + e < N)) {
                        nib |= (uint32_t)(x[e] > thr) << e;
                        n_hi += x[e] > thr_hi;
                        n_lo += x[e] > thr_lo;
                    }
                }
                n_area += __popc(nib);
                uint32_t word = nib << (4 * (lane & 7));
                word |= __shfl_xor_sync(0xffffffffu, word, 1);
                word |= __shfl_xor_sync(0xffffffffu, word, 2);
                word |= __shfl_xor_sync(0xffffffffu, word, 4);
                const int w = it * 4 + (lane >> 3);
                if ((lane & 7) == 0 && w < W) bp[w] = word;
            }
        }
    } else {
        // a warp iteration covers 32 points = one word, built by a ballot
        for (int it0 = warp * U; it0 < W; it0 += nw * U) {
            float v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int p = (it0 + u) * 32 + lane;
                v[u] = p < N ? __ldcs(rp + p) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int it = it0 + u;
                if (it >= W) break;  // warp-uniform
                const bool in = it * 32 + lane < N;
                const bool b = in && v[u] > thr;
                n_hi += in && v[u] > thr_hi;
                n_lo += in && v[u] > thr_lo;
                const uint32_t word = __ballot_sync(0xffffffffu, b);
                n_area += b;
                if (lane == 0) bp[it] = word;
            }
        }
    }
    __shared__ int red[3][kCandThreads / 32];
    n_area = __reduce_add_sync(0xffffffffu, n_area);
    n_hi = __reduce_add_sync(0xffffffffu, n_hi);
    n_lo = __reduce_add_sync(0xffffffffu, n_lo);
    if (lane == 0) {
        red[0][warp] = n_area;
        red[1][warp] = n_hi;
        red[2][warp] = n_lo;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int a = 0, h = 0, l = 0;
        for (int i = 0; i < nw; ++i) {
            a += red[0][i];
            h += red[1][i];
            l += red[2][i];
        }
        const float stab = __fdiv_rn(__int2float_rn(h), __int2float_rn(l));
        const float iou = iou_preds[row];
        area_out[slot] = a;
        stab_out[slot] = stab;
        bool keep = candidate_survives(iou, stab, a, iou_t, stab_t, min_area);
        if constexpr (VARLEN) keep = keep && (slot - cloud * cloud_stride) / C < min(P, N);
        score_out[slot] = keep ? iou : -INFINITY;
    }
}

// ---- NMS workspace: one block per cloud of cloud_bytes = psam_mask_nms_workspace_bytes(K, W) bytes ---------------
//   [0, 16)                 the valid count
//   [16, 16 + order bytes)  the sorted slot order
//   then                    the K x ceil(K / 64) suppression words
__host__ __device__ __forceinline__ size_t nms_order_bytes(int K) { return ((size_t)K * sizeof(int) + 15) / 16 * 16; }

struct NmsCloud {
    int* count;
    int* order;
    unsigned long long* mat;
};

__device__ __forceinline__ NmsCloud nms_cloud(char* ws, size_t cloud_bytes, int K, int b) {
    char* c = ws + (size_t)b * cloud_bytes;
    return {reinterpret_cast<int*>(c), reinterpret_cast<int*>(c + 16), reinterpret_cast<unsigned long long*>(c + 16 + nms_order_bytes(K))};
}

// ---- NMS a: order ------------------------------------------------------------------------------------------------
// One CTA per cloud (blockIdx.x); the cloud's K scores start at score + b * K.
__global__ void __launch_bounds__(1024) nms_order_kernel(const float* __restrict__ score, int K, int P2, char* __restrict__ ws,
                                                         size_t cloud_bytes) {
    psam::pdl_prologue();
    const NmsCloud cw = nms_cloud(ws, cloud_bytes, K, blockIdx.x);
    score += (size_t)blockIdx.x * K;
    int* __restrict__ order = cw.order;
    extern __shared__ unsigned long long keys[];
    __shared__ int n_valid;
    if (threadIdx.x == 0) n_valid = 0;
    __syncthreads();
    int valid = 0;
    for (int i = threadIdx.x; i < P2; i += blockDim.x) {
        unsigned long long k = ~0ull;  // dropped and padding entries sort last
        if (i < K) {
            const float s = score[i];
            if (s > -INFINITY) {  // -inf (filtered) and NaN are dropped
                // + 0: -0.0 becomes +0.0, so the two zeros share a key and the slot decides, as for any other tie
                uint32_t u = __float_as_uint(__fadd_rn(s, 0.f));
                u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // monotone in s
                k = ((unsigned long long)(~u) << 32) | (uint32_t)i;  // ascending key = score descending, slot ascending
                ++valid;
            }
        }
        keys[i] = k;
    }
    if (valid) atomicAdd(&n_valid, valid);
    for (int k = 2; k <= P2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int p = threadIdx.x; p < (P2 >> 1); p += blockDim.x) {
                const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1));
                const int l = i + j;
                const bool up = (i & k) == 0;
                const unsigned long long a = keys[i], b = keys[l];
                if ((a > b) == up) {
                    keys[i] = b;
                    keys[l] = a;
                }
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K; i += blockDim.x) order[i] = (int)(uint32_t)(keys[i] & 0xffffffffull);
    if (threadIdx.x == 0) *cw.count = n_valid;
}

// ---- NMS b: pairwise suppression bits ---------------------------------------------------------------------------
// Tile (bi, bj), bj >= bi, of sorted positions of cloud blockIdx.z, whose candidates start at bits + b * K * W and
// area + b * K.  Thread (ty, tx) of 16 x 16 owns rows ty*4 + r and columns tx + 16 c.
__global__ void __launch_bounds__(256) nms_pairs_kernel(const uint32_t* __restrict__ bits, const int* __restrict__ area, int K, int W,
                                                        float nms_thresh, char* __restrict__ ws, size_t cloud_bytes, int ldm) {
    psam::pdl_prologue();
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bj < bi) return;
    const NmsCloud cw = nms_cloud(ws, cloud_bytes, K, blockIdx.z);
    const int count = *cw.count;
    if (bj * kTile >= count) return;  // beyond the cloud's valid candidates (bi <= bj)
    const int* __restrict__ order = cw.order;
    unsigned long long* __restrict__ mat = cw.mat;
    bits += (size_t)blockIdx.z * K * W;
    area += (size_t)blockIdx.z * K;
    __shared__ __align__(16) uint32_t sa[kTileWords][kTile];
    __shared__ __align__(16) uint32_t sb[kTileWords][kTile];
    __shared__ int slot_a[kTile], slot_b[kTile], area_a[kTile], area_b[kTile];
    const int tid = threadIdx.x;
    if (tid < 2 * kTile) {
        const int r = tid & (kTile - 1);
        const int pos = (tid < kTile ? bi : bj) * kTile + r;
        const int s = pos < count ? order[pos] : -1;
        const int a = s >= 0 ? area[s] : 0;
        if (tid < kTile) {
            slot_a[r] = s;
            area_a[r] = a;
        } else {
            slot_b[r] = s;
            area_b[r] = a;
        }
    }
    __syncthreads();
    const int tx = tid & 15, ty = tid >> 4;
    uint32_t acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0;
    for (int w0 = 0; w0 < W; w0 += kTileWords) {
        const int kw = min(kTileWords, W - w0);
        for (int e = tid; e < kTileWords * kTile; e += blockDim.x) {
            const int r = e & (kTile - 1), w = e >> 6;
            const int ga = slot_a[r], gb = slot_b[r];
            const bool inw = w < kw;
            sa[w][r] = (ga >= 0 && inw) ? bits[(size_t)ga * W + w0 + w] : 0u;
            sb[w][r] = (gb >= 0 && inw) ? bits[(size_t)gb * W + w0 + w] : 0u;
        }
        __syncthreads();
#pragma unroll 4
        for (int w = 0; w < kw; ++w) {
            const uint4 a4 = *reinterpret_cast<const uint4*>(&sa[w][ty * 4]);
            const uint32_t a[4] = {a4.x, a4.y, a4.z, a4.w};
            const uint32_t b[4] = {sb[w][tx], sb[w][tx + 16], sb[w][tx + 32], sb[w][tx + 48]};
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] += __popc(a[r] & b[c]);
        }
        __syncthreads();
    }
    // epilogue: one ballot per (r, c); the half-warp of each ty contributes 16 columns
    const int half = (tid >> 4) & 1;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int li = ty * 4 + r;
        const int gi = bi * kTile + li;
        unsigned long long word = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int lj = tx + 16 * c;
            const int gj = bj * kTile + lj;
            bool sup = false;
            if (gi < count && gj < count && gj > gi) {
                const int inter = (int)acc[r][c];
                const int uni = area_a[li] + area_b[lj] - inter;
                sup = __fdiv_rn(__int2float_rn(inter), __int2float_rn(uni)) > nms_thresh;
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, sup);
            word |= (unsigned long long)((bal >> (16 * half)) & 0xffffu) << (16 * c);
        }
        if (tx == 0 && gi < count) mat[(size_t)gi * ldm + bj] = word;
    }
}

// ---- NMS c: greedy scan ------------------------------------------------------------------------------------------
// One CTA per cloud (blockIdx.x): keep + b * K, keep_count + b.
__global__ void __launch_bounds__(kScanThreads) nms_scan_kernel(const char* __restrict__ ws, size_t cloud_bytes, int K, int ldm,
                                                                int* __restrict__ keep, int* __restrict__ keep_count) {
    psam::pdl_prologue();
    __shared__ unsigned long long removed[kNmsMaxK / kTile];
    __shared__ int kept_rows[kTile];
    __shared__ int n_block, n_kept;
    const NmsCloud cw = nms_cloud(const_cast<char*>(ws), cloud_bytes, K, blockIdx.x);
    const unsigned long long* __restrict__ mat = cw.mat;
    const int* __restrict__ order = cw.order;
    keep += (size_t)blockIdx.x * K;
    keep_count += blockIdx.x;
    const int count = *cw.count;
    const int nb = (count + kTile - 1) / kTile;
    const int tid = threadIdx.x;
    for (int c = tid; c < nb; c += blockDim.x) removed[c] = 0ull;
    if (tid == 0) n_kept = 0;
    __syncthreads();
    for (int b = 0; b < nb; ++b) {
        if (tid < 32) {
            const int lane = tid;
            const int rows = min(kTile, count - b * kTile);
            const size_t r0 = (size_t)b * kTile;
            const unsigned long long d0 = lane < rows ? mat[(r0 + lane) * ldm + b] : 0ull;
            const unsigned long long d1 = lane + 32 < rows ? mat[(r0 + lane + 32) * ldm + b] : 0ull;
            unsigned long long rem = removed[b], km = 0ull;
            for (int i = 0; i < rows; ++i) {
                const unsigned long long di = __shfl_sync(0xffffffffu, i < 32 ? d0 : d1, i & 31);
                if (!((rem >> i) & 1ull)) {
                    km |= 1ull << i;
                    rem |= di;
                }
            }
            const int base = n_kept;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int pos = lane + 32 * h;
                if ((km >> pos) & 1ull) {
                    const int rank = __popcll(km & ((1ull << pos) - 1ull));
                    keep[base + rank] = order[r0 + pos];
                    kept_rows[rank] = pos;
                }
            }
            __syncwarp();
            if (lane == 0) {
                n_block = __popcll(km);
                n_kept = base + n_block;
            }
        }
        __syncthreads();
        const int ncols = nb - b - 1;
        const int total = n_block * ncols;
        for (int e = tid; e < total; e += blockDim.x) {
            const int r = e / ncols, c = b + 1 + e % ncols;
            const unsigned long long v = mat[((size_t)b * kTile + kept_rows[r]) * ldm + c];
            if (v) atomicOr(&removed[c], v);
        }
        __syncthreads();
    }
    if (tid == 0) *keep_count = n_kept;
}

// ---- small-region post-processing: connected components over the kNN graph ------------------------------------------
// One CTA per kept mask (persistent over the ranks).  par[] is a union-find forest over the points of the working set with
// par[i] <= i at all times, so every root is the smallest point of its component and the forest's final shape does not
// depend on the order in which edges are hooked.  After flattening, a root's entry holds -(component size).
constexpr int kRegionThreads = 1024;
constexpr int kRegionSmemMaxN = 49152;        // 4 B of labels + 1 bit of mask per point in shared memory
constexpr int kRegionMaxN = 1 << 20;           // the mask words (N / 8 bytes) always stay in shared memory: 128 KB
constexpr long long kRegionL2Bytes = 24ll << 20;  // workspace form: label slices meant to stay L2-resident
constexpr int kRegionMaxSlices = 132;

// label slices of the workspace form (one per CTA), shared by all clouds of a launch: as many as fit kRegionL2Bytes, at
// most kRegionMaxSlices and the number of items
int region_slices(long long items, int N) {
    long long fit = kRegionL2Bytes / ((long long)N * 4);
    fit = fit < 1 ? 1 : (fit > kRegionMaxSlices ? kRegionMaxSlices : fit);
    return (int)(items < fit ? items : fit);
}

__device__ __forceinline__ bool region_member(const uint32_t* sw, int i, int N, bool invert) {
    return i < N && (((sw[i >> 5] >> (i & 31)) & 1u) != (uint32_t)invert);
}

// root of i with path halving (ECL-CC), used while edges are hooked.  A stale halving store still writes an ancestor,
// which is all the hooking needs.  The flatten pass does not use it (see there).
__device__ __forceinline__ int region_find(volatile int* par, int i) {
    int cur = par[i];
    if (cur != i) {
        int prev = i, next;
        while (cur > (next = par[cur])) {
            par[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

// Labels the components of {i < N : bit i of sw != invert} under the edges {i, nbr[i*k1 + t]}.  On return, for a member i:
// par[i] < 0 -> i is a root of a component of -par[i] points; otherwise par[i] is its root.
__device__ void region_components(const uint32_t* sw, bool invert, int N, const long long* __restrict__ nbr, int k1, int* par) {
    volatile int* vp = par;
    for (int i = threadIdx.x; i < N; i += blockDim.x) par[i] = i;
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        if (!region_member(sw, i, N, invert)) continue;
        const long long* row = nbr + (size_t)i * k1;
        for (int t = 0; t < k1; ++t) {
            const long long jj = row[t];
            if (jj < 0 || jj >= N || jj == i) continue;  // an index outside the cloud is no edge
            const int j = (int)jj;
            if (!region_member(sw, j, N, invert)) continue;
            int a = region_find(vp, i), b = region_find(vp, j);
            while (a != b) {  // hook the larger root under the smaller one; on a lost race climb to the winner
                if (a < b) {
                    const int r = atomicCAS(par + b, b, a);
                    if (r == b) break;
                    b = r;
                } else {
                    const int r = atomicCAS(par + a, a, b);
                    if (r == a) break;
                    a = r;
                }
            }
        }
    }
    __syncthreads();
    // flatten: a read-only walk, and each thread writes only its own entry.  Path halving here could let a stale store
    // re-point an entry that another thread has already set to its root.  Every concurrent write replaces an ancestor by
    // the root, so each walk still ends at the root.
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        if (!region_member(sw, i, N, invert)) continue;
        int r = vp[i], n;
        while (r > (n = vp[r])) r = n;
        vp[i] = r;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x)
        if (par[i] == i && region_member(sw, i, N, invert)) par[i] = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const int r = par[i];
        if (r >= 0 && r != i && region_member(sw, i, N, invert)) atomicSub(par + r, 1);
    }
    __syncthreads();
}

__device__ __forceinline__ int region_root(const int* par, int i) { return par[i] < 0 ? i : par[i]; }

// Items it = b * K + p of B clouds: cloud b's candidates start at bits + b * cloud_slots * W, its graph at nbr + b * N * k1,
// its keep list and outputs at b * K; its count is keep_count[b].
// VARLEN: cloud b's working sets hold only its first lengths[b] points (clamped to [0, N]); N stays the stride of the graph.
template <bool SMEM, bool VARLEN>
__global__ void __launch_bounds__(kRegionThreads) mask_regions_kernel(const uint32_t* __restrict__ bits, long long cloud_slots, int B,
                                                                      int K, int W, int Ns, const int* __restrict__ lengths,
                                                                      const int* __restrict__ keep,
                                                                      const int* __restrict__ keep_count,
                                                                      const long long* __restrict__ nbr, int k1, int min_area,
                                                                      uint32_t* __restrict__ bits_out, int* __restrict__ area_out,
                                                                      float* __restrict__ score_out, int* __restrict__ workspace) {
    psam::pdl_prologue();
    extern __shared__ __align__(16) uint32_t region_smem[];
    uint32_t* sw = region_smem;
    int* par = SMEM ? reinterpret_cast<int*>(region_smem + ((((Ns + 31) >> 5) + 3) & ~3)) : workspace + (size_t)blockIdx.x * Ns;
    __shared__ int changed, any_small, area_red;
    __shared__ unsigned long long best;  // (size << 32) | ~root: the largest component, smallest root on equal sizes
    const int lane = threadIdx.x & 31;
    const long long items = (long long)B * K;
    for (long long it = blockIdx.x; it < items; it += gridDim.x) {
        const int b = (int)(it / K), p = (int)(it - (long long)b * K);
        if (p >= keep_count[b]) {
            if (threadIdx.x == 0) score_out[it] = -INFINITY;
            continue;
        }
        const int N = VARLEN ? min(max(lengths[b], 0), Ns) : Ns;
        const int Wn = (N + 31) >> 5;
        const uint32_t* src = bits + ((size_t)b * cloud_slots + keep[it]) * W;
        const long long* cnbr = nbr + (size_t)b * Ns * k1;
        for (int w = threadIdx.x; w < Wn; w += blockDim.x) {
            const int tail = N - 32 * w;
            sw[w] = tail >= 32 ? src[w] : src[w] & ((1u << tail) - 1u);
        }
        if (threadIdx.x == 0) {
            changed = 0;
            any_small = 0;
            area_red = 0;
            best = 0ull;
        }
        __syncthreads();
        // 1. holes: components of the complement smaller than min_area join the mask
        region_components(sw, true, N, cnbr, k1, par);
        for (int i = threadIdx.x; i < Wn * 32; i += blockDim.x) {  // a warp owns whole words
            const uint32_t word = sw[i >> 5];
            const bool in = (word >> (i & 31)) & 1u;
            const bool fill = !in && i < N && -par[region_root(par, i)] < min_area;
            const uint32_t add = __ballot_sync(0xffffffffu, fill);
            if (lane == 0 && add) {
                sw[i >> 5] = word | add;
                changed = 1;
            }
        }
        __syncthreads();
        // 2. islands: components of the mask smaller than min_area leave it; if none reaches min_area, the largest stays
        region_components(sw, false, N, cnbr, k1, par);
        for (int i = threadIdx.x; i < N; i += blockDim.x) {
            if (par[i] < 0 && region_member(sw, i, N, false)) {
                const int size = -par[i];
                if (size < min_area) any_small = 1;
                atomicMax(&best, ((unsigned long long)size << 32) | (uint32_t)~i);
            }
        }
        __syncthreads();
        const bool drop = any_small != 0;
        const int keep_root = (int)~(uint32_t)(best & 0xffffffffull);
        const bool none_big = (int)(best >> 32) < min_area;
        int a = 0;
        for (int i = threadIdx.x; i < Wn * 32; i += blockDim.x) {
            const uint32_t word = sw[i >> 5];
            bool in = (word >> (i & 31)) & 1u;
            if (drop && in) {
                const int r = region_root(par, i);
                in = none_big ? r == keep_root : -par[r] >= min_area;
            }
            const uint32_t out = __ballot_sync(0xffffffffu, in);
            if (lane == 0) bits_out[(size_t)it * W + (i >> 5)] = out;
            a += in;
        }
        for (int w = Wn + threadIdx.x; w < W; w += blockDim.x) bits_out[(size_t)it * W + w] = 0u;
        a = __reduce_add_sync(0xffffffffu, a);
        if (lane == 0 && a) atomicAdd(&area_red, a);
        __syncthreads();
        if (threadIdx.x == 0) {
            area_out[it] = area_red;
            score_out[it] = (changed || drop) ? 0.f : 1.f;
        }
        __syncthreads();  // sw, par and the shared flags are reused by the next rank
    }
}

}  // namespace

namespace {

int mask_candidates_launch(const float* logits, const float* iou_preds, int B, int Zc, int C, int N, const int* lengths, int P,
                           float mask_threshold, float stability_offset, float pred_iou_thresh, float stability_thresh,
                           int min_area, long long base, long long cloud_stride, int W, uint32_t* bits, int* area,
                           float* stability, float* score, cudaStream_t stream) {
    if (!logits || !iou_preds || !bits || !area || !stability || !score) return PSAM_ERR_ARG;
    if (B <= 0 || Zc <= 0 || C <= 0 || N <= 0 || base < 0 || W < psam::ceil_div(N, 32)) return PSAM_ERR_ARG;
    if ((long long)B * Zc * C > 0x7fffffffLL) return PSAM_ERR_ARG;
    if (B > 1 && cloud_stride < base + (long long)Zc * C) return PSAM_ERR_ARG;  // the clouds' slot blocks must not overlap
    const float thr_hi = mask_threshold + stability_offset, thr_lo = mask_threshold - stability_offset;
    const bool vec = (N % 4 == 0) && (reinterpret_cast<uintptr_t>(logits) % 16 == 0);
    auto kernel = lengths ? (vec ? mask_candidates_kernel<true, true> : mask_candidates_kernel<false, true>)
                          : (vec ? mask_candidates_kernel<true, false> : mask_candidates_kernel<false, false>);
    PSAM_CUDA_TRY(psam::launch(kernel, dim3(B * Zc * C), dim3(kCandThreads), (size_t)0, stream, logits, iou_preds, N, mask_threshold,
                               thr_hi, thr_lo, pred_iou_thresh, stability_thresh, min_area, base, Zc * C, cloud_stride, W, lengths,
                               P, C, bits, area, stability, score));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

}  // namespace

extern "C" int psam_mask_candidates_batched_f32(const float* logits, const float* iou_preds, int B, int Zc, int C, int N,
                                                float mask_threshold, float stability_offset, float pred_iou_thresh,
                                                float stability_thresh, int min_area, long long base, long long cloud_stride,
                                                int W, uint32_t* bits, int* area, float* stability, float* score,
                                                cudaStream_t stream) {
    return mask_candidates_launch(logits, iou_preds, B, Zc, C, N, nullptr, 0, mask_threshold, stability_offset, pred_iou_thresh,
                                  stability_thresh, min_area, base, cloud_stride, W, bits, area, stability, score, stream);
}

extern "C" int psam_mask_candidates_varlen_f32(const float* logits, const float* iou_preds, const int* lengths, int B, int Zc, int C,
                                               int N_max, int P, float mask_threshold, float stability_offset, float pred_iou_thresh,
                                               float stability_thresh, int min_area, long long base, long long cloud_stride, int W,
                                               uint32_t* bits, int* area, float* stability, float* score, cudaStream_t stream) {
    if (!lengths || P < 0) return PSAM_ERR_ARG;
    return mask_candidates_launch(logits, iou_preds, B, Zc, C, N_max, lengths, P, mask_threshold, stability_offset, pred_iou_thresh,
                                  stability_thresh, min_area, base, cloud_stride, W, bits, area, stability, score, stream);
}

extern "C" int psam_mask_candidates_f32(const float* logits, const float* iou_preds, int Z, int C, int N, float mask_threshold,
                                        float stability_offset, float pred_iou_thresh, float stability_thresh, int min_area,
                                        long long base, int W, uint32_t* bits, int* area, float* stability, float* score,
                                        cudaStream_t stream) {
    return psam_mask_candidates_batched_f32(logits, iou_preds, 1, Z, C, N, mask_threshold, stability_offset, pred_iou_thresh,
                                            stability_thresh, min_area, base, 0, W, bits, area, stability, score, stream);
}

extern "C" size_t psam_mask_nms_workspace_bytes(int K, int W) {
    (void)W;
    if (K < 0 || K > kNmsMaxK) return 0;
    const size_t ldm = (size_t)(K + kTile - 1) / kTile;
    return 16 + nms_order_bytes(K) + (size_t)K * ldm * sizeof(unsigned long long);
}

extern "C" size_t psam_mask_nms_batched_workspace_bytes(int B, int K, int W) {
    if (B < 1 || B > kNmsMaxClouds) return 0;
    return (size_t)B * psam_mask_nms_workspace_bytes(K, W);
}

extern "C" int psam_mask_nms_batched(const uint32_t* bits, const int* area, const float* score, int B, int K, int W,
                                     float nms_thresh, int* keep, int* keep_count, void* workspace, cudaStream_t stream) {
    if (!keep || !keep_count || !workspace || B < 1 || B > kNmsMaxClouds || K < 0 || K > kNmsMaxK) return PSAM_ERR_ARG;
    if (K > 0 && (!bits || !area || !score || W <= 0)) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    char* ws = static_cast<char*>(workspace);
    const size_t cloud_bytes = psam_mask_nms_workspace_bytes(K, W);
    const int ldm = (K + kTile - 1) / kTile;
    int P2 = 2;
    while (P2 < K) P2 <<= 1;
    const size_t smem = (size_t)P2 * sizeof(unsigned long long);
    if (smem > 48 * 1024)
        PSAM_CUDA_TRY(cudaFuncSetAttribute(nms_order_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSAM_CUDA_TRY(psam::launch(nms_order_kernel, dim3(B), dim3(1024), smem, stream, score, K, P2, ws, cloud_bytes));
    PSAM_LAUNCH_CHECK();
    if (K > 0) {
        PSAM_CUDA_TRY(psam::launch(nms_pairs_kernel, dim3(ldm, ldm, B), dim3(256), (size_t)0, stream, bits, area, K, W, nms_thresh, ws,
                                   cloud_bytes, ldm));
        PSAM_LAUNCH_CHECK();
    }
    PSAM_CUDA_TRY(psam::launch(nms_scan_kernel, dim3(B), dim3(kScanThreads), (size_t)0, stream, (const char*)ws, cloud_bytes, K, ldm,
                               keep, keep_count));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mask_nms(const uint32_t* bits, const int* area, const float* score, int K, int W, float nms_thresh,
                             int* keep, int* keep_count, void* workspace, cudaStream_t stream) {
    return psam_mask_nms_batched(bits, area, score, 1, K, W, nms_thresh, keep, keep_count, workspace, stream);
}

extern "C" size_t psam_mask_regions_batched_workspace_bytes(int B, int K, int N) {
    if (B < 1 || K < 0 || K > kNmsMaxK || N <= 0 || N > kRegionMaxN) return 0;
    if (N <= kRegionSmemMaxN) return 16;
    const size_t bytes = ((size_t)region_slices((long long)B * K, N) * N * sizeof(int) + 15) / 16 * 16;
    return bytes < 16 ? 16 : bytes;
}

extern "C" size_t psam_mask_regions_workspace_bytes(int K, int N) { return psam_mask_regions_batched_workspace_bytes(1, K, N); }

namespace {

int mask_regions_launch(const uint32_t* bits, long long cloud_slots, int B, int K, int W, int N, const int* lengths, const int* keep,
                        const int* keep_count, const long long* nbr, int k1, int min_area, uint32_t* bits_out, int* area_out,
                        float* score_out, void* workspace, cudaStream_t stream) {
    if (!keep_count || !nbr || !workspace) return PSAM_ERR_ARG;
    if (K > 0 && (!bits || !keep || !bits_out || !area_out || !score_out)) return PSAM_ERR_ARG;
    if (N <= 0 || N > kRegionMaxN || W < psam::ceil_div(N, 32) || k1 < 1 || k1 > N || K < 0 || K > kNmsMaxK || min_area < 1)
        return PSAM_ERR_ARG;
    if (B < 1 || cloud_slots < 0 || (B > 1 && cloud_slots < 1)) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    if (K == 0) return PSAM_OK;
    // persistent grid over the B * K items: two CTAs per SM in the shared-memory form, one per label slice (at most one per
    // SM) otherwise
    const long long items = (long long)B * K;
    int dev = 0, sms = 0;
    PSAM_CUDA_TRY(cudaGetDevice(&dev));
    PSAM_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int grid = N <= kRegionSmemMaxN ? (int)(items < 2 * sms ? items : 2 * sms) : min(region_slices(items, N), sms);
    const size_t words = (size_t)(psam::ceil_div(N, 32) + 3) / 4 * 4 * sizeof(uint32_t);
    if (N <= kRegionSmemMaxN) {
        const size_t smem = words + (size_t)N * sizeof(int);
        auto kernel = lengths ? mask_regions_kernel<true, true> : mask_regions_kernel<true, false>;
        PSAM_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        PSAM_CUDA_TRY(psam::launch(kernel, dim3(grid), dim3(kRegionThreads), smem, stream, bits, cloud_slots, B, K, W, N, lengths, keep,
                                   keep_count, nbr, k1, min_area, bits_out, area_out, score_out, (int*)nullptr));
    } else {
        auto kernel = lengths ? mask_regions_kernel<false, true> : mask_regions_kernel<false, false>;
        PSAM_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)words));
        PSAM_CUDA_TRY(psam::launch(kernel, dim3(grid), dim3(kRegionThreads), words, stream, bits, cloud_slots, B, K, W, N, lengths,
                                   keep, keep_count, nbr, k1, min_area, bits_out, area_out, score_out, static_cast<int*>(workspace)));
    }
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

}  // namespace

extern "C" int psam_mask_regions_batched(const uint32_t* bits, long long cloud_slots, int B, int K, int W, int N, const int* keep,
                                         const int* keep_count, const long long* nbr, int k1, int min_area, uint32_t* bits_out,
                                         int* area_out, float* score_out, void* workspace, cudaStream_t stream) {
    return mask_regions_launch(bits, cloud_slots, B, K, W, N, nullptr, keep, keep_count, nbr, k1, min_area, bits_out, area_out,
                               score_out, workspace, stream);
}

extern "C" int psam_mask_regions_varlen(const uint32_t* bits, long long cloud_slots, const int* lengths, int B, int K, int W, int N_max,
                                        const int* keep, const int* keep_count, const long long* nbr, int k1, int min_area,
                                        uint32_t* bits_out, int* area_out, float* score_out, void* workspace, cudaStream_t stream) {
    if (!lengths) return PSAM_ERR_ARG;
    return mask_regions_launch(bits, cloud_slots, B, K, W, N_max, lengths, keep, keep_count, nbr, k1, min_area, bits_out, area_out,
                               score_out, workspace, stream);
}

extern "C" int psam_mask_regions(const uint32_t* bits, int K, int W, int N, const int* keep, const int* keep_count,
                                 const long long* nbr, int k1, int min_area, uint32_t* bits_out, int* area_out, float* score_out,
                                 void* workspace, cudaStream_t stream) {
    return psam_mask_regions_batched(bits, 0, 1, K, W, N, keep, keep_count, nbr, k1, min_area, bits_out, area_out, score_out,
                                     workspace, stream);
}
