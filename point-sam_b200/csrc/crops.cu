// Crop layers of automatic mask generation (SAM's crop_n_layers) on a point cloud: the crop layout, the crop gather, the
// edge filter and the uncrop, all on the device.  The semantics are stated in include/psam_b200.h.
//
//   crop_layout_kernel        one CTA: bounding box (min / max reduction), every crop box of every layer, duplicate flags.
//   crop_count_kernel         grid-stride over the points: closed-box membership of every crop, counted per CTA in shared
//                             memory by ballots, then one atomicAdd per crop and CTA (integer sums: order-independent).
//   crop_gather_count_kernel  one CTA per chunk of 1024 points: the chunk's member count and its largest squared distance to
//                             the box centre (fmax: order-independent); zeroes the edge bitset.
//   crop_gather_write_kernel  one CTA per chunk: its offset = the sum of the earlier chunks' counts, so the compaction is
//                             stable (ascending global index) and the same on every run; writes indices, renormalised xyz,
//                             rgb and the edge bits.
//   crop_edge_filter_kernel   one warp per candidate: any(bits & edge) -> score = -inf.
//   crop_uncrop_kernel        persistent CTAs over the kept ranks: zero the global row, scatter the local bits through the
//                             crop's index list, copy the per-mask fields; appends at a device-side offset.
//
// Batches of clouds: every kernel takes a compile-time BATCH flag that adds a grid dimension (blockIdx.y = cloud for the
// layout and count, = (cloud, crop) pair for the gather, = crop for the edge filter, = crop run for the uncrop).  The
// single-cloud entry points instantiate BATCH = false, whose code is the code from before the flag.
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace {

constexpr int kCropMaxLayers = 3;  // 1 + 8 + 64 + 512 = 585 crops
constexpr int kLayoutThreads = 1024;
constexpr int kCountThreads = 256;
constexpr int kCountMaxBlocks = 512;
constexpr int kChunk = 1024;  // points per CTA of the gather (one per thread)
constexpr int kUncropThreads = 256;
constexpr int kUncropMaxBlocks = 264;
constexpr int kFilterWarps = 8;

__host__ __device__ inline int crop_total(int layers) {
    int t = 0, m = 1;
    for (int i = 0; i <= layers; ++i, m *= 8) t += m;
    return t;
}

// crop t -> (layer, n = 2^layer, jx, jy, jz)
__device__ inline void crop_coords(int t, int& layer, int& n, int (&j)[3]) {
    int base = 0, m = 1;
    layer = 0;
    while (t >= base + m) {
        base += m;
        m *= 8;
        ++layer;
    }
    n = 1 << layer;
    const int q = t - base;
    j[0] = q / (n * n);
    j[1] = (q / n) % n;
    j[2] = q % n;
}

// one axis of crop j of n (the evaluation order of include/psam_b200.h; explicit _rn intrinsics, so nothing is contracted)
__device__ inline void crop_bounds(float lo, float hi, int n, int j, float r, float& b0, float& b1) {
    const float L = __fsub_rn(hi, lo);
    const float o = __fdiv_rn(__fmul_rn(__fmul_rn(r, L), 2.f), (float)n);
    const float s = __fdiv_rn(__fadd_rn(L, __fmul_rn(o, (float)(n - 1))), (float)n);
    b0 = __fadd_rn(lo, __fmul_rn((float)j, __fsub_rn(s, o)));
    b1 = j == n - 1 ? hi : __fadd_rn(b0, s);
}

__device__ __forceinline__ bool in_box(float x, float y, float z, const float* b) {
    return b[0] <= x && x <= b[3] && b[1] <= y && y <= b[4] && b[2] <= z && z <= b[5];
}

// BATCH: cloud blockIdx.y of B clouds [B, N, 3] (N = N_max), its first clamp(lengths[b], 0, N) points when lengths is given;
// boxes [B, T, 6], counts [B, T].  !BATCH is psam_crop_layout_f32's single cloud (lengths unused).
template <bool BATCH>
__global__ void __launch_bounds__(kLayoutThreads) crop_layout_kernel(const float* __restrict__ xyz, int N, int layers, float r,
                                                                     float* __restrict__ boxes, int* __restrict__ counts,
                                                                     const int* __restrict__ lengths) {
    psam::pdl_prologue();
    if constexpr (BATCH) {
        const int b = blockIdx.y, T = crop_total(layers);
        xyz += (size_t)b * N * 3;
        boxes += (size_t)b * T * 6;
        counts += (size_t)b * T;
        if (lengths) N = min(max(lengths[b], 0), N);
    }
    extern __shared__ float sbox[];  // [T, 6]
    __shared__ float red[6][kLayoutThreads / 32];
    __shared__ float bb[6];
    // fminf / fmaxf ignore NaN and order -0.0 below +0.0 (PTX min / max), so the box is the same in any reduction order
    float v[6] = {INFINITY, INFINITY, INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float p = xyz[(size_t)i * 3 + a];
            v[a] = fminf(v[a], p);
            v[3 + a] = fmaxf(v[3 + a], p);
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        for (int off = 16; off; off >>= 1) {
            const float u = __shfl_xor_sync(0xffffffffu, v[a], off);
            v[a] = a < 3 ? fminf(v[a], u) : fmaxf(v[a], u);
        }
        if (lane == 0) red[a][warp] = v[a];
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        const int a = threadIdx.x;
        float m = red[a][0];
        for (int w = 1; w < nw; ++w) m = a < 3 ? fminf(m, red[a][w]) : fmaxf(m, red[a][w]);
        bb[a] = m;
    }
    __syncthreads();
    const int T = crop_total(layers);
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        int layer, n, j[3];
        crop_coords(t, layer, n, j);
#pragma unroll
        for (int a = 0; a < 3; ++a) crop_bounds(bb[a], bb[3 + a], n, j[a], r, sbox[t * 6 + a], sbox[t * 6 + 3 + a]);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) {
        int layer, n, j[3];
        crop_coords(t, layer, n, j);
        const int start = layer == 0 ? 0 : crop_total(layer - 1);  // the first crop of this layer
        bool dup = false;
        for (int u = start; u < t && !dup; ++u) {
            bool same = true;
#pragma unroll
            for (int e = 0; e < 6; ++e) same = same && sbox[u * 6 + e] == sbox[t * 6 + e];
            dup = same;
        }
#pragma unroll
        for (int e = 0; e < 6; ++e) boxes[t * 6 + e] = sbox[t * 6 + e];
        counts[t] = dup ? -1 : 0;
    }
}

template <bool BATCH>
__global__ void __launch_bounds__(kCountThreads) crop_count_kernel(const float* __restrict__ xyz, int N, int T,
                                                                   const float* __restrict__ boxes, int* __restrict__ counts,
                                                                   const int* __restrict__ lengths) {
    psam::pdl_prologue();
    if constexpr (BATCH) {  // cloud blockIdx.y, as crop_layout_kernel<true>: padded rows are never read
        const int b = blockIdx.y;
        xyz += (size_t)b * N * 3;
        boxes += (size_t)b * T * 6;
        counts += (size_t)b * T;
        if (lengths) N = min(max(lengths[b], 0), N);
    }
    extern __shared__ float cbox[];  // [T, 6] boxes, then T counters (-1: duplicate crop, not counted)
    int* scnt = reinterpret_cast<int*>(cbox + 6 * T);
    for (int e = threadIdx.x; e < 6 * T; e += blockDim.x) cbox[e] = boxes[e];
    for (int t = threadIdx.x; t < T; t += blockDim.x) scnt[t] = counts[t] < 0 ? -1 : 0;  // the sign is set by the layout
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int base = blockIdx.x * blockDim.x; base < N; base += gridDim.x * blockDim.x) {
        const int i = base + threadIdx.x;
        const bool valid = i < N;
        const float x = valid ? xyz[(size_t)i * 3] : 0.f, y = valid ? xyz[(size_t)i * 3 + 1] : 0.f,
                    z = valid ? xyz[(size_t)i * 3 + 2] : 0.f;
        for (int t = 0; t < T; ++t) {
            if (scnt[t] < 0) continue;  // block-uniform
            const uint32_t b = __ballot_sync(0xffffffffu, valid && in_box(x, y, z, cbox + t * 6));
            if (lane == 0 && b) atomicAdd(scnt + t, __popc(b));
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x)
        if (scnt[t] > 0) atomicAdd(counts + t, scnt[t]);
}

// squared distance to the box centre, in the evaluation order of include/psam_b200.h
__device__ __forceinline__ void crop_centre(const float* box, float (&c)[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = __fmul_rn(__fadd_rn(box[a], box[3 + a]), 0.5f);
}

// Pair blockIdx.y of the batched gather: pairs [3, P] holds the clouds, crops and counts.  Returns its cloud, crop and count,
// and turns N (N_max on entry) into the number of the cloud's points to scan; a pair outside its ranges scans none and has
// count 0 (its rows stay zero).
__device__ __forceinline__ void gather_pair(const int* __restrict__ pairs, int P, int B, int n_crops, int n_max,
                                            const int* __restrict__ lengths, int& N, int& crop, int& count, int& cloud) {
    const int p = blockIdx.y;
    cloud = pairs[p];
    crop = pairs[P + p];
    count = pairs[2 * P + p];
    if (cloud < 0 || cloud >= B || crop < 0 || crop >= n_crops || count < 0 || count > n_max) {
        cloud = crop = count = N = 0;
        return;
    }
    if (lengths) N = min(max(lengths[cloud], 0), N);
}

// BATCH: pair blockIdx.y of the batched gather (gather_pair); `box` is then the boxes [B, n_crops, 6] of every cloud, and the
// pair's rows [count, n_max) of idx_out / xyz_out / rgb_out [P, n_max(, 3)] are zeroed here (the write kernel fills the
// others).  !BATCH is psam_crop_gather_f32's single crop (the batch arguments unused).
template <bool BATCH>
__global__ void __launch_bounds__(kChunk) crop_gather_count_kernel(const float* __restrict__ xyz, int N, const float* __restrict__ box,
                                                                   int* __restrict__ chunk_cnt, uint32_t* __restrict__ chunk_max,
                                                                   uint32_t* __restrict__ edge, int We, const int* __restrict__ pairs,
                                                                   int P, int B, int n_crops, int n_max, const int* __restrict__ lengths,
                                                                   int* __restrict__ idx_out, float* __restrict__ xyz_out,
                                                                   float* __restrict__ rgb_out) {
    psam::pdl_prologue();
    if constexpr (BATCH) {
        int crop, count, cloud;
        const int N_max = N;
        gather_pair(pairs, P, B, n_crops, n_max, lengths, N, crop, count, cloud);
        xyz += (size_t)cloud * N_max * 3;
        box += ((size_t)cloud * n_crops + crop) * 6;
        const size_t p = blockIdx.y;
        chunk_cnt += p * gridDim.x;
        chunk_max += p * gridDim.x;
        edge += p * We;
        for (int q = count + blockIdx.x * kChunk + threadIdx.x; q < n_max; q += gridDim.x * kChunk) {
            idx_out[p * n_max + q] = 0;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                xyz_out[(p * n_max + q) * 3 + a] = 0.f;
                rgb_out[(p * n_max + q) * 3 + a] = 0.f;
            }
        }
    }
    __shared__ int wc[kChunk / 32];
    __shared__ float wm[kChunk / 32];
    const int i = blockIdx.x * kChunk + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float c[3];
    crop_centre(box, c);
    bool in = false;
    float d2 = 0.f;
    if (i < N) {
        const float p[3] = {xyz[(size_t)i * 3], xyz[(size_t)i * 3 + 1], xyz[(size_t)i * 3 + 2]};
        in = in_box(p[0], p[1], p[2], box);
        if (in) {
            const float dx = __fsub_rn(p[0], c[0]), dy = __fsub_rn(p[1], c[1]), dz = __fsub_rn(p[2], c[2]);
            d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        }
    }
    const int cnt = __popc(__ballot_sync(0xffffffffu, in));
    for (int off = 16; off; off >>= 1) d2 = fmaxf(d2, __shfl_xor_sync(0xffffffffu, d2, off));
    if (lane == 0) {
        wc[warp] = cnt;
        wm[warp] = d2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        float m = 0.f;
        for (int w = 0; w < kChunk / 32; ++w) {
            s += wc[w];
            m = fmaxf(m, wm[w]);
        }
        chunk_cnt[blockIdx.x] = s;
        chunk_max[blockIdx.x] = __float_as_uint(m);
    }
    for (int w = blockIdx.x * kChunk + threadIdx.x; w < We; w += gridDim.x * kChunk) edge[w] = 0u;
}

// BATCH: pair blockIdx.y (gather_pair); `bbox` is then the boxes [B, n_crops, 6] of every cloud, and the outputs are the
// pair's rows of idx_out / xyz_out / rgb_out [P, n_max(, 3)] and edge [P, We].
template <bool BATCH>
__global__ void __launch_bounds__(kChunk) crop_gather_write_kernel(const float* __restrict__ xyz, const float* __restrict__ rgb, int N,
                                                                   const float* __restrict__ bbox, const float* __restrict__ box,
                                                                   float margin, int n_out, const int* __restrict__ chunk_cnt,
                                                                   const uint32_t* __restrict__ chunk_max, int nchunks,
                                                                   int* __restrict__ idx_out, float* __restrict__ xyz_out,
                                                                   float* __restrict__ rgb_out, uint32_t* __restrict__ edge,
                                                                   const int* __restrict__ pairs, int P, int B, int n_crops,
                                                                   int n_max, const int* __restrict__ lengths, int We) {
    psam::pdl_prologue();
    if constexpr (BATCH) {
        int crop, cloud;
        const int N_max = N;
        gather_pair(pairs, P, B, n_crops, n_max, lengths, N, crop, n_out, cloud);
        xyz += (size_t)cloud * N_max * 3;
        rgb += (size_t)cloud * N_max * 3;
        bbox += (size_t)cloud * n_crops * 6;
        box = bbox + (size_t)crop * 6;
        const size_t p = blockIdx.y;
        chunk_cnt += p * nchunks;
        chunk_max += p * nchunks;
        idx_out += p * n_max;
        xyz_out += p * n_max * 3;
        rgb_out += p * n_max * 3;
        edge += p * We;
    }
    __shared__ int wpre[kChunk / 32 + 1];
    __shared__ int red_s[kChunk / 32];
    __shared__ float red_m[kChunk / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // this chunk's offset (earlier chunks only) and the crop's largest squared distance (all chunks)
    int pre = 0;
    float m = 0.f;
    for (int k = threadIdx.x; k < nchunks; k += blockDim.x) {
        if (k < (int)blockIdx.x) pre += chunk_cnt[k];
        m = fmaxf(m, __uint_as_float(chunk_max[k]));
    }
    pre = __reduce_add_sync(0xffffffffu, pre);
    for (int off = 16; off; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) {
        red_s[warp] = pre;
        red_m[warp] = m;
    }
    const int i = blockIdx.x * kChunk + threadIdx.x;
    float c[3], p[3] = {0.f, 0.f, 0.f};
    crop_centre(box, c);
    bool in = false;
    if (i < N) {
        p[0] = xyz[(size_t)i * 3];
        p[1] = xyz[(size_t)i * 3 + 1];
        p[2] = xyz[(size_t)i * 3 + 2];
        in = in_box(p[0], p[1], p[2], box);
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, in);
    if (lane == 0) wpre[warp + 1] = __popc(bal);
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        float mm = 0.f;
        for (int w = 0; w < kChunk / 32; ++w) {
            s += red_s[w];
            mm = fmaxf(mm, red_m[w]);
        }
        red_s[0] = s;
        red_m[0] = mm;
        wpre[0] = 0;
        for (int w = 1; w <= kChunk / 32; ++w) wpre[w] += wpre[w - 1];
    }
    __syncthreads();
    if (!in) return;
    const int pos = red_s[0] + wpre[warp] + __popc(bal & ((1u << lane) - 1u));
    if (pos >= n_out) return;
    const float scale = __fsqrt_rn(red_m[0]);
    idx_out[pos] = i;
    bool near = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float d = __fsub_rn(p[a], c[a]);
        xyz_out[(size_t)pos * 3 + a] = scale > 0.f ? __fdiv_rn(d, scale) : 0.f;
        rgb_out[(size_t)pos * 3 + a] = rgb[(size_t)i * 3 + a];
        const float ma = __fmul_rn(margin, __fsub_rn(bbox[3 + a], bbox[a]));
        near = near || (box[a] != bbox[a] && __fsub_rn(p[a], box[a]) <= ma) ||
               (box[3 + a] != bbox[3 + a] && __fsub_rn(box[3 + a], p[a]) <= ma);
    }
    if (near) atomicOr(edge + (pos >> 5), 1u << (pos & 31));
}

// BATCH: crop blockIdx.y of bits [T, K, W], edge [T, W] and score [T, K].
template <bool BATCH>
__global__ void __launch_bounds__(kFilterWarps * 32) crop_edge_filter_kernel(const uint32_t* __restrict__ bits, int K, int W,
                                                                             const uint32_t* __restrict__ edge, float* __restrict__ score) {
    psam::pdl_prologue();
    if constexpr (BATCH) {
        const size_t t = blockIdx.y;
        bits += t * K * W;
        edge += t * W;
        score += t * K;
    }
    const int lane = threadIdx.x & 31;
    for (int k = blockIdx.x * kFilterWarps + (threadIdx.x >> 5); k < K; k += gridDim.x * kFilterWarps) {
        uint32_t hit = 0;
        for (int w = lane; w < W; w += 32) hit |= bits[(size_t)k * W + w] & edge[w];
        if (__any_sync(0xffffffffu, hit != 0) && lane == 0) score[k] = -INFINITY;
    }
}

// BATCH: run blockIdx.y of runs[] supplies the crop's arguments, and the outputs are its cloud's rows of [B, cloud_rows(, Wg)];
// the offset is the exclusive prefix of the keep counts of the cloud's earlier runs (runs[first .. blockIdx.y)), and only the
// cloud's last run writes its lifted count and overflow flag.  !BATCH is psam_crop_uncrop (runs / cloud_rows / lifted unused).
template <bool BATCH>
__global__ void __launch_bounds__(kUncropThreads) crop_uncrop_kernel(
    const uint32_t* __restrict__ bits, const int* __restrict__ area, const float* __restrict__ score,
    const float* __restrict__ stability, int W, const int* __restrict__ keep, const int* __restrict__ keep_count,
    const int* __restrict__ idx, int n, const long long* __restrict__ prompt_index, int slots, int crop, float layer_score,
    int Wg, int capacity, const int* __restrict__ offset_in, int* __restrict__ offset_out, uint32_t* __restrict__ gbits,
    int* __restrict__ garea, float* __restrict__ giou, float* __restrict__ gstab, long long* __restrict__ gprompt,
    int* __restrict__ gslot, int* __restrict__ gcrop, float* __restrict__ gscore, int* __restrict__ overflow,
    const psam_crop_run* __restrict__ runs, int cloud_rows, int* __restrict__ lifted) {
    psam::pdl_prologue();
    int count, base;
    if constexpr (BATCH) {
        __shared__ int red[kUncropThreads / 32];
        const psam_crop_run& r = runs[blockIdx.y];
        bits = r.bits;
        area = r.area;
        score = r.score;
        stability = r.stability;
        W = r.W;
        keep = r.keep;
        idx = r.idx;
        n = r.n;
        prompt_index = r.prompt_index;
        slots = r.slots;
        crop = r.crop;
        layer_score = r.layer_score;
        capacity = min(r.capacity, cloud_rows);
        const size_t c = r.cloud, rows = (size_t)c * cloud_rows;
        gbits += rows * Wg;
        garea += rows;
        giou += rows;
        gstab += rows;
        gprompt += rows;
        gslot += rows;
        gcrop += rows;
        gscore += rows;
        int pre = 0;
        for (int u = r.first + threadIdx.x; u < (int)blockIdx.y; u += blockDim.x) pre += *runs[u].keep_count;
        pre = __reduce_add_sync(0xffffffffu, pre);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = pre;
        __syncthreads();
        base = 0;
#pragma unroll
        for (int w = 0; w < kUncropThreads / 32; ++w) base += red[w];
        count = *r.keep_count;
        if (blockIdx.x == 0 && threadIdx.x == 0 && r.last) {
            lifted[c] = base + count;
            overflow[c] = base + count > capacity ? 1 : 0;
        }
    } else {
        count = *keep_count;
        base = *offset_in;
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            *offset_out = base + count;
            if (base + count > capacity) *overflow = 1;
        }
    }
    for (int p = blockIdx.x; p < count; p += gridDim.x) {
        const int dst = base + p;
        if (dst >= capacity) break;
        const int s = keep[p];
        uint32_t* row = gbits + (size_t)dst * Wg;
        for (int w = threadIdx.x; w < Wg; w += blockDim.x) row[w] = 0u;
        __syncthreads();
        for (int w = threadIdx.x; w < W; w += blockDim.x) {
            uint32_t word = bits[(size_t)s * W + w];
            while (word) {
                const int k = w * 32 + __ffs(word) - 1;
                word &= word - 1u;
                if (k >= n) break;
                const int g = idx[k];
                atomicOr(row + (g >> 5), 1u << (g & 31));
            }
        }
        if (threadIdx.x == 0) {
            const int z = s / slots;
            garea[dst] = area[s];
            giou[dst] = score[s];
            gstab[dst] = stability[s];
            gprompt[dst] = idx[prompt_index[z]];
            gslot[dst] = s - z * slots;
            gcrop[dst] = crop;
            gscore[dst] = layer_score;
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" int psam_crop_total(int n_layers) { return n_layers < 0 || n_layers > kCropMaxLayers ? 0 : crop_total(n_layers); }

extern "C" int psam_crop_layout_f32(const float* xyz, int N, int n_layers, float overlap_ratio, float* boxes, int* counts,
                                    cudaStream_t stream) {
    if (!xyz || !boxes || !counts || N <= 0 || n_layers < 0 || n_layers > kCropMaxLayers) return PSAM_ERR_ARG;
    if (!(overlap_ratio >= 0.f && overlap_ratio < 1.f)) return PSAM_ERR_ARG;
    const int T = crop_total(n_layers);
    PSAM_CUDA_TRY(psam::launch(crop_layout_kernel<false>, dim3(1), dim3(kLayoutThreads), (size_t)T * 6 * sizeof(float), stream, xyz,
                               N, n_layers, overlap_ratio, boxes, counts, (const int*)nullptr));
    PSAM_LAUNCH_CHECK();
    const int grid = min(psam::ceil_div(N, kCountThreads), kCountMaxBlocks);
    PSAM_CUDA_TRY(psam::launch(crop_count_kernel<false>, dim3(grid), dim3(kCountThreads), (size_t)T * 7 * sizeof(float), stream, xyz, N,
                               T, (const float*)boxes, counts, (const int*)nullptr));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" size_t psam_crop_gather_workspace_bytes(int N) {
    if (N <= 0) return 0;
    return (size_t)psam::ceil_div(N, kChunk) * 8 + 16;
}

extern "C" int psam_crop_gather_f32(const float* xyz, const float* rgb, int N, const float* boxes, int crop, int n_crops,
                                    float edge_margin, int n_out, int* idx_out, float* xyz_out, float* rgb_out, uint32_t* edge,
                                    void* workspace, cudaStream_t stream) {
    if (!xyz || !rgb || !boxes || !idx_out || !xyz_out || !rgb_out || !edge || !workspace) return PSAM_ERR_ARG;
    if (N <= 0 || n_crops < 1 || crop < 0 || crop >= n_crops || n_out < 1 || n_out > N || !(edge_margin >= 0.f)) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    const int nchunks = psam::ceil_div(N, kChunk);
    int* chunk_cnt = static_cast<int*>(workspace);
    uint32_t* chunk_max = reinterpret_cast<uint32_t*>(static_cast<char*>(workspace) + (size_t)psam::ceil_div(nchunks, 4) * 16);
    const float* box = boxes + (size_t)crop * 6;
    PSAM_CUDA_TRY(psam::launch(crop_gather_count_kernel<false>, dim3(nchunks), dim3(kChunk), (size_t)0, stream, xyz, N, box,
                               chunk_cnt, chunk_max, edge, psam::ceil_div(n_out, 32), (const int*)nullptr, 0, 0, 0, 0,
                               (const int*)nullptr, (int*)nullptr, (float*)nullptr, (float*)nullptr));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(crop_gather_write_kernel<false>, dim3(nchunks), dim3(kChunk), (size_t)0, stream, xyz, rgb, N, boxes,
                               box, edge_margin, n_out, (const int*)chunk_cnt, (const uint32_t*)chunk_max, nchunks, idx_out,
                               xyz_out, rgb_out, edge, (const int*)nullptr, 0, 0, 0, 0, (const int*)nullptr, 0));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_crop_edge_filter(const uint32_t* bits, int K, int W, const uint32_t* edge, float* score, cudaStream_t stream) {
    if (K < 0 || (K > 0 && (!bits || !edge || !score || W <= 0))) return PSAM_ERR_ARG;
    if (K == 0) return PSAM_OK;
    const int grid = min(psam::ceil_div(K, kFilterWarps), 1024);
    PSAM_CUDA_TRY(psam::launch(crop_edge_filter_kernel<false>, dim3(grid), dim3(kFilterWarps * 32), (size_t)0, stream, bits, K, W, edge,
                               score));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_crop_uncrop(const uint32_t* bits, const int* area, const float* score, const float* stability, int K, int W,
                                const int* keep, const int* keep_count, const int* idx, int n, const long long* prompt_index,
                                int slots, int crop, float layer_score, int N, int Wg, int capacity, const int* offset_in,
                                int* offset_out, uint32_t* gbits, int* garea, float* giou, float* gstab, long long* gprompt,
                                int* gslot, int* gcrop, float* gscore, int* overflow, cudaStream_t stream) {
    if (!bits || !area || !score || !stability || !keep || !keep_count || !idx || !prompt_index || !offset_in || !offset_out ||
        !gbits || !garea || !giou || !gstab || !gprompt || !gslot || !gcrop || !gscore || !overflow)
        return PSAM_ERR_ARG;
    if (K < 1 || n < 1 || n > N || W < psam::ceil_div(n, 32) || slots < 1 || crop < 0 || Wg < psam::ceil_div(N, 32) ||
        capacity < 1 || capacity > 16384)
        return PSAM_ERR_ARG;
    const int grid = min(K, kUncropMaxBlocks);
    PSAM_CUDA_TRY(psam::launch(crop_uncrop_kernel<false>, dim3(grid), dim3(kUncropThreads), (size_t)0, stream, bits, area, score,
                               stability, W, keep, keep_count, idx, n, prompt_index, slots, crop, layer_score, Wg, capacity,
                               offset_in, offset_out, gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore, overflow,
                               (const psam_crop_run*)nullptr, 0, (int*)nullptr));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" size_t psam_crop_run_bytes(void) { return sizeof(psam_crop_run); }

extern "C" int psam_crop_layout_batched_f32(const float* xyz, const int* lengths, int B, int N_max, int n_layers, float overlap_ratio,
                                            float* boxes, int* counts, cudaStream_t stream) {
    if (!xyz || !boxes || !counts || B < 1 || B > 65535 || N_max <= 0 || n_layers < 0 || n_layers > kCropMaxLayers) return PSAM_ERR_ARG;
    if (!(overlap_ratio >= 0.f && overlap_ratio < 1.f)) return PSAM_ERR_ARG;
    const int T = crop_total(n_layers);
    PSAM_CUDA_TRY(psam::launch(crop_layout_kernel<true>, dim3(1, B), dim3(kLayoutThreads), (size_t)T * 6 * sizeof(float), stream,
                               xyz, N_max, n_layers, overlap_ratio, boxes, counts, lengths));
    PSAM_LAUNCH_CHECK();
    const int grid = min(psam::ceil_div(N_max, kCountThreads), kCountMaxBlocks);
    PSAM_CUDA_TRY(psam::launch(crop_count_kernel<true>, dim3(grid, B), dim3(kCountThreads), (size_t)T * 7 * sizeof(float), stream,
                               xyz, N_max, T, (const float*)boxes, counts, lengths));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" size_t psam_crop_gather_batched_workspace_bytes(int P, int N_max) {
    if (P < 1 || P > 65535 || N_max <= 0) return 0;
    return (size_t)P * psam::ceil_div(psam::ceil_div(N_max, kChunk), 4) * 32;
}

extern "C" int psam_crop_gather_batched_f32(const float* xyz, const float* rgb, const int* lengths, int B, int N_max, const float* boxes,
                                            int n_crops, const int* pairs, int P, int n_max, float edge_margin, int* idx_out,
                                            float* xyz_out, float* rgb_out, uint32_t* edge, void* workspace, cudaStream_t stream) {
    if (!xyz || !rgb || !boxes || !pairs || !idx_out || !xyz_out || !rgb_out || !edge || !workspace) return PSAM_ERR_ARG;
    if (B < 1 || N_max <= 0 || n_crops < 1 || P < 1 || P > 65535 || n_max < 1 || n_max > N_max || !(edge_margin >= 0.f))
        return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    const int nchunks = psam::ceil_div(N_max, kChunk), We = psam::ceil_div(n_max, 32);
    int* chunk_cnt = static_cast<int*>(workspace);
    uint32_t* chunk_max = reinterpret_cast<uint32_t*>(static_cast<char*>(workspace) + (size_t)P * psam::ceil_div(nchunks, 4) * 16);
    PSAM_CUDA_TRY(psam::launch(crop_gather_count_kernel<true>, dim3(nchunks, P), dim3(kChunk), (size_t)0, stream, xyz, N_max, boxes,
                               chunk_cnt, chunk_max, edge, We, pairs, P, B, n_crops, n_max, lengths, idx_out, xyz_out, rgb_out));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(crop_gather_write_kernel<true>, dim3(nchunks, P), dim3(kChunk), (size_t)0, stream, xyz, rgb, N_max,
                               boxes, boxes, edge_margin, 0, (const int*)chunk_cnt, (const uint32_t*)chunk_max, nchunks, idx_out,
                               xyz_out, rgb_out, edge, pairs, P, B, n_crops, n_max, lengths, We));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_crop_edge_filter_batched(const uint32_t* bits, int T, int K, int W, const uint32_t* edge, float* score,
                                             cudaStream_t stream) {
    if (T < 1 || T > 65535 || K < 0 || (K > 0 && (!bits || !edge || !score || W <= 0))) return PSAM_ERR_ARG;
    if (K == 0) return PSAM_OK;
    const int grid = min(psam::ceil_div(K, kFilterWarps), 1024);
    PSAM_CUDA_TRY(psam::launch(crop_edge_filter_kernel<true>, dim3(grid, T), dim3(kFilterWarps * 32), (size_t)0, stream, bits, K, W,
                               edge, score));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_crop_uncrop_batched(const psam_crop_run* runs, int R, int K_max, int B, int N_max, int Wg, int cloud_rows,
                                        uint32_t* gbits, int* garea, float* giou, float* gstab, long long* gprompt, int* gslot,
                                        int* gcrop, float* gscore, int* lifted, int* overflow, cudaStream_t stream) {
    if (!runs || !gbits || !garea || !giou || !gstab || !gprompt || !gslot || !gcrop || !gscore || !lifted || !overflow)
        return PSAM_ERR_ARG;
    if (R < 1 || R > 65535 || K_max < 1 || B < 1 || N_max < 1 || Wg < psam::ceil_div(N_max, 32) || cloud_rows < 1 ||
        cloud_rows > 16384)
        return PSAM_ERR_ARG;
    const int grid = min(K_max, max(16, 2 * kUncropMaxBlocks / R));
    PSAM_CUDA_TRY(psam::launch(crop_uncrop_kernel<true>, dim3(grid, R), dim3(kUncropThreads), (size_t)0, stream, (const uint32_t*)nullptr,
                               (const int*)nullptr, (const float*)nullptr, (const float*)nullptr, 0, (const int*)nullptr,
                               (const int*)nullptr, (const int*)nullptr, 0, (const long long*)nullptr, 0, 0, 0.f, Wg, 0,
                               (const int*)nullptr, (int*)nullptr, gbits, garea, giou, gstab, gprompt, gslot, gcrop, gscore, overflow,
                               runs, cloud_rows, lifted));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
