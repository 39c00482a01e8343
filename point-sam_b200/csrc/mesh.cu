// Meshes and dense clouds: area-weighted surface sampling of a triangle mesh, face centres, and the two kernels that carry
// bit-packed masks over S points back to M other points (a mesh's vertices or faces, or the points of a dense scan) and
// turn a set of masks into one part label per point.  The semantics are stated in include/psam_b200.h.
//
//   mesh_area_kernel        one thread per face: twice the area (fp32, stated order), validity, the largest area as an
//                           atomicMax on its bit pattern and the bad-face counts as integer atomics (order-independent).
//   mesh_scan_block_kernel  one CTA per chunk of 1024 faces: the fixed-point weight of each face (exact fp64 scaling of
//                           its area by the power of two of the largest) and the chunk's inclusive prefix sums (uint64).
//   mesh_scan_sums_kernel   one CTA: exclusive scan of the chunk totals in place; the total weight goes to the stats.
//   mesh_scan_add_kernel    one CTA per chunk: adds the chunk's offset, so cdf[] is the exact inclusive prefix sum.
//   mesh_sample_kernel      one thread per sample: counter-based hash streams, face by binary search in cdf[], the
//                           barycentric point clamped to the face's box, and the colour.
//   mesh_centers_kernel     one thread per face.
//   mask_lift_kernel        one warp per 4 output words: each lane keeps its nearest index in a register across all rows,
//                           gathers its bit from the (L2-resident) source row, and a ballot forms the word.
//   mask_area_kernel        one warp per row: popcount of the lifted row.
//   mask_label_kernel       one thread per point, the rows' priorities staged in shared memory: min over (priority, row).
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace {

constexpr int kAreaThreads = 256;
constexpr int kScan = 1024;  // faces per CTA of the scan (one per thread)
constexpr int kSampleThreads = 256;
constexpr int kLiftWarps = 8;
constexpr int kLiftWords = 4;  // output words per warp
constexpr int kAreaWarps = 8;
constexpr int kLabelThreads = 256;
constexpr int kLabelTile = 1024;  // priorities staged per pass

struct Tri {
    float a[3], b[3], c[3];
};

__device__ __forceinline__ bool load_tri(const float* __restrict__ v, int V, const int* __restrict__ faces, long long f, Tri& t) {
    const int i0 = faces[f * 3], i1 = faces[f * 3 + 1], i2 = faces[f * 3 + 2];
    if (i0 < 0 || i0 >= V || i1 < 0 || i1 >= V || i2 < 0 || i2 >= V) return false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        t.a[a] = v[(size_t)i0 * 3 + a];
        t.b[a] = v[(size_t)i1 * 3 + a];
        t.c[a] = v[(size_t)i2 * 3 + a];
    }
    return true;
}

// twice the triangle's area: e1 = b - a, e2 = c - a, n = e1 x e2, sqrt((nx*nx + ny*ny) + nz*nz); every operation rounded
// on its own
__device__ __forceinline__ float twice_area(const Tri& t) {
    float e1[3], e2[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        e1[a] = __fsub_rn(t.b[a], t.a[a]);
        e2[a] = __fsub_rn(t.c[a], t.a[a]);
    }
    const float nx = __fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
    const float ny = __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
    const float nz = __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
}

__global__ void __launch_bounds__(kAreaThreads) mesh_area_kernel(const float* __restrict__ v, int V, const int* __restrict__ faces,
                                                                 int F, float* __restrict__ a2, unsigned* __restrict__ maxbits,
                                                                 long long* __restrict__ stats) {
    psam::pdl_prologue();
    const long long f = (long long)blockIdx.x * kAreaThreads + threadIdx.x;
    bool bad = false, bad_index = false;
    if (f < F) {
        Tri t;
        float A = 0.f;
        if (!load_tri(v, V, faces, f, t)) {
            bad = bad_index = true;
        } else {
            A = twice_area(t);
            bad = !(A > 0.f && A <= 3.402823466e38f);  // NaN, zero or infinite
            if (bad) A = 0.f;
        }
        a2[f] = A;
        if (!bad) atomicMax(maxbits, __float_as_uint(A));  // positive floats order like their bit patterns
    }
    const int nbad = __syncthreads_count(bad), nidx = __syncthreads_count(bad_index);
    if (threadIdx.x == 0) {
        if (nbad) atomicAdd(reinterpret_cast<unsigned long long*>(stats + 1), (unsigned long long)nbad);
        if (nidx) atomicAdd(reinterpret_cast<unsigned long long*>(stats + 2), (unsigned long long)nidx);
    }
}

// E with 2^(E-1) <= x < 2^E for a positive finite float x (normal or subnormal)
__device__ __forceinline__ int pow2_exponent(unsigned bits) {
    const int e = (int)((bits >> 23) & 0xffu);
    if (e) return e - 126;
    return (31 - __clz((int)(bits & 0x7fffffu))) - 148;
}

__global__ void __launch_bounds__(kScan) mesh_scan_block_kernel(const float* __restrict__ a2, int F, const unsigned* __restrict__ maxbits,
                                                                unsigned long long* __restrict__ cdf, unsigned long long* __restrict__ bsum) {
    psam::pdl_prologue();
    __shared__ unsigned long long sw[32];
    const unsigned mb = *maxbits;
    const double scale = mb ? ldexp(1.0, 32 - pow2_exponent(mb)) : 0.0;
    const long long f = (long long)blockIdx.x * kScan + threadIdx.x;
    // q = floor(A2 * 2^(32 - E)) < 2^32: the product of a float and a power of two is exact in fp64
    const unsigned long long q = f < F ? (unsigned long long)floor(__dmul_rn((double)a2[f], scale)) : 0ull;
    unsigned long long total;
    const unsigned long long x = psam::block_scan_u64<kScan>(q, sw, total);
    if (f < F) cdf[f] = x;
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScan) mesh_scan_sums_kernel(unsigned long long* __restrict__ bsum, int nb, long long* __restrict__ stats) {
    psam::pdl_prologue();
    psam::scan_block_sums<kScan>(bsum, nb, reinterpret_cast<unsigned long long*>(stats));  // the total weight goes to stats[0]
}

__global__ void __launch_bounds__(kScan) mesh_scan_add_kernel(unsigned long long* __restrict__ cdf, int F,
                                                              const unsigned long long* __restrict__ bsum) {
    psam::pdl_prologue();
    const long long f = (long long)blockIdx.x * kScan + threadIdx.x;
    if (blockIdx.x && f < F) cdf[f] += bsum[blockIdx.x];
}

// splitmix64 finaliser of seed + (3 s + j + 1) * golden: stream j of sample s
__device__ __forceinline__ unsigned long long mesh_hash(unsigned long long seed, long long s, int j) {
    unsigned long long z = seed + (unsigned long long)(3 * s + j + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// (w0 * a + w1 * b) + w2 * c
__device__ __forceinline__ float bary(float w0, float w1, float w2, float a, float b, float c) {
    return __fadd_rn(__fadd_rn(__fmul_rn(w0, a), __fmul_rn(w1, b)), __fmul_rn(w2, c));
}

// fminf / fmaxf (PTX min / max) order -0.0 below +0.0, the header's rule: a zero p inside the box keeps its sign
__device__ __forceinline__ float clamp3(float p, float a, float b, float c) {
    return fminf(fmaxf(p, fminf(fminf(a, b), c)), fmaxf(fmaxf(a, b), c));
}

// texel coordinate floor(t * n + 0.5) clamped into 0 .. n - 1 (a NaN gives 0)
__device__ __forceinline__ int texel(float t, int n) {
    const float x = floorf(__fadd_rn(__fmul_rn(t, (float)n), 0.5f));
    return x >= (float)(n - 1) ? n - 1 : (x > 0.f ? (int)x : 0);
}

__global__ void __launch_bounds__(kSampleThreads) mesh_sample_kernel(
    const float* __restrict__ v, const int* __restrict__ faces, int F, const unsigned long long* __restrict__ cdf,
    const long long* __restrict__ stats, int S, unsigned long long seed, const float* __restrict__ vcol, const float* __restrict__ uv,
    const unsigned char* __restrict__ tex, int H, int Wt, int C, float* __restrict__ xyz, float* __restrict__ rgb,
    int* __restrict__ face_out) {
    psam::pdl_prologue();
    const long long s = (long long)blockIdx.x * kSampleThreads + threadIdx.x;
    if (s >= S) return;
    const unsigned long long total = (unsigned long long)stats[0];
    if (total == 0ull) {
#pragma unroll
        for (int a = 0; a < 3; ++a) xyz[s * 3 + a] = rgb[s * 3 + a] = 0.f;
        face_out[s] = -1;
        return;
    }
    const unsigned long long u = __umul64hi(mesh_hash(seed, s, 0), total);
    int lo = 0, hi = F - 1;  // smallest f with cdf[f] > u; cdf[F - 1] = total > u
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (cdf[mid] > u) hi = mid;
        else lo = mid + 1;
    }
    const int f = lo;
    const int i0 = faces[(size_t)f * 3], i1 = faces[(size_t)f * 3 + 1], i2 = faces[(size_t)f * 3 + 2];
    const float r1 = (float)(mesh_hash(seed, s, 1) >> 40) * 0x1p-24f;
    const float r2 = (float)(mesh_hash(seed, s, 2) >> 40) * 0x1p-24f;
    const float sq = __fsqrt_rn(r1);
    const float w0 = __fsub_rn(1.f, sq), w1 = __fmul_rn(sq, __fsub_rn(1.f, r2)), w2 = __fmul_rn(sq, r2);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float pa = v[(size_t)i0 * 3 + a], pb = v[(size_t)i1 * 3 + a], pc = v[(size_t)i2 * 3 + a];
        xyz[s * 3 + a] = clamp3(bary(w0, w1, w2, pa, pb, pc), pa, pb, pc);
    }
    if (tex) {
        const float tu = bary(w0, w1, w2, uv[(size_t)i0 * 2], uv[(size_t)i1 * 2], uv[(size_t)i2 * 2]);
        const float tv = bary(w0, w1, w2, uv[(size_t)i0 * 2 + 1], uv[(size_t)i1 * 2 + 1], uv[(size_t)i2 * 2 + 1]);
        const int x = texel(tu, Wt), y = texel(__fsub_rn(1.f, tv), H);
        const unsigned char* px = tex + ((size_t)y * Wt + x) * C;
#pragma unroll
        for (int a = 0; a < 3; ++a) rgb[s * 3 + a] = __fdiv_rn((float)px[a], 255.f);
    } else if (vcol) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float ca = vcol[(size_t)i0 * 3 + a], cb = vcol[(size_t)i1 * 3 + a], cc = vcol[(size_t)i2 * 3 + a];
            rgb[s * 3 + a] = clamp3(bary(w0, w1, w2, ca, cb, cc), ca, cb, cc);
        }
    } else {
#pragma unroll
        for (int a = 0; a < 3; ++a) rgb[s * 3 + a] = 0.5f;
    }
    face_out[s] = f;
}

__global__ void __launch_bounds__(kAreaThreads) mesh_centers_kernel(const float* __restrict__ v, int V, const int* __restrict__ faces,
                                                                    int F, float* __restrict__ centers) {
    psam::pdl_prologue();
    const long long f = (long long)blockIdx.x * kAreaThreads + threadIdx.x;
    if (f >= F) return;
    Tri t;
    const bool ok = load_tri(v, V, faces, f, t);
#pragma unroll
    for (int a = 0; a < 3; ++a)
        centers[f * 3 + a] = ok ? __fdiv_rn(__fadd_rn(__fadd_rn(t.a[a], t.b[a]), t.c[a]), 3.f) : __int_as_float(0x7fffffff);
}

__global__ void __launch_bounds__(kLiftWarps * 32) mask_lift_kernel(const uint32_t* __restrict__ bits, int K, int Ws, int S,
                                                                    const long long* __restrict__ nearest, int M, int Wm,
                                                                    uint32_t* __restrict__ out) {
    psam::pdl_prologue();
    const int lane = threadIdx.x & 31;
    const long long w0 = ((long long)blockIdx.x * kLiftWarps + (threadIdx.x >> 5)) * kLiftWords;
    if (w0 >= Wm) return;
    int src[kLiftWords];  // source bit of this lane's point in each of the warp's words, -1: none
#pragma unroll
    for (int j = 0; j < kLiftWords; ++j) {
        const long long t = (w0 + j) * 32 + lane;
        const long long n = t < M ? nearest[t] : -1;
        src[j] = n >= 0 && n < S ? (int)n : -1;
    }
    for (int k = 0; k < K; ++k) {
        const uint32_t* row = bits + (size_t)k * Ws;
        uint32_t word[kLiftWords];
#pragma unroll
        for (int j = 0; j < kLiftWords; ++j) {
            const bool b = src[j] >= 0 && ((__ldg(row + (src[j] >> 5)) >> (src[j] & 31)) & 1u);
            word[j] = __ballot_sync(0xffffffffu, b);
        }
#pragma unroll
        for (int j = 0; j < kLiftWords; ++j)
            if (lane == j && w0 + j < Wm) out[(size_t)k * Wm + w0 + j] = word[j];
    }
}

__global__ void __launch_bounds__(kAreaWarps * 32) mask_area_kernel(const uint32_t* __restrict__ bits, int K, int W, int* __restrict__ area) {
    psam::pdl_prologue();
    const int k = blockIdx.x * kAreaWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (k >= K) return;
    int c = 0;
    for (int w = lane; w < W; w += 32) c += __popc(bits[(size_t)k * W + w]);
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) area[k] = c;
}

__global__ void __launch_bounds__(kLabelThreads) mask_label_kernel(const uint32_t* __restrict__ bits, int K, int W,
                                                                   const int* __restrict__ priority, int N, int* __restrict__ labels) {
    psam::pdl_prologue();
    __shared__ unsigned sprio[kLabelTile];
    const int n = blockIdx.x * kLabelThreads + threadIdx.x;
    const int w = min(n, N - 1) >> 5;  // the same word for the whole warp
    const uint32_t m = 1u << (n & 31);
    unsigned long long best = ~0ull;  // (priority with the sign bit flipped: unsigned order = signed order) << 32 | row
    for (int k0 = 0; k0 < K; k0 += kLabelTile) {
        const int kn = min(kLabelTile, K - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < kn; i += kLabelThreads) sprio[i] = (unsigned)priority[k0 + i] ^ 0x80000000u;
        __syncthreads();
        for (int i = 0; i < kn; ++i)
            if (bits[(size_t)(k0 + i) * W + w] & m) {
                const unsigned long long key = ((unsigned long long)sprio[i] << 32) | (unsigned)(k0 + i);
                best = key < best ? key : best;
            }
    }
    if (n < N) labels[n] = best == ~0ull ? -1 : (int)(best & 0xffffffffu);
}

// workspace layout of psam_mesh_sample_f32: [16 B header: max bits][a2: F floats][cdf: F uint64][chunk sums: nb uint64]
size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace

extern "C" size_t psam_mesh_sample_workspace_bytes(int F) {
    if (F <= 0) return 0;
    const int nb = psam::ceil_div(F, kScan);
    return 16 + align16((size_t)F * 4) + (size_t)F * 8 + align16((size_t)nb * 8);
}

extern "C" int psam_mesh_sample_f32(const float* vertices, int V, const int* faces, int F, int S, unsigned long long seed,
                                    const float* vertex_colors, const float* uv, const unsigned char* texture, int tex_h, int tex_w,
                                    int tex_c, float* xyz_out, float* rgb_out, int* face_out, long long* stats, void* workspace,
                                    cudaStream_t stream) {
    if (!vertices || !faces || !xyz_out || !rgb_out || !face_out || !stats || !workspace) return PSAM_ERR_ARG;
    if (V <= 0 || F <= 0 || S <= 0) return PSAM_ERR_ARG;
    if (texture && (!uv || vertex_colors || tex_h <= 0 || tex_w <= 0 || (tex_c != 3 && tex_c != 4))) return PSAM_ERR_ARG;
    if (!texture && uv) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    const int nb = psam::ceil_div(F, kScan);
    char* ws = static_cast<char*>(workspace);
    unsigned* maxbits = reinterpret_cast<unsigned*>(ws);
    float* a2 = reinterpret_cast<float*>(ws + 16);
    unsigned long long* cdf = reinterpret_cast<unsigned long long*>(ws + 16 + align16((size_t)F * 4));
    unsigned long long* bsum = cdf + F;
    PSAM_CUDA_TRY(cudaMemsetAsync(maxbits, 0, 4, stream));
    PSAM_CUDA_TRY(cudaMemsetAsync(stats, 0, 3 * sizeof(long long), stream));
    PSAM_CUDA_TRY(psam::launch(mesh_area_kernel, dim3(psam::ceil_div(F, kAreaThreads)), dim3(kAreaThreads), (size_t)0, stream, vertices, V,
                               faces, F, a2, maxbits, stats));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(mesh_scan_block_kernel, dim3(nb), dim3(kScan), (size_t)0, stream, (const float*)a2, F,
                               (const unsigned*)maxbits, cdf, bsum));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(mesh_scan_sums_kernel, dim3(1), dim3(kScan), (size_t)0, stream, bsum, nb, stats));
    PSAM_LAUNCH_CHECK();
    if (nb > 1) {
        PSAM_CUDA_TRY(psam::launch(mesh_scan_add_kernel, dim3(nb), dim3(kScan), (size_t)0, stream, cdf, F, (const unsigned long long*)bsum));
        PSAM_LAUNCH_CHECK();
    }
    PSAM_CUDA_TRY(psam::launch(mesh_sample_kernel, dim3(psam::ceil_div(S, kSampleThreads)), dim3(kSampleThreads), (size_t)0, stream,
                               vertices, faces, F, (const unsigned long long*)cdf, (const long long*)stats, S, seed, vertex_colors, uv,
                               texture, tex_h, tex_w, tex_c, xyz_out, rgb_out, face_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mesh_face_centers_f32(const float* vertices, int V, const int* faces, int F, float* centers, cudaStream_t stream) {
    if (!vertices || !faces || !centers || V <= 0 || F <= 0) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(mesh_centers_kernel, dim3(psam::ceil_div(F, kAreaThreads)), dim3(kAreaThreads), (size_t)0, stream,
                               vertices, V, faces, F, centers));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mask_lift(const uint32_t* bits, int K, int Ws, int S, const long long* nearest, int M, int Wm, uint32_t* bits_out,
                              int* area_out, cudaStream_t stream) {
    if (K < 0 || S <= 0 || M <= 0 || Ws < psam::ceil_div(S, 32) || Wm < psam::ceil_div(M, 32)) return PSAM_ERR_ARG;
    if (K == 0) return PSAM_OK;
    if (!bits || !nearest || !bits_out || !area_out) return PSAM_ERR_ARG;
    const long long groups = psam::ceil_div_ll(Wm, kLiftWords);
    PSAM_CUDA_TRY(psam::launch(mask_lift_kernel, dim3((unsigned)psam::ceil_div_ll(groups, kLiftWarps)), dim3(kLiftWarps * 32), (size_t)0,
                               stream, bits, K, Ws, S, nearest, M, Wm, bits_out));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(mask_area_kernel, dim3(psam::ceil_div(K, kAreaWarps)), dim3(kAreaWarps * 32), (size_t)0, stream,
                               (const uint32_t*)bits_out, K, Wm, area_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mask_label_map(const uint32_t* bits, int K, int W, const int* priority, int N, int* labels, cudaStream_t stream) {
    if (K < 0 || N <= 0 || !labels || W < psam::ceil_div(N, 32)) return PSAM_ERR_ARG;
    if (K > 0 && (!bits || !priority)) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(mask_label_kernel, dim3(psam::ceil_div(N, kLabelThreads)), dim3(kLabelThreads), (size_t)0, stream, bits, K,
                               W, priority, N, labels));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
