// Memory-bound glue kernels of the Point-SAM hot path (LayerNorm family, SwiGLU, mini-PointNet first
// layer, group max-pool, softmax, positional encoding, small attention, upsampling, mask product).
// Each kernel cites the reference op it replaces in include/psam_b200.h.
#include <cstdlib>
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ void store_split(__nv_bfloat16* hi, long long plane, long long off, float v) {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[off] = h;
    hi[off + plane] = l;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm family.  Values are read ONCE and kept in registers; mean/variance are the two-pass form
// of F.layer_norm.  Two mappings: one warp per row (many rows) or one CTA per row (few, wide rows -
// the 512-token ViT stream would otherwise occupy 64 CTAs only).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_256(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();  // protect `red` from the previous use
    if (l == 0) red[w] = v;
    __syncthreads();
    float t = (l < 8) ? red[l] : 0.f;
    return warp_sum(t);
}

__device__ __forceinline__ float ln_input(const psam_ln_args& a, const float* x, const float* r, const float* gb, int c) {
    float v = x[c];
    if (r) v += r[c];
    if (gb) v += gb[c];
    return v;
}

__device__ __forceinline__ void ln_store(const psam_ln_args& a, long long row, int c, float v) {
    v = apply_act(v, a.act);
    if (a.y) a.y[row * a.ldy + c] = v;
    if (a.y_hi) store_split((__nv_bfloat16*)a.y_hi, a.y_plane, row * a.ldy_s + c, v);
    if (a.y2_hi) store_split((__nv_bfloat16*)a.y2_hi, a.y2_plane, row * a.ldy2_s + c, v + a.post_add[row * a.ld_post + c]);
}

template <int VPL>  // values per lane, D <= 32*VPL
__global__ void __launch_bounds__(256) layernorm_warp_kernel(const psam_ln_args a) {
    pdl_prologue();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= a.rows) return;
    const float* x = a.x + row * a.ldx;
    const float* r = a.r ? a.r + row * a.ldr : nullptr;
    const float* gb = a.gbias ? a.gbias + (row / a.group_rows) * a.ld_gbias : nullptr;
    float v[VPL];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int c = lane + 32 * i;
        v[i] = c < a.D ? ln_input(a, x, r, gb, c) : 0.f;
        s += v[i];
    }
    const float mean = warp_sum(s) / (float)a.D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i)
        if (lane + 32 * i < a.D) q += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(warp_sum(q) / (float)a.D + a.eps);
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
        const int c = lane + 32 * i;
        if (c < a.D) ln_store(a, row, c, (v[i] - mean) * rstd * a.gamma[c] + a.beta[c]);
    }
    if (a.y_hi)
        for (int c = a.D + lane; c < a.pitch; c += 32) store_split((__nv_bfloat16*)a.y_hi, a.y_plane, row * a.ldy_s + c, 0.f);
}

template <int VPT>  // values per thread, D <= 256*VPT
__global__ void __launch_bounds__(256) layernorm_block_kernel(const psam_ln_args a) {
    pdl_prologue();
    __shared__ float red[8];
    const long long row = blockIdx.x;
    const float* x = a.x + row * a.ldx;
    const float* r = a.r ? a.r + row * a.ldr : nullptr;
    const float* gb = a.gbias ? a.gbias + (row / a.group_rows) * a.ld_gbias : nullptr;
    float v[VPT];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + 256 * i;
        v[i] = c < a.D ? ln_input(a, x, r, gb, c) : 0.f;
        s += v[i];
    }
    const float mean = block_sum_256(s, red) / (float)a.D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i)
        if (threadIdx.x + 256 * i < a.D) q += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(block_sum_256(q, red) / (float)a.D + a.eps);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + 256 * i;
        if (c < a.D) ln_store(a, row, c, (v[i] - mean) * rstd * a.gamma[c] + a.beta[c]);
    }
    if (a.y_hi)
        for (int c = a.D + threadIdx.x; c < a.pitch; c += 256) store_split((__nv_bfloat16*)a.y_hi, a.y_plane, row * a.ldy_s + c, 0.f);
}


// ---- float4-vectorised variants (D % 4 == 0, 16-byte aligned rows): 128-bit loads, 64-bit split stores ----
__device__ __forceinline__ float4 ln_input4(const psam_ln_args& a, const float* x, const float* r, const float* gb, int c) {
    float4 v = *reinterpret_cast<const float4*>(x + c);
    if (r) {
        const float4 t = *reinterpret_cast<const float4*>(r + c);
        v.x += t.x, v.y += t.y, v.z += t.z, v.w += t.w;
    }
    if (gb) {
        const float4 t = *reinterpret_cast<const float4*>(gb + c);
        v.x += t.x, v.y += t.y, v.z += t.z, v.w += t.w;
    }
    return v;
}

__device__ __forceinline__ void ln_store4(const psam_ln_args& a, long long row, int c, float4 v, float mean, float rstd) {
    const float4 g = *reinterpret_cast<const float4*>(a.gamma + c);
    const float4 b = *reinterpret_cast<const float4*>(a.beta + c);
    v.x = apply_act((v.x - mean) * rstd * g.x + b.x, a.act);
    v.y = apply_act((v.y - mean) * rstd * g.y + b.y, a.act);
    v.z = apply_act((v.z - mean) * rstd * g.z + b.z, a.act);
    v.w = apply_act((v.w - mean) * rstd * g.w + b.w, a.act);
    if (a.y) *reinterpret_cast<float4*>(a.y + row * a.ldy + c) = v;
    if (a.y_hi) {
        __nv_bfloat16 h0, h1, h2, h3, l0, l1, l2, l3;
        split_bf16(v.x, h0, l0);
        split_bf16(v.y, h1, l1);
        split_bf16(v.z, h2, l2);
        split_bf16(v.w, h3, l3);
        __nv_bfloat16* p = (__nv_bfloat16*)a.y_hi + row * a.ldy_s + c;
        *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
        *reinterpret_cast<uint2*>(p + a.y_plane) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
    }
    if (a.y2_hi) {
        const float4 t = *reinterpret_cast<const float4*>(a.post_add + row * a.ld_post + c);
        __nv_bfloat16 h0, h1, h2, h3, l0, l1, l2, l3;
        split_bf16(v.x + t.x, h0, l0);
        split_bf16(v.y + t.y, h1, l1);
        split_bf16(v.z + t.z, h2, l2);
        split_bf16(v.w + t.w, h3, l3);
        __nv_bfloat16* p = (__nv_bfloat16*)a.y2_hi + row * a.ldy2_s + c;
        *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
        *reinterpret_cast<uint2*>(p + a.y2_plane) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
    }
}

template <int NV>  // float4 per lane, D <= 128*NV
__global__ void __launch_bounds__(256) layernorm_warp_v4_kernel(const psam_ln_args a) {
    pdl_prologue();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= a.rows) return;
    const float* x = a.x + row * a.ldx;
    const float* r = a.r ? a.r + row * a.ldr : nullptr;
    const float* gb = a.gbias ? a.gbias + (row / a.group_rows) * a.ld_gbias : nullptr;
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        v[i] = c < a.D ? ln_input4(a, x, r, gb, c) : make_float4(0.f, 0.f, 0.f, 0.f);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) / (float)a.D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
        if (4 * lane + 128 * i < a.D) {
            const int c = 4 * lane + 128 * i;
            const float d0 = v[i].x - mean, d1 = c + 1 < a.D ? v[i].y - mean : 0.f, d2 = c + 2 < a.D ? v[i].z - mean : 0.f,
                        d3 = c + 3 < a.D ? v[i].w - mean : 0.f;
            q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
    const float rstd = rsqrtf(warp_sum(q) / (float)a.D + a.eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < a.D) ln_store4(a, row, c, v[i], mean, rstd);
    }
    if (a.y_hi)
        for (int c = a.D + lane; c < a.pitch; c += 32) store_split((__nv_bfloat16*)a.y_hi, a.y_plane, row * a.ldy_s + c, 0.f);
}

template <int NV>  // float4 per thread, D <= 1024*NV
__global__ void __launch_bounds__(256) layernorm_block_v4_kernel(const psam_ln_args a) {
    pdl_prologue();
    __shared__ float red[8];
    const long long row = blockIdx.x;
    const float* x = a.x + row * a.ldx;
    const float* r = a.r ? a.r + row * a.ldr : nullptr;
    const float* gb = a.gbias ? a.gbias + (row / a.group_rows) * a.ld_gbias : nullptr;
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = 4 * threadIdx.x + 1024 * i;
        v[i] = c < a.D ? ln_input4(a, x, r, gb, c) : make_float4(0.f, 0.f, 0.f, 0.f);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = block_sum_256(s, red) / (float)a.D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
        if (4 * threadIdx.x + 1024 * i < a.D) {
            const int c = 4 * threadIdx.x + 1024 * i;
            const float d0 = v[i].x - mean, d1 = c + 1 < a.D ? v[i].y - mean : 0.f, d2 = c + 2 < a.D ? v[i].z - mean : 0.f,
                        d3 = c + 3 < a.D ? v[i].w - mean : 0.f;
            q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
    const float rstd = rsqrtf(block_sum_256(q, red) / (float)a.D + a.eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int c = 4 * threadIdx.x + 1024 * i;
        if (c < a.D) ln_store4(a, row, c, v[i], mean, rstd);
    }
    if (a.y_hi)
        for (int c = a.D + threadIdx.x; c < a.pitch; c += 256) store_split((__nv_bfloat16*)a.y_hi, a.y_plane, row * a.ldy_s + c, 0.f);
}

// SwiGLU + inner LayerNorm, one CTA per row, h = silu(g)*x computed once and kept in registers.
template <int VPT>
__global__ void __launch_bounds__(256)
swiglu_ln_kernel(const float* __restrict__ gx, long long ld, long long x_off, int rows, int H, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, __nv_bfloat16* __restrict__ yh, long long y_plane, long long ldy_s,
                 long long pitch) {
    pdl_prologue();
    __shared__ float red[8];
    const long long row = blockIdx.x;
    const float* g = gx + row * ld;
    const float* x = g + x_off;
    float v[VPT];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + 256 * i;
        v[i] = c < H ? silu(g[c]) * x[c] : 0.f;
        s += v[i];
    }
    const float mean = block_sum_256(s, red) / (float)H;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i)
        if (threadIdx.x + 256 * i < H) q += (v[i] - mean) * (v[i] - mean);
    const float rstd = rsqrtf(block_sum_256(q, red) / (float)H + eps);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int c = threadIdx.x + 256 * i;
        if (c < H) store_split(yh, y_plane, row * ldy_s + c, (v[i] - mean) * rstd * gamma[c] + beta[c]);
    }
    for (int c = H + threadIdx.x; c < pitch; c += 256) store_split(yh, y_plane, row * ldy_s + c, 0.f);
}

// y = act(LN?(x W^T + b)); Cin <= 16; one warp per row, lane owns outputs lane, lane+32, ...
template <int CPL>  // outputs per lane = Cout / 32
__global__ void small_in_linear_kernel(const float* __restrict__ x, int rows, int Cin, const float* __restrict__ W,
                                       const float* __restrict__ b, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, float eps, int use_ln, int act,
                                       __nv_bfloat16* __restrict__ yh, long long y_plane, long long ldy_s) {
    pdl_prologue();
    extern __shared__ float s_w[];  // [Cout*Cin] + [Cout] bias
    const int Cout = CPL * 32;
    for (int i = threadIdx.x; i < Cout * Cin; i += blockDim.x) s_w[i] = W[i];
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) s_w[Cout * Cin + i] = b ? b[i] : 0.f;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int wpb = blockDim.x >> 5;
    for (long long row = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * wpb) {
        float xin[16];
#pragma unroll
        for (int c = 0; c < 16; ++c) xin[c] = c < Cin ? x[row * Cin + c] : 0.f;
        float o[CPL];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < CPL; ++i) {
            const int n = lane + 32 * i;
            float acc = s_w[Cout * Cin + n];
            for (int c = 0; c < Cin; ++c) acc = fmaf(xin[c], s_w[n * Cin + c], acc);
            o[i] = acc;
            s += acc;
        }
        if (use_ln) {
            const float mean = warp_sum(s) / (float)Cout;
            float q = 0.f;
#pragma unroll
            for (int i = 0; i < CPL; ++i) q += (o[i] - mean) * (o[i] - mean);
            const float rstd = rsqrtf(warp_sum(q) / (float)Cout + eps);
#pragma unroll
            for (int i = 0; i < CPL; ++i) o[i] = (o[i] - mean) * rstd * gamma[lane + 32 * i] + beta[lane + 32 * i];
        }
#pragma unroll
        for (int i = 0; i < CPL; ++i) store_split(yh, y_plane, row * ldy_s + lane + 32 * i, apply_act(o[i], act));
    }
}

// Voronoi tokenizer (NNGrouper.forward / group_with_centers_and_nn, pc_sam/model/common.py:190-236): every point is
// described relative to its nearest centre: [ unit direction (3), distance (1), features (C) ].  Also writes the
// split-bf16 copy (row pitch `pitch`, zero padded) that feeds in_proj on the tensor cores.
__global__ void voronoi_features_kernel(const float* __restrict__ xyz, const float* __restrict__ centers,
                                        const long long* __restrict__ nn_idx, const float* __restrict__ feats, int B2, int rep,
                                        int N, int G, int C, float* __restrict__ out, __nv_bfloat16* __restrict__ yh,
                                        long long y_plane, long long pitch) {
    pdl_prologue();
    const long long total = (long long)B2 * N;
    const int CO = 4 + C;
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
        const int b2 = (int)(r / N), b = b2 / rep;
        const long long n = r % N;
        const float* p = xyz + ((size_t)b * N + n) * 3;
        const float* c = centers + ((size_t)b * G + nn_idx[(size_t)b * N + n]) * 3;
        const float dx = p[0] - c[0], dy = p[1] - c[1], dz = p[2] - c[2];
        const float dist = sqrtf(dx * dx + dy * dy + dz * dz);  // torch.linalg.norm: sqrt of the plain sum of squares
        const float inv = 1.0f / fmaxf(dist, 1e-8f);            // nbr_xyz / clamp(dist, min=1e-8)
        float v[4] = {dx * inv, dy * inv, dz * inv, dist};
        float* o = out ? out + (size_t)r * CO : nullptr;
        const float* f = feats + (size_t)r * C;
        for (int ch = 0; ch < CO; ++ch) {
            const float x = ch < 4 ? v[ch] : f[ch - 4];
            if (o) o[ch] = x;
            if (yh) store_split(yh, y_plane, r * pitch + ch, x);
        }
        if (yh)
            for (long long ch = CO; ch < pitch; ++ch) store_split(yh, y_plane, r * pitch + ch, 0.f);
    }
}

__global__ void fill_f32_kernel(float* __restrict__ y, long long n, float v) {
    pdl_prologue();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = v;
}

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// y[b, nn_idx[b, n], :] = max over the points n of a cell (scatter_reduce_("amax", include_self=False) on a zero tensor,
// pc_encoder.py:189-193): y is pre-filled with -inf, cells that receive no point are reset to the zero the reference keeps.
__global__ void scatter_amax_kernel(const float* __restrict__ x, const long long* __restrict__ nn_idx, long long rows, int N, int G,
                                    int D, float* __restrict__ y) {
    pdl_prologue();
    const long long total = rows * (D / 4);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / (D / 4);
        const int c4 = (int)(i % (D / 4)) * 4;
        const float4 v = *reinterpret_cast<const float4*>(x + r * D + c4);
        float* o = y + ((r / N) * G + nn_idx[r]) * (long long)D + c4;
        atomic_max_float(o, v.x), atomic_max_float(o + 1, v.y), atomic_max_float(o + 2, v.z), atomic_max_float(o + 3, v.w);
    }
}

__global__ void scatter_amax_finish_kernel(float* __restrict__ y, long long n) {
    pdl_prologue();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        if (y[i] == __int_as_float(0xff800000)) y[i] = 0.f;
}

__global__ void group_max_kernel(const float* __restrict__ x, long long ldx, int groups, int K, int D, float* __restrict__ y,
                                 long long ldy, __nv_bfloat16* __restrict__ yh, long long y_plane, long long ldy_s) {
    pdl_prologue();
    const int g = blockIdx.x;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        const float* p = x + (long long)g * K * ldx + c;
        float m = p[0];
        for (int k = 1; k < K; ++k) m = fmaxf(m, p[(long long)k * ldx]);
        if (y) y[(long long)g * ldy + c] = m;
        if (yh) store_split(yh, y_plane, (long long)g * ldy_s + c, m);
    }
}

__global__ void softmax_split_kernel(const float* __restrict__ s, long long lds, long long rows, int L, float scale,
                                     __nv_bfloat16* __restrict__ ph, long long p_plane, long long ldp) {
    pdl_prologue();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* x = s + row * lds;
    float m = -3.4e38f;
    for (int c = lane; c < L; c += 32) m = fmaxf(m, x[c] * scale);
    m = warp_max(m);
    float sum = 0.f;
    for (int c = lane; c < L; c += 32) sum += __expf(x[c] * scale - m);
    const float inv = 1.0f / warp_sum(sum);
    for (int c = lane; c < L; c += 32) store_split(ph, p_plane, row * ldp + c, __expf(x[c] * scale - m) * inv);
}

__global__ void transpose_split_kernel(const __nv_bfloat16* __restrict__ src, long long src_plane, long long src_ld,
                                       long long src_z1, long long src_z2, __nv_bfloat16* __restrict__ dst,
                                       long long dst_plane, long long dst_ld, long long dst_z1, long long dst_z2, int rows,
                                       int cols, int nz1) {
    pdl_prologue();
    __shared__ __nv_bfloat16 tile[2][32][34];
    const int z = blockIdx.z, z1 = z % nz1, z2 = z / nz1;
    src += z1 * src_z1 + z2 * src_z2;
    dst += z1 * dst_z1 + z2 * dst_z2;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) {
            tile[0][i][threadIdx.x] = src[(long long)r * src_ld + c];
            tile[1][i][threadIdx.x] = src[(long long)r * src_ld + c + src_plane];
        }
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) {
            dst[(long long)c * dst_ld + r] = tile[0][threadIdx.x][i];
            dst[(long long)c * dst_ld + r + dst_plane] = tile[1][threadIdx.x][i];
        }
    }
}

__global__ void posenc_kernel(const float* __restrict__ coords, long long rows, const float* __restrict__ gauss, int F,
                              const int* __restrict__ labels, const float* __restrict__ emb0, const float* __restrict__ emb1,
                              float* __restrict__ out, int* __restrict__ bad_flag) {
    pdl_prologue();
    const long long row = blockIdx.x;
    if (row >= rows) return;
    const float x = coords[row * 3], y = coords[row * 3 + 1], z = coords[row * 3 + 2];
    if (threadIdx.x == 0 && bad_flag) {
        const float lo = -1.0f - 1e-6f, hi = 1.0f + 1e-6f;
        if (x < lo || y < lo || z < lo || x > hi || y > hi || z > hi) *bad_flag = 1;
    }
    const float* emb = nullptr;
    if (labels) {
        const int l = labels[row];
        emb = l == 0 ? emb0 : (l == 1 ? emb1 : nullptr);
    }
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        // coords @ G accumulates x*g0 + y*g1 + z*g2 in that order, then * 2*pi (prompt_encoder.py:30-32)
        float t = x * gauss[f];
        t = fmaf(y, gauss[F + f], t);
        t = fmaf(z, gauss[2 * F + f], t);
        t *= 6.283185307179586f;
        float sv, cv;
        sincosf(t, &sv, &cv);
        if (emb) {
            sv += emb[f];
            cv += emb[F + f];
        }
        out[row * 2 * F + f] = sv;
        out[row * 2 * F + F + f] = cv;
    }
}

// one warp per (z, head, query); scores kept in shared memory (Lk <= 4096).  Both phases split the KEYS across
// lanes (the value phase accumulates dh partial sums per lane and reduces them with shuffles), so long
// key sequences (tokens -> 512 patches) do not serialise on one lane.
template <int DH, int WPI>  // WPI warps cooperate on one (z, head, query) item, each taking a slice of the keys
__global__ void attention_small_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                       float* __restrict__ o, int Z, int Lq, int Lk, int H, long long ldq, long long ldk,
                                       long long ldv, long long ldo) {
    pdl_prologue();
    extern __shared__ float s_sc[];  // per warp: [Lk scores (only its slice used)] + [DH query] ; then WPI*(DH+2) combine area per item
    const int wpb = blockDim.x >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ipb = wpb / WPI;                 // items per block
    const int sub = w % WPI;                   // key slice of this warp
    const long long item = (long long)blockIdx.x * ipb + w / WPI;
    const bool active = item < (long long)Z * H * Lq;
    const int i = active ? (int)(item % Lq) : 0;
    const int h = active ? (int)((item / Lq) % H) : 0;
    const int z = active ? (int)(item / ((long long)Lq * H)) : 0;
    float* sc = s_sc + (size_t)w * (Lk + DH);
    float* sq = sc + Lk;
    float* comb = s_sc + (size_t)wpb * (Lk + DH) + (size_t)(w / WPI) * WPI * (DH + 2);
    const float* qp = q + ((long long)z * Lq + i) * ldq + h * DH;
    for (int d = lane; d < DH; d += 32) sq[d] = qp[d];
    __syncwarp();
    const float scale = rsqrtf((float)DH);
    const int kchunk = (Lk + WPI - 1) / WPI;
    const int jbeg = sub * kchunk, jend = min(Lk, jbeg + kchunk);
    float m = -3.4e38f;
    for (int j = jbeg + lane; j < jend; j += 32) {
        const float* kp = k + ((long long)z * Lk + j) * ldk + h * DH;
        float acc = 0.f;
#pragma unroll
        for (int d = 0; d < DH; ++d) acc = fmaf(sq[d], kp[d], acc);
        acc *= scale;
        sc[j] = acc;
        m = fmaxf(m, acc);
    }
    m = warp_max(m);
    float sum = 0.f;
    float acc[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = 0.f;
    for (int j = jbeg + lane; j < jend; j += 32) {
        const float e = __expf(sc[j] - m);
        sum += e;
        const float* vp = v + ((long long)z * Lk + j) * ldv + h * DH;
#pragma unroll
        for (int d = 0; d < DH; ++d) acc[d] = fmaf(e, vp[d], acc[d]);
    }
    sum = warp_sum(sum);
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = warp_sum(acc[d]);
    float* op = o + ((long long)z * Lq + i) * ldo + h * DH;
    if (WPI == 1) {
        const float inv = 1.0f / sum;
#pragma unroll
        for (int d = 0; d < DH; ++d)
            if (active && lane == (d & 31)) op[d] = acc[d] * inv;
    } else {
        // combine the WPI partial (max, sum, acc) triples through shared memory
        if (lane == 0) {
            comb[sub * (DH + 2)] = m;
            comb[sub * (DH + 2) + 1] = sum;
        }
#pragma unroll
        for (int d = 0; d < DH; ++d)
            if (lane == (d & 31)) comb[sub * (DH + 2) + 2 + d] = acc[d];
        __syncthreads();
        if (sub == 0 && active) {
            float gm = -3.4e38f;
            for (int t = 0; t < WPI; ++t) gm = fmaxf(gm, comb[t * (DH + 2)]);
            float gs = 0.f;
            for (int t = 0; t < WPI; ++t) gs += comb[t * (DH + 2) + 1] * __expf(comb[t * (DH + 2)] - gm);
            for (int d = lane; d < DH; d += 32) {
                float a2 = 0.f;
                for (int t = 0; t < WPI; ++t) a2 += comb[t * (DH + 2) + 2 + d] * __expf(comb[t * (DH + 2)] - gm);
                op[d] = a2 / gs;
            }
        }
    }
}

__global__ void decoder_prepare_kernel(const float* __restrict__ iou_token, const float* __restrict__ mask_tokens, int nmt,
                                       const float* __restrict__ sparse, int P, const float* __restrict__ pc_emb,
                                       const float* __restrict__ dense, long long dense_z, long long dense_g, int Z, int rep,
                                       int G, int D, float* __restrict__ tokens, float* __restrict__ src) {
    pdl_prologue();
    const int T = 1 + nmt + P;
    const long long n_tok = (long long)Z * T * D, n_src = (long long)Z * G * D;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_tok + n_src; i += (long long)gridDim.x * blockDim.x) {
        if (i < n_tok) {
            const int d = (int)(i % D);
            const int t = (int)((i / D) % T);
            const int z = (int)(i / ((long long)D * T));
            float v;
            if (t == 0) v = iou_token[d];
            else if (t <= nmt) v = mask_tokens[(t - 1) * D + d];
            else v = sparse[((long long)z * P + (t - 1 - nmt)) * D + d];
            tokens[i] = v;
        } else {
            const long long j = i - n_tok;
            const int d = (int)(j % D);
            const int g = (int)((j / D) % G);
            const int z = (int)(j / ((long long)D * G));
            src[j] = pc_emb[((long long)(z / rep) * G + g) * D + d] + dense[z * dense_z + g * dense_g + d];
        }
    }
}

// one warp per point; D % 128 == 0, D <= 1024: lane owns float4 columns 4*lane + 128*i (128-bit loads, 64-bit split stores)
template <int NV>
__global__ void __launch_bounds__(256)
interp_ln_gelu_kernel(const float* __restrict__ f, int Z, int rep, int G, int D, const long long* __restrict__ idx,
                      const float* __restrict__ w, int N, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      __nv_bfloat16* __restrict__ yh, long long y_plane, long long ldy_s) {
    pdl_prologue();
    const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
    const long long total = (long long)Z * N;
    for (long long pt = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); pt < total; pt += (long long)gridDim.x * wpb) {
        const int z = (int)(pt / N);
        const int n = (int)(pt % N);
        const long long o3 = ((long long)(z / rep) * N + n) * 3;
        const float w0 = w[o3], w1 = w[o3 + 1], w2 = w[o3 + 2];
        const float* f0 = f + ((long long)z * G + idx[o3]) * D;
        const float* f1 = f + ((long long)z * G + idx[o3 + 1]) * D;
        const float* f2 = f + ((long long)z * G + idx[o3 + 2]) * D;
        float4 v[NV];
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = 4 * lane + 128 * i;
            const float4 a = *reinterpret_cast<const float4*>(f0 + c), b = *reinterpret_cast<const float4*>(f1 + c),
                         d = *reinterpret_cast<const float4*>(f2 + c);
            v[i].x = (a.x * w0 + b.x * w1) + d.x * w2;
            v[i].y = (a.y * w0 + b.y * w1) + d.y * w2;
            v[i].z = (a.z * w0 + b.z * w1) + d.z * w2;
            v[i].w = (a.w * w0 + b.w * w1) + d.w * w2;
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
        const float mean = warp_sum(s) / (float)D;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const float d0 = v[i].x - mean, d1 = v[i].y - mean, d2 = v[i].z - mean, d3 = v[i].w - mean;
            q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
        const float rstd = rsqrtf(warp_sum(q) / (float)D + eps);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = 4 * lane + 128 * i;
            const float4 g = *reinterpret_cast<const float4*>(gamma + c), b = *reinterpret_cast<const float4*>(beta + c);
            __nv_bfloat16 h0, h1, h2, h3, l0, l1, l2, l3;
            split_bf16(gelu_erf((v[i].x - mean) * rstd * g.x + b.x), h0, l0);
            split_bf16(gelu_erf((v[i].y - mean) * rstd * g.y + b.y), h1, l1);
            split_bf16(gelu_erf((v[i].z - mean) * rstd * g.z + b.z), h2, l2);
            split_bf16(gelu_erf((v[i].w - mean) * rstd * g.w + b.w), h3, l3);
            __nv_bfloat16* p = yh + pt * ldy_s + c;
            *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
            *reinterpret_cast<uint2*>(p + y_plane) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
        }
    }
}

__global__ void mask_dot_kernel(const float* __restrict__ u, long long ldu, const float* __restrict__ hyper, int Z, int C, int N,
                                int D, float* __restrict__ masks) {
    pdl_prologue();
    extern __shared__ float s_h[];  // [C*D] for this z
    const int z = blockIdx.y;
    for (int i = threadIdx.x; i < C * D; i += blockDim.x) s_h[i] = hyper[(long long)z * C * D + i];
    __syncthreads();
    const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
    for (int n = blockIdx.x * wpb + (threadIdx.x >> 5); n < N; n += gridDim.x * wpb) {
        const float* up = u + ((long long)z * N + n) * ldu;
        float acc[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = 0.f;
        for (int d = lane; d < D; d += 32) {
            const float x = up[d];
#pragma unroll
            for (int c = 0; c < 8; ++c)
                if (c < C) acc[c] = fmaf(x, s_h[c * D + d], acc[c]);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (c < C) {
                const float r = warp_sum(acc[c]);
                if (lane == 0) masks[((long long)z * C + c) * N + n] = r;
            }
    }
}

__global__ void add_bcast_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, long long chunk,
                                 long long rep, long long period, float* __restrict__ out) {
    pdl_prologue();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long bi = ((i / chunk) / rep) * chunk + (i % chunk);
        out[i] = a[i] + b[bi % period];
    }
}

__global__ void split_f32_kernel(const float* __restrict__ x, const float* __restrict__ add, long long ld, long long rows, int D,
                                 __nv_bfloat16* __restrict__ yh, long long y_plane, long long ldy_s, long long pitch) {
    pdl_prologue();
    const long long total = rows * pitch;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / pitch;
        const int c = (int)(i % pitch);
        float v = c < D ? x[r * ld + c] : 0.f;
        if (add && c < D) v += add[r * ld + c];
        store_split(yh, y_plane, r * ldy_s + c, v);
    }
}

// fp32 SIMT linear: 64x64 tile, 256 threads, 4x4 per thread
__global__ void __launch_bounds__(256) linear_f32_kernel(const psam_linear_args a) {
    pdl_prologue();
    __shared__ float sx[16][65];
    __shared__ float sw[16][65];
    const int z = blockIdx.z;
    const float* x = a.x + z * a.x_z;
    const float* x2 = a.x2 ? a.x2 + z * a.x2_z : nullptr;
    const float* w = a.w + z * a.w_z;
    const float* b = a.b ? a.b + z * a.b_z : nullptr;
    const float* r = a.r ? a.r + z * a.r_z : nullptr;
    float* y = a.y + z * a.y_z;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < a.K; k0 += 16) {
        for (int i = threadIdx.x; i < 64 * 16; i += 256) {
            const int rr = i >> 4, kk = i & 15;
            const int m = m0 + rr, n = n0 + rr, k = k0 + kk;
            float xv = 0.f, wv = 0.f;
            if (k < a.K) {
                if (m < a.M) {
                    xv = x[(long long)m * a.ldx + k];
                    if (x2) xv += x2[(long long)m * a.ldx + k];
                }
                if (n < a.N) wv = w[(long long)n * a.ldw + k];
            }
            sx[kk][rr] = xv;
            sw[kk][rr] = wv;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            float xa[4], wb[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xa[i] = sx[kk][ty * 4 + i], wb[i] = sw[kk][tx * 4 + i];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xa[i], wb[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
            if (m < a.M && n < a.N) {
                float v = acc[i][j];
                if (b) v += b[n];
                v = apply_act(v, a.act);
                if (r) v += r[(long long)m * a.ldy + n];
                y[(long long)m * a.ldy + n] = v;
            }
        }
}


// fp32 SIMT linear for mid-size M (keys side of the decoder): 32x64 tile, BK=32, float4 loads along K,
// all loads of a k-step in flight before the barrier.  Requires K%4==0, ldx%4==0, ldw%4==0.
__global__ void __launch_bounds__(256) linear_f32_v4_kernel(const psam_linear_args a) {
    pdl_prologue();
    __shared__ float sx[32][33];
    __shared__ float sw[32][65];
    const int z = blockIdx.z;
    const float* x = a.x + z * a.x_z;
    const float* x2 = a.x2 ? a.x2 + z * a.x2_z : nullptr;
    const float* w = a.w + z * a.w_z;
    const float* b = a.b ? a.b + z * a.b_z : nullptr;
    const float* r = a.r ? a.r + z * a.r_z : nullptr;
    float* y = a.y + z * a.y_z;
    const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 64;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, each 2 (m) x 4 (n)
    const int lr = threadIdx.x >> 3, lk = (threadIdx.x & 7) * 4;  // loader: row 0..31, k offset 0..28
    float acc[2][4] = {};
    for (int k0 = 0; k0 < a.K; k0 += 32) {
        float4 xv = make_float4(0.f, 0.f, 0.f, 0.f), w0 = xv, w1 = xv;
        const int k = k0 + lk;
        if (k < a.K) {
            if (m0 + lr < a.M) {
                xv = *reinterpret_cast<const float4*>(x + (long long)(m0 + lr) * a.ldx + k);
                if (x2) {
                    const float4 t = *reinterpret_cast<const float4*>(x2 + (long long)(m0 + lr) * a.ldx + k);
                    xv.x += t.x, xv.y += t.y, xv.z += t.z, xv.w += t.w;
                }
            }
            if (n0 + lr < a.N) w0 = *reinterpret_cast<const float4*>(w + (long long)(n0 + lr) * a.ldw + k);
            if (n0 + 32 + lr < a.N) w1 = *reinterpret_cast<const float4*>(w + (long long)(n0 + 32 + lr) * a.ldw + k);
        }
        __syncthreads();
        sx[lk][lr] = xv.x, sx[lk + 1][lr] = xv.y, sx[lk + 2][lr] = xv.z, sx[lk + 3][lr] = xv.w;
        sw[lk][lr] = w0.x, sw[lk + 1][lr] = w0.y, sw[lk + 2][lr] = w0.z, sw[lk + 3][lr] = w0.w;
        sw[lk][lr + 32] = w1.x, sw[lk + 1][lr + 32] = w1.y, sw[lk + 2][lr + 32] = w1.z, sw[lk + 3][lr + 32] = w1.w;
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 32; ++kk) {
            const float xa0 = sx[kk][ty * 2], xa1 = sx[kk][ty * 2 + 1];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float wb = sw[kk][tx + 16 * j];
                acc[0][j] = fmaf(xa0, wb, acc[0][j]);
                acc[1][j] = fmaf(xa1, wb, acc[1][j]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + ty * 2 + i, n = n0 + tx + 16 * j;
            if (m < a.M && n < a.N) {
                float v = acc[i][j];
                if (b) v += b[n];
                v = apply_act(v, a.act);
                if (r) v += r[(long long)m * a.ldy + n];
                y[(long long)m * a.ldy + n] = v;
            }
        }
}

// Small-M fp32 linear (M <= 16): one warp per output column, lanes stride over K (coalesced weight
// reads), all M rows accumulated at once.  The token side of the prompt decoder is all of this shape.
template <int MR, bool VEC>
__global__ void __launch_bounds__(256) linear_gemv_kernel(const psam_linear_args a) {
    pdl_prologue();
    const int z = blockIdx.y;
    const float* x = a.x + z * a.x_z;
    const float* x2 = a.x2 ? a.x2 + z * a.x2_z : nullptr;
    const float* w = a.w + z * a.w_z;
    const float* b = a.b ? a.b + z * a.b_z : nullptr;
    const float* r = a.r ? a.r + z * a.r_z : nullptr;
    float* y = a.y + z * a.y_z;
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= a.N) return;
    const float* wr = w + (long long)n * a.ldw;
    float acc[MR];
#pragma unroll
    for (int m = 0; m < MR; ++m) acc[m] = 0.f;
    if (VEC) {
#pragma unroll 2
        for (int k = lane * 4; k < a.K; k += 128) {
            const float4 wv = *reinterpret_cast<const float4*>(wr + k);
#pragma unroll
            for (int m = 0; m < MR; ++m)
                if (m < a.M) {
                    float4 xv = *reinterpret_cast<const float4*>(x + (long long)m * a.ldx + k);
                    if (x2) {
                        const float4 t = *reinterpret_cast<const float4*>(x2 + (long long)m * a.ldx + k);
                        xv.x += t.x, xv.y += t.y, xv.z += t.z, xv.w += t.w;
                    }
                    acc[m] = fmaf(xv.x, wv.x, fmaf(xv.y, wv.y, fmaf(xv.z, wv.z, fmaf(xv.w, wv.w, acc[m]))));
                }
        }
    } else {
        for (int k = lane; k < a.K; k += 32) {
            const float wv = wr[k];
#pragma unroll
            for (int m = 0; m < MR; ++m)
                if (m < a.M) {
                    float xv = x[(long long)m * a.ldx + k];
                    if (x2) xv += x2[(long long)m * a.ldx + k];
                    acc[m] = fmaf(xv, wv, acc[m]);
                }
        }
    }
#pragma unroll
    for (int m = 0; m < MR; ++m) {
        const float t = warp_sum(acc[m]);
        if (lane == 0 && m < a.M) {
            float v = t;
            if (b) v += b[n];
            v = apply_act(v, a.act);
            if (r) v += r[(long long)m * a.ldy + n];
            y[(long long)m * a.ldy + n] = v;
        }
    }
}


// Small-M fp32 linear, K split across the 8 warps of a CTA (each CTA owns 8 output columns): every lane issues
// independent 128-bit loads over its K slice, partial sums meet in shared memory.  Used when K is long enough
// that one-warp-per-column would serialise (token-side MLP lin2: K = 2048).  Requires K % 4 == 0, 16-byte rows.
template <int MR>
__global__ void __launch_bounds__(256) linear_gemv_ksplit_kernel(const psam_linear_args a) {
    pdl_prologue();
    __shared__ float part[8][8][MR];  // [warp][column][row]
    const int z = blockIdx.y;
    const float* x = a.x + z * a.x_z;
    const float* x2 = a.x2 ? a.x2 + z * a.x2_z : nullptr;
    const float* w = a.w + z * a.w_z;
    const float* b = a.b ? a.b + z * a.b_z : nullptr;
    const float* r = a.r ? a.r + z * a.r_z : nullptr;
    float* y = a.y + z * a.y_z;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int n0 = blockIdx.x * 8;
    const int kslice = ((a.K / 4 + 7) / 8) * 4;  // per-warp K range, multiple of 4
    const int kbeg = warp * kslice, kend = min(a.K, kbeg + kslice);
    float acc[8][MR];
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int m = 0; m < MR; ++m) acc[c][m] = 0.f;
    for (int k = kbeg + lane * 4; k < kend; k += 128) {
        float4 xv[MR];
#pragma unroll
        for (int m = 0; m < MR; ++m) {
            xv[m] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < a.M) {
                xv[m] = *reinterpret_cast<const float4*>(x + (long long)m * a.ldx + k);
                if (x2) {
                    const float4 t = *reinterpret_cast<const float4*>(x2 + (long long)m * a.ldx + k);
                    xv[m].x += t.x, xv[m].y += t.y, xv[m].z += t.z, xv[m].w += t.w;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (n0 + c < a.N) {
                const float4 wv = *reinterpret_cast<const float4*>(w + (long long)(n0 + c) * a.ldw + k);
#pragma unroll
                for (int m = 0; m < MR; ++m)
                    acc[c][m] = fmaf(xv[m].x, wv.x, fmaf(xv[m].y, wv.y, fmaf(xv[m].z, wv.z, fmaf(xv[m].w, wv.w, acc[c][m]))));
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int m = 0; m < MR; ++m) {
            const float t = warp_sum(acc[c][m]);
            if (lane == 0) part[warp][c][m] = t;
        }
    __syncthreads();
    if (threadIdx.x < 8 * MR) {
        const int c = threadIdx.x / MR, m = threadIdx.x % MR;
        const int n = n0 + c;
        if (n < a.N && m < a.M) {
            float v = 0.f;
#pragma unroll
            for (int wq = 0; wq < 8; ++wq) v += part[wq][c][m];
            if (b) v += b[n];
            v = apply_act(v, a.act);
            if (r) v += r[(long long)m * a.ldy + n];
            y[(long long)m * a.ldy + n] = v;
        }
    }
}

static inline int grid_for(long long work, int per_block, int max_blocks = 132 * 32) {
    long long g = (work + per_block - 1) / per_block;
    if (g < 1) g = 1;
    if (g > max_blocks) g = max_blocks;
    return (int)g;
}

}  // namespace psam

using namespace psam;

extern "C" int psam_layernorm_f32(const psam_ln_args* a, cudaStream_t stream) {
    if (!a || !a->x || !a->gamma || !a->beta || a->rows <= 0 || a->D <= 0 || (!a->y && !a->y_hi)) return PSAM_ERR_ARG;
    if (a->gbias && a->group_rows <= 0) return PSAM_ERR_ARG;
    if (a->y2_hi && !a->post_add) return PSAM_ERR_ARG;
    if (a->D > 4096) return PSAM_ERR_UNSUPPORTED;
    // Short token streams (512 rows of the ViT): a CTA per row finishes sooner (latency policy), a warp per row costs fewer
    // SM-cycles (throughput policy, several clouds in flight): +1.2 % clouds/s at depth 8, +0.3 ms single-stream.
    const bool block_per_row = (a->D > 1024) || (a->D >= 256 && a->rows <= 8192 && a->policy != 1);
    auto al = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
    const bool vec = (a->D % 4 == 0 || a->padded) && a->ldx % 4 == 0 && al(a->x) && al(a->gamma) && al(a->beta) &&
                     (!a->r || (a->ldr % 4 == 0 && al(a->r))) && (!a->gbias || (a->ld_gbias % 4 == 0 && al(a->gbias))) &&
                     (!a->y || (a->ldy % 4 == 0 && al(a->y))) &&
                     (!a->y_hi || (a->ldy_s % 4 == 0 && a->y_plane % 4 == 0 && ((uintptr_t)a->y_hi & 7) == 0)) &&
                     (!a->y2_hi || (a->ldy2_s % 4 == 0 && a->y2_plane % 4 == 0 && ((uintptr_t)a->y2_hi & 7) == 0 &&
                                    a->ld_post % 4 == 0 && al(a->post_add)));
    if (block_per_row && vec) {
        const int nv = ceil_div(a->D, 1024);
        if (nv <= 1) PSAM_CUDA_TRY(psam::launch(layernorm_block_v4_kernel<1>, dim3(a->rows), dim3(256), (size_t)0, stream, *a));
        else if (nv <= 2) PSAM_CUDA_TRY(psam::launch(layernorm_block_v4_kernel<2>, dim3(a->rows), dim3(256), (size_t)0, stream, *a));
        else PSAM_CUDA_TRY(psam::launch(layernorm_block_v4_kernel<4>, dim3(a->rows), dim3(256), (size_t)0, stream, *a));
    } else if (!block_per_row && vec) {
        const int nv = ceil_div(a->D, 128);
        const int blocks = ceil_div(a->rows, 8);
        if (nv <= 1) PSAM_CUDA_TRY(psam::launch(layernorm_warp_v4_kernel<1>, dim3(blocks), dim3(256), (size_t)0, stream, *a));
        else if (nv <= 2) PSAM_CUDA_TRY(psam::launch(layernorm_warp_v4_kernel<2>, dim3(blocks), dim3(256), (size_t)0, stream, *a));
        else if (nv <= 4) PSAM_CUDA_TRY(psam::launch(layernorm_warp_v4_kernel<4>, dim3(blocks), dim3(256), (size_t)0, stream, *a));
        else PSAM_CUDA_TRY(psam::launch(layernorm_warp_v4_kernel<8>, dim3(blocks), dim3(256), (size_t)0, stream, *a));
    } else if (block_per_row) {
        const int vpt = ceil_div(a->D, 256);
        if (vpt <= 1) PSAM_CUDA_TRY(psam::launch(layernorm_block_kernel<1>, dim3(a->rows), dim3(256), (size_t)(0), stream, *a));
        else if (vpt <= 2) PSAM_CUDA_TRY(psam::launch(layernorm_block_kernel<2>, dim3(a->rows), dim3(256), (size_t)(0), stream, *a));
        else if (vpt <= 4) PSAM_CUDA_TRY(psam::launch(layernorm_block_kernel<4>, dim3(a->rows), dim3(256), (size_t)(0), stream, *a));
        else if (vpt <= 8) PSAM_CUDA_TRY(psam::launch(layernorm_block_kernel<8>, dim3(a->rows), dim3(256), (size_t)(0), stream, *a));
        else PSAM_CUDA_TRY(psam::launch(layernorm_block_kernel<16>, dim3(a->rows), dim3(256), (size_t)(0), stream, *a));
    } else {
        const int vpl = ceil_div(a->D, 32);
        const int blocks = ceil_div(a->rows, 8);
        if (vpl <= 4) PSAM_CUDA_TRY(psam::launch(layernorm_warp_kernel<4>, dim3(blocks), dim3(256), (size_t)(0), stream, *a));
        else if (vpl <= 8) PSAM_CUDA_TRY(psam::launch(layernorm_warp_kernel<8>, dim3(blocks), dim3(256), (size_t)(0), stream, *a));
        else if (vpl <= 16) PSAM_CUDA_TRY(psam::launch(layernorm_warp_kernel<16>, dim3(blocks), dim3(256), (size_t)(0), stream, *a));
        else PSAM_CUDA_TRY(psam::launch(layernorm_warp_kernel<32>, dim3(blocks), dim3(256), (size_t)(0), stream, *a));
    }
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_swiglu_ln(const float* gx, long long ld, long long x_off, int rows, int H, const float* gamma,
                              const float* beta, float eps, void* y_hi, long long y_plane, long long ldy_s, long long pitch,
                              cudaStream_t stream) {
    if (!gx || !gamma || !beta || !y_hi || rows <= 0 || H <= 0 || pitch < H) return PSAM_ERR_ARG;
    if (H > 8192) return PSAM_ERR_UNSUPPORTED;
    __nv_bfloat16* yh = (__nv_bfloat16*)y_hi;
    const int vpt = ceil_div(H, 256);
#define PSAM_SWI(V) PSAM_CUDA_TRY(psam::launch(swiglu_ln_kernel<V>, dim3(rows), dim3(256), (size_t)(0), stream, gx, ld, x_off, rows, H, gamma, beta, eps, yh, y_plane, ldy_s, pitch))
    if (vpt <= 2) PSAM_SWI(2);
    else if (vpt <= 4) PSAM_SWI(4);
    else if (vpt <= 8) PSAM_SWI(8);
    else if (vpt <= 12) PSAM_SWI(12);
    else if (vpt <= 16) PSAM_SWI(16);
    else if (vpt <= 24) PSAM_SWI(24);
    else PSAM_SWI(32);
#undef PSAM_SWI
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_small_in_linear(const float* x, int rows, int Cin, const float* W, const float* b, const float* gamma,
                                    const float* beta, float eps, int use_ln, int act, int Cout, void* y_hi,
                                    long long y_plane, long long ldy_s, cudaStream_t stream) {
    if (!x || !W || !y_hi || rows <= 0 || Cin <= 0 || Cin > 16 || Cout % 32 || Cout <= 0 || Cout > 512) return PSAM_ERR_ARG;
    if (use_ln && (!gamma || !beta)) return PSAM_ERR_ARG;
    const size_t smem = (size_t)(Cout * Cin + Cout) * sizeof(float);
    const int blocks = grid_for(rows, 8, 132 * 8);
    __nv_bfloat16* yh = (__nv_bfloat16*)y_hi;
#define PSAM_SIL(CPL)                                                                                                     \
    PSAM_CUDA_TRY(psam::launch(small_in_linear_kernel<CPL>, dim3(blocks), dim3(256), (size_t)(smem), stream, x, rows, Cin, W, b, gamma, beta, eps, use_ln, act, yh, \
                                                                 y_plane, ldy_s))
    switch (Cout / 32) {
        case 1: PSAM_SIL(1); break;
        case 2: PSAM_SIL(2); break;
        case 4: PSAM_SIL(4); break;
        case 8: PSAM_SIL(8); break;
        case 16: PSAM_SIL(16); break;
        default: return PSAM_ERR_UNSUPPORTED;
    }
#undef PSAM_SIL
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_group_max(const float* x, long long ldx, int groups, int K, int D, float* y, long long ldy, void* y_hi,
                              long long y_plane, long long ldy_s, cudaStream_t stream) {
    if (!x || groups <= 0 || K <= 0 || D <= 0 || (!y && !y_hi)) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(group_max_kernel, dim3(groups), dim3(256), (size_t)(0), stream, x, ldx, groups, K, D, y, ldy, (__nv_bfloat16*)y_hi, y_plane, ldy_s));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_softmax_split(const float* s, long long lds, long long rows, int L, float scale, void* p_hi,
                                  long long p_plane, long long ldp, cudaStream_t stream) {
    if (!s || !p_hi || rows <= 0 || L <= 0) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(softmax_split_kernel, dim3((unsigned)ceil_div_ll(rows, 8)), dim3(256), (size_t)(0), stream, s, lds, rows, L, scale, (__nv_bfloat16*)p_hi, p_plane, ldp));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_transpose_split(const void* src_hi, long long src_plane, long long src_ld, long long src_z1,
                                    long long src_z2, void* dst_hi, long long dst_plane, long long dst_ld, long long dst_z1,
                                    long long dst_z2, int rows, int cols, int nz1, int nz2, cudaStream_t stream) {
    if (!src_hi || !dst_hi || rows <= 0 || cols <= 0 || nz1 <= 0 || nz2 <= 0) return PSAM_ERR_ARG;
    dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32), nz1 * nz2);
    PSAM_CUDA_TRY(psam::launch(transpose_split_kernel, dim3(grid), dim3(dim3(32, 8)), (size_t)(0), stream, (const __nv_bfloat16*)src_hi, src_plane, src_ld, src_z1, src_z2,
                                                             (__nv_bfloat16*)dst_hi, dst_plane, dst_ld, dst_z1, dst_z2, rows,
                                                             cols, nz1));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_posenc_f32(const float* coords, long long rows, const float* gauss, int F, const int* labels,
                               const float* emb0, const float* emb1, float* out, int* bad_flag, cudaStream_t stream) {
    if (!coords || !gauss || !out || rows <= 0 || F <= 0) return PSAM_ERR_ARG;
    if (labels && (!emb0 || !emb1)) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(posenc_kernel, dim3((unsigned)rows), dim3(128), (size_t)(0), stream, coords, rows, gauss, F, labels, emb0, emb1, out, bad_flag));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_attention_f32(const float* q, const float* k, const float* v, float* o, int Z, int Lq, int Lk, int H,
                                  int dh, long long ldq, long long ldk, long long ldv, long long ldo, cudaStream_t stream) {
    if (!q || !k || !v || !o || Z <= 0 || Lq <= 0 || Lk <= 0 || H <= 0 || dh <= 0) return PSAM_ERR_ARG;
    const int wpb = 4;
    const long long items = (long long)Z * H * Lq;
    const bool split = items <= 512 && Lk >= 128;  // few queries, many keys: 4 warps per item split the keys
    const int wpi = split ? 4 : 1;
    const size_t smem = (size_t)wpb * (Lk + dh) * sizeof(float) + (size_t)(wpb / wpi) * wpi * (dh + 2) * sizeof(float);
    if (smem > 200 * 1024) return PSAM_ERR_UNSUPPORTED;
    const unsigned grid = (unsigned)ceil_div_ll(items, wpb / wpi);
#define PSAM_ATT(DH)                                                                                                              \
    {                                                                                                                             \
        if (split) {                                                                                                              \
            PSAM_CUDA_TRY(cudaFuncSetAttribute(attention_small_kernel<DH, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            PSAM_CUDA_TRY(psam::launch(attention_small_kernel<DH, 4>, dim3(grid), dim3(wpb * 32), smem, stream, q, k, v, o, Z, Lq, Lk, H, ldq, ldk, ldv, ldo)); \
        } else {                                                                                                                  \
            PSAM_CUDA_TRY(cudaFuncSetAttribute(attention_small_kernel<DH, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
            PSAM_CUDA_TRY(psam::launch(attention_small_kernel<DH, 1>, dim3(grid), dim3(wpb * 32), smem, stream, q, k, v, o, Z, Lq, Lk, H, ldq, ldk, ldv, ldo)); \
        }                                                                                                                         \
    }
    if (dh == 16) PSAM_ATT(16)
    else if (dh == 32) PSAM_ATT(32)
    else if (dh == 64) PSAM_ATT(64)
    else if (dh == 8) PSAM_ATT(8)
    else return PSAM_ERR_UNSUPPORTED;
#undef PSAM_ATT
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_decoder_prepare(const float* iou_token, const float* mask_tokens, int n_mask_tokens, const float* sparse,
                                    int P, const float* pc_emb, const float* dense, long long dense_z, long long dense_g, int Z,
                                    int rep, int G, int D, float* tokens, float* src, cudaStream_t stream) {
    if (!iou_token || !mask_tokens || !pc_emb || !dense || !tokens || !src || Z <= 0 || rep <= 0 || (P > 0 && !sparse)) return PSAM_ERR_ARG;
    const long long total = (long long)Z * (1 + n_mask_tokens + P) * D + (long long)Z * G * D;
    PSAM_CUDA_TRY(psam::launch(decoder_prepare_kernel, dim3(grid_for(total, 256)), dim3(256), (size_t)(0), stream, iou_token, mask_tokens, n_mask_tokens, sparse, P, pc_emb,
                                                                     dense, dense_z, dense_g, Z, rep, G, D, tokens, src));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_interp_ln_gelu(const float* f, int Z, int rep, int G, int D, const long long* idx, const float* w, int N,
                                   const float* gamma, const float* beta, float eps, void* y_hi, long long y_plane,
                                   long long ldy_s, cudaStream_t stream) {
    if (!f || !idx || !w || !gamma || !beta || !y_hi || Z <= 0 || rep <= 0 || D <= 0) return PSAM_ERR_ARG;
    if (D % 128 || D > 1024 || (ldy_s & 3) || (y_plane & 3)) return PSAM_ERR_UNSUPPORTED;
    const dim3 grid(grid_for((long long)Z * N, 8)), block(256);
    __nv_bfloat16* yh = (__nv_bfloat16*)y_hi;
#define PSAM_INT(NV) PSAM_CUDA_TRY(psam::launch(interp_ln_gelu_kernel<NV>, grid, block, (size_t)0, stream, f, Z, rep, G, D, idx, w, N, gamma, beta, eps, yh, y_plane, ldy_s))
    switch (D / 128) {
        case 1: PSAM_INT(1); break;
        case 2: PSAM_INT(2); break;
        case 4: PSAM_INT(4); break;
        case 8: PSAM_INT(8); break;
        default: return PSAM_ERR_UNSUPPORTED;
    }
#undef PSAM_INT
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mask_dot(const float* u, long long ldu, const float* hyper, int Z, int C, int N, int D, float* masks,
                             cudaStream_t stream) {
    if (!u || !hyper || !masks || Z <= 0 || C <= 0 || C > 8 || N <= 0 || D <= 0) return PSAM_ERR_ARG;
    const size_t smem = (size_t)C * D * sizeof(float);
    dim3 grid(grid_for(N, 8, 132 * 8), Z);
    PSAM_CUDA_TRY(psam::launch(mask_dot_kernel, dim3(grid), dim3(256), (size_t)(smem), stream, u, ldu, hyper, Z, C, N, D, masks));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_add_bcast_f32(const float* a, const float* b, long long n, long long chunk, long long rep,
                                  long long b_period, float* out, cudaStream_t stream) {
    if (!a || !b || !out || n <= 0 || b_period <= 0 || chunk <= 0 || rep <= 0) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(add_bcast_kernel, dim3(grid_for(n, 256)), dim3(256), (size_t)(0), stream, a, b, n, chunk, rep, b_period, out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_split_f32(const float* x, long long ld, long long rows, int D, void* y_hi, long long y_plane,
                              long long ldy_s, long long pitch, cudaStream_t stream) {
    if (!x || !y_hi || rows <= 0 || D <= 0 || pitch < D) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(split_f32_kernel, dim3(grid_for(rows * pitch, 256)), dim3(256), (size_t)(0), stream, x, (const float*)nullptr, ld, rows, D, (__nv_bfloat16*)y_hi, y_plane, ldy_s, pitch));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_split_add_f32(const float* x, const float* add, long long ld, long long rows, int D, void* y_hi, long long y_plane,
                                  long long ldy_s, long long pitch, cudaStream_t stream) {
    if (!x || !y_hi || rows <= 0 || D <= 0 || pitch < D) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(split_f32_kernel, dim3(grid_for(rows * pitch, 256)), dim3(256), (size_t)(0), stream, x, add, ld, rows, D, (__nv_bfloat16*)y_hi, y_plane, ldy_s, pitch));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_linear_f32(const psam_linear_args* a, cudaStream_t stream) {
    if (!a || !a->x || !a->w || !a->y || a->M <= 0 || a->N <= 0 || a->K <= 0 || a->Z <= 0) return PSAM_ERR_ARG;
    const bool vec_ok = a->K % 4 == 0 && a->ldx % 4 == 0 && a->ldw % 4 == 0 && ((uintptr_t)a->x % 16) == 0 && ((uintptr_t)a->w % 16) == 0 &&
                        (!a->x2 || (uintptr_t)a->x2 % 16 == 0) && a->x_z % 4 == 0 && a->w_z % 4 == 0 && a->x2_z % 4 == 0;
    if (a->M <= 8 && vec_ok && a->K >= 512) {
        dim3 grid(ceil_div(a->N, 8), a->Z);
        if (a->M <= 1) PSAM_CUDA_TRY(psam::launch(linear_gemv_ksplit_kernel<1>, grid, dim3(256), (size_t)0, stream, *a));
        else if (a->M <= 4) PSAM_CUDA_TRY(psam::launch(linear_gemv_ksplit_kernel<4>, grid, dim3(256), (size_t)0, stream, *a));
        else PSAM_CUDA_TRY(psam::launch(linear_gemv_ksplit_kernel<8>, grid, dim3(256), (size_t)0, stream, *a));
    } else if (a->M <= 16) {
        dim3 grid(ceil_div(a->N, 8), a->Z);
#define PSAM_GEMV(MR)                                                                                              \
    if (vec_ok) PSAM_CUDA_TRY(psam::launch(linear_gemv_kernel<MR, true>, grid, dim3(256), (size_t)0, stream, *a)); \
    else PSAM_CUDA_TRY(psam::launch(linear_gemv_kernel<MR, false>, grid, dim3(256), (size_t)0, stream, *a))
        if (a->M <= 1) { PSAM_GEMV(1); }
        else if (a->M <= 4) { PSAM_GEMV(4); }
        else if (a->M <= 8) { PSAM_GEMV(8); }
        else { PSAM_GEMV(16); }
#undef PSAM_GEMV
    } else if (vec_ok) {
        dim3 grid(ceil_div(a->N, 64), ceil_div(a->M, 32), a->Z);
        PSAM_CUDA_TRY(psam::launch(linear_f32_v4_kernel, dim3(grid), dim3(256), (size_t)(0), stream, *a));
    } else {
        dim3 grid(ceil_div(a->N, 64), ceil_div(a->M, 64), a->Z);
        PSAM_CUDA_TRY(psam::launch(linear_f32_kernel, dim3(grid), dim3(256), (size_t)(0), stream, *a));
    }
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" const char* psam_version(void) { return "psam_b200 0.1 (sm_90a)"; }

extern "C" int psam_voronoi_features_f32(const float* xyz, const float* centers, const long long* nn_idx, const float* feats, int B,
                                         int rep, int N, int G, int C, float* out, void* y_hi, long long y_plane, long long pitch,
                                         cudaStream_t stream) {
    using namespace psam;
    if (!xyz || !centers || !nn_idx || !feats || (!out && !y_hi) || B <= 0 || rep <= 0 || N <= 0 || G <= 0 || C < 0) return PSAM_ERR_ARG;
    if (y_hi && pitch < 4 + C) return PSAM_ERR_ARG;
    const long long total = (long long)B * rep * N;
    const int blocks = (int)min((long long)132 * 16, ceil_div_ll(total, 256));
    PSAM_CUDA_TRY(psam::launch(voronoi_features_kernel, dim3(blocks), dim3(256), (size_t)0, stream, xyz, centers, nn_idx, feats, B * rep, rep, N, G,
                               C, out, (__nv_bfloat16*)y_hi, y_plane, pitch));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_scatter_amax_f32(const float* x, const long long* nn_idx, int B, int N, int G, int D, float* y, cudaStream_t stream) {
    using namespace psam;
    if (!x || !nn_idx || !y || B <= 0 || N <= 0 || G <= 0 || D <= 0 || (D & 3)) return PSAM_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) return PSAM_ERR_ARG;
    const long long n = (long long)B * G * D;
    {
        // -inf fill, scatter, reset of the empty cells
        const int fb = (int)min((long long)132 * 8, ceil_div_ll(n, 256));
        PSAM_CUDA_TRY(psam::launch(fill_f32_kernel, dim3(fb), dim3(256), (size_t)0, stream, y, n, -INFINITY));
        const long long work = (long long)B * N * (D / 4);
        const int sb = (int)min((long long)132 * 16, ceil_div_ll(work, 256));
        PSAM_CUDA_TRY(psam::launch(scatter_amax_kernel, dim3(sb), dim3(256), (size_t)0, stream, x, nn_idx, (long long)B * N, N, G, D, y));
        PSAM_CUDA_TRY(psam::launch(scatter_amax_finish_kernel, dim3(fb), dim3(256), (size_t)0, stream, y, n));
    }
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
