// Encoder fine-tuning: the row-wise backward kernels of a timm EvaBlock (pre-LN attention + SwiGLU / GELU MLP).  The block's
// matrix products (dX = dY W, dW = dY^T X, and the per-(cloud, head) attention products) run on the split-bf16 GEMM; these
// kernels are the elementwise and per-row steps between them.  Semantics in include/psam_b200.h.
//
//   ln_bwd_kernel<false>  LayerNorm backward: one warp per row recomputes mean / rstd with the forward's two-pass
//                         arithmetic, then dx = rstd (dy g - mean(dy g) - x_hat mean(dy g x_hat)) (+ dres); afterwards one
//                         thread per column sums dy x_hat and dy over the CTA's rows in row order (dgamma / dbeta partials).
//   ln_bwd_kernel<true>   the same over the SwiGLU hidden row h = silu(g) * x, read from the interleaved pre-activation
//                         [g0 x0 g1 x1 ...]: writes d[g | x] interleaved (fp32 and split-bf16) and the recomputed LN(h) as
//                         split-bf16 (the fc2 operand of the weight gradient); columns Hd..Hp are written as zeros.
//   gelu_bwd_kernel       da = dh * GELU'(a) (exact-erf derivative), and GELU(a) with the forward's arithmetic.
//   softmax_bwd_kernel    one warp per row: P recomputed from the raw scores as psam_softmax_split does, then
//                         dS = scale P (dP - sum(dP P)) as split-bf16.
// No atomics: every output is a fixed-order function of the inputs.
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {
namespace {

constexpr int ENC_WARPS = 8;
constexpr int MAX_RB = 1024;  // rows per CTA of the LayerNorm backward (their statistics sit in shared memory)

__device__ __forceinline__ float rsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float rmax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// d/dx of the exact-erf GELU: Phi(x) + x phi(x)
__device__ __forceinline__ float gelu_grad_exact(float x) {
    return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * expf(-0.5f * x * x);
}

__device__ __forceinline__ void put_split(__nv_bfloat16* hi, long long plane, long long o, float v) {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[o] = h;
    hi[o + plane] = l;
}

// the LayerNorm input at column c of a row: x itself, or silu(g) * x of the interleaved SwiGLU pre-activation
template <bool SWIGLU>
__device__ __forceinline__ float ln_in(const float* __restrict__ row, int c) {
    if constexpr (SWIGLU) {
        const float2 gx = *reinterpret_cast<const float2*>(row + 2 * c);
        return silu(gx.x) * gx.y;
    } else {
        return row[c];
    }
}

template <bool SWIGLU>
__global__ void __launch_bounds__(ENC_WARPS * 32)
ln_bwd_kernel(const float* __restrict__ x, long long ldx, int M, int D, int Dp, const float* __restrict__ dy, long long ldy,
              const float* __restrict__ gamma, const float* __restrict__ beta, float eps, const float* __restrict__ dres, long long ldr,
              float* __restrict__ out, long long ldo, __nv_bfloat16* __restrict__ out_hi, long long out_plane, long long out_ld,
              __nv_bfloat16* __restrict__ hn_hi, long long hn_plane, long long hn_ld, float* __restrict__ part, int rb) {
    pdl_prologue();
    extern __shared__ float2 s_stat[];  // (mean, rstd) of the CTA's rows
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long r0 = (long long)blockIdx.x * rb, r1 = min((long long)M, r0 + rb);
    const float invD = 1.0f / (float)D;
    for (long long r = r0 + warp; r < r1; r += ENC_WARPS) {
        const float* xr = x + r * ldx;
        const float* dr = dy + r * ldy;
        float s = 0.f;
        for (int c = lane; c < D; c += 32) s += ln_in<SWIGLU>(xr, c);
        const float mean = rsum(s) * invD;
        float q = 0.f;
        for (int c = lane; c < D; c += 32) {
            const float d = ln_in<SWIGLU>(xr, c) - mean;
            q = fmaf(d, d, q);
        }
        const float rstd = rsqrtf(rsum(q) * invD + eps);
        float s1 = 0.f, s2 = 0.f;
        for (int c = lane; c < D; c += 32) {
            const float xh = (ln_in<SWIGLU>(xr, c) - mean) * rstd;
            const float g = dr[c] * gamma[c];
            s1 += g;
            s2 = fmaf(g, xh, s2);
        }
        const float m1 = rsum(s1) * invD, m2 = rsum(s2) * invD;
        for (int c = lane; c < Dp; c += 32) {
            float dh = 0.f, xh = 0.f;
            if (c < D) {
                xh = (ln_in<SWIGLU>(xr, c) - mean) * rstd;
                dh = rstd * (dr[c] * gamma[c] - m1 - xh * m2);
            }
            if constexpr (SWIGLU) {
                float dg = 0.f, dv = 0.f, hn = 0.f;
                if (c < D) {
                    const float2 gx = *reinterpret_cast<const float2*>(xr + 2 * c);
                    const float sg = 1.0f / (1.0f + expf(-gx.x));
                    dg = dh * gx.y * sg * (1.0f + gx.x * (1.0f - sg));  // d silu(g) / dg = sg (1 + g (1 - sg))
                    dv = dh * silu(gx.x);
                    hn = fmaf(xh, gamma[c], beta[c]);
                }
                *reinterpret_cast<float2*>(out + r * ldo + 2 * c) = make_float2(dg, dv);
                if (out_hi) {
                    put_split(out_hi, out_plane, r * out_ld + 2 * c, dg);
                    put_split(out_hi, out_plane, r * out_ld + 2 * c + 1, dv);
                }
                if (hn_hi) put_split(hn_hi, hn_plane, r * hn_ld + c, hn);
            } else {
                const float v = dres ? dh + dres[r * ldr + c] : dh;
                out[r * ldo + c] = v;
                if (out_hi) put_split(out_hi, out_plane, r * out_ld + c, v);
            }
        }
        if (lane == 0) s_stat[r - r0] = make_float2(mean, rstd);
    }
    __syncthreads();
    float* pb = part + (long long)blockIdx.x * 2 * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
        float ag = 0.f, ab = 0.f;
        for (long long r = r0; r < r1; ++r) {
            const float2 st = s_stat[r - r0];
            const float xh = (ln_in<SWIGLU>(x + r * ldx, c) - st.x) * st.y;
            const float d = dy[r * ldy + c];
            ag = fmaf(d, xh, ag);
            ab += d;
        }
        pb[c] = ag;
        pb[D + c] = ab;
    }
}

__global__ void gelu_bwd_kernel(const float* __restrict__ a, long long lda, int M, int n, const float* __restrict__ dh, long long ldd,
                                float* __restrict__ da, long long ldo, __nv_bfloat16* __restrict__ da_hi, long long da_plane, long long da_ld,
                                __nv_bfloat16* __restrict__ h_hi, long long h_plane, long long h_ld) {
    pdl_prologue();
    const long long total = (long long)M * n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / n;
        const int c = (int)(i % n);
        const float av = a[r * lda + c];
        const float g = dh[r * ldd + c] * gelu_grad_exact(av);
        if (da) da[r * ldo + c] = g;
        if (da_hi) put_split(da_hi, da_plane, r * da_ld + c, g);
        if (h_hi) put_split(h_hi, h_plane, r * h_ld + c, gelu_erf(av));
    }
}

__global__ void softmax_bwd_kernel(const float* __restrict__ s, long long lds, const float* __restrict__ dp, long long lddp, long long rows,
                                   int L, float scale, __nv_bfloat16* __restrict__ ds_hi, long long ds_plane, long long ds_ld) {
    pdl_prologue();
    const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* x = s + row * lds;
    const float* g = dp + row * lddp;
    // P exactly as softmax_split_kernel computes it
    float m = -3.4e38f;
    for (int c = lane; c < L; c += 32) m = fmaxf(m, x[c] * scale);
    m = rmax(m);
    float sum = 0.f;
    for (int c = lane; c < L; c += 32) sum += __expf(x[c] * scale - m);
    const float inv = 1.0f / rsum(sum);
    float t = 0.f;
    for (int c = lane; c < L; c += 32) t = fmaf(g[c], __expf(x[c] * scale - m) * inv, t);
    t = rsum(t);
    for (int c = lane; c < L; c += 32) {
        const float p = __expf(x[c] * scale - m) * inv;
        put_split(ds_hi, ds_plane, row * ds_ld + c, scale * p * (g[c] - t));
    }
}

inline unsigned grid_of(long long work, int per_block, long long max_blocks = 132 * 32) {
    long long b = (work + per_block - 1) / per_block;
    return (unsigned)(b < 1 ? 1 : (b > max_blocks ? max_blocks : b));
}

}  // namespace
}  // namespace psam

using namespace psam;

extern "C" int psam_layernorm_backward(const float* x, long long ldx, int M, int D, const float* dy, long long ldy, const float* gamma,
                                       float eps, const float* dres, long long ldr, float* dx, long long ldo, void* dx_hi,
                                       long long dx_plane, long long dx_ld, float* part, int rows_per_block, cudaStream_t stream) {
    if (!x || !dy || !gamma || !dx || !part || M <= 0 || D <= 0 || ldx < D || ldy < D || ldo < D || (dres && ldr < D) ||
        (dx_hi && (dx_ld < D || dx_plane < 0)) || rows_per_block <= 0 || rows_per_block > MAX_RB || !(eps >= 0.0f))
        return PSAM_ERR_ARG;
    const unsigned blocks = (unsigned)((M + rows_per_block - 1) / rows_per_block);
    PSAM_CUDA_TRY(psam::launch(ln_bwd_kernel<false>, dim3(blocks), dim3(ENC_WARPS * 32), (size_t)rows_per_block * sizeof(float2), stream,
                               x, ldx, M, D, D, dy, ldy, gamma, (const float*)nullptr, eps, dres, ldr, dx, ldo, (__nv_bfloat16*)dx_hi,
                               dx_plane, dx_ld, (__nv_bfloat16*)nullptr, 0LL, 0LL, part, rows_per_block));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_swiglu_ln_backward(const float* a, long long lda, int M, int Hd, int Hp, const float* dhn, long long ldd,
                                       const float* gamma, const float* beta, float eps, float* da, long long ldo, void* da_hi,
                                       long long da_plane, long long da_ld, void* hn_hi, long long hn_plane, long long hn_ld, float* part,
                                       int rows_per_block, cudaStream_t stream) {
    if (!a || !dhn || !gamma || !beta || !da || !part || M <= 0 || Hd <= 0 || Hp < Hd || lda < 2LL * Hp || lda % 2 || ldd < Hd ||
        ldo < 2LL * Hp || ldo % 2 || (da_hi && (da_ld < 2LL * Hp || da_plane < 0)) || (hn_hi && (hn_ld < Hp || hn_plane < 0)) ||
        rows_per_block <= 0 || rows_per_block > MAX_RB || !(eps >= 0.0f))
        return PSAM_ERR_ARG;
    const unsigned blocks = (unsigned)((M + rows_per_block - 1) / rows_per_block);
    PSAM_CUDA_TRY(psam::launch(ln_bwd_kernel<true>, dim3(blocks), dim3(ENC_WARPS * 32), (size_t)rows_per_block * sizeof(float2), stream,
                               a, lda, M, Hd, Hp, dhn, ldd, gamma, beta, eps, (const float*)nullptr, 0LL, da, ldo, (__nv_bfloat16*)da_hi,
                               da_plane, da_ld, (__nv_bfloat16*)hn_hi, hn_plane, hn_ld, part, rows_per_block));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_gelu_backward(const float* a, long long lda, int M, int n, const float* dh, long long ldd, float* da, long long ldo,
                                  void* da_hi, long long da_plane, long long da_ld, void* h_hi, long long h_plane, long long h_ld,
                                  cudaStream_t stream) {
    if (!a || !dh || (!da && !da_hi && !h_hi) || M <= 0 || n <= 0 || lda < n || ldd < n || (da && ldo < n) ||
        (da_hi && (da_ld < n || da_plane < 0)) || (h_hi && (h_ld < n || h_plane < 0)))
        return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(gelu_bwd_kernel, dim3(grid_of((long long)M * n, 256)), dim3(256), (size_t)0, stream, a, lda, M, n, dh, ldd,
                               da, ldo, (__nv_bfloat16*)da_hi, da_plane, da_ld, (__nv_bfloat16*)h_hi, h_plane, h_ld));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_softmax_backward(const float* s, long long lds, const float* dp, long long lddp, long long rows, int L, float scale,
                                     void* ds_hi, long long ds_plane, long long ds_ld, cudaStream_t stream) {
    if (!s || !dp || !ds_hi || rows <= 0 || L <= 0 || lds < L || lddp < L || ds_ld < L || ds_plane < 0 || (rows + 7) / 8 > 2147483647LL)
        return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(softmax_bwd_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), (size_t)0, stream, s, lds, dp, lddp, rows,
                               L, scale, (__nv_bfloat16*)ds_hi, ds_plane, ds_ld));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
