// Decoder fine-tuning: the reference's mask loss (sigmoid focal + dice, loss.py:58-77) with its hard IoU, and the backward
// of the per-point mask head (output_upscaling[1..4] after the 3-NN interpolation, and the hyper-network product,
// mask_decoder.py:146-176).  The semantics are stated in include/psam_b200.h.
//
//   mask_loss_stats_kernel     one CTA per (row z, mask c): sums of focal, p t, p^2, t (fp64 per element and accumulator)
//                              and the integer intersection / union of (logit > 0, gt).  Fixed reduction tree.
//   mask_loss_grad_kernel      one thread per logit: d loss[z, c] / d logit scaled by the upstream gradient; rows whose
//                              upstream gradient is zero (the masks the criterion did not select) are written as zeros.
//   interp_inverse_kernel      one CTA per cloud: counting sort of the 3 N interpolation entries by patch, stable (entry
//                              order within a patch is ascending n * 3 + k), so the interpolation backward is a gather.
//   head_dp_kernel             one CTA per (chunk of points, row z), one thread per column: dp = GELU'(p) sum_c dm hyper_c
//                              as split-bf16, and per-chunk partial sums of dhyper and db3.
//   interp_ln_gelu_bwd_kernel  one warp per point (as the forward): recomputes the interpolation and LayerNorm, back through
//                              GELU and LayerNorm in place; per-CTA partial sums of dgamma / dbeta (fixed warp order).
//   interp_bwd_kernel          one warp per (row z, patch g): df[z, g] = sum over the patch's entries of w * dv, in the
//                              inverse index's order.
//   sum_partials_kernel        out = sum over s of part[s] in order s = 0, 1, ... (fp64 accumulator).
// No float atomics anywhere: every result is bitwise reproducible run to run.
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {
namespace {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double wsum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int wsum_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// d/dx of the exact-erf GELU: Phi(x) + x phi(x)
__device__ __forceinline__ float gelu_grad(float x) {
    return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * expf(-0.5f * x * x);
}

struct LogitTerms {
    double p, q, ce, s;  // sigmoid(x), 1 - p_t, BCE with logits, p (1 - p)
};

// Stable forms: BCE = max(x, 0) - x t + log1p(exp(-|x|)); sigmoid(+-x) from e = exp(-|x|) without 1 - p cancellation, so
// (1 - p_t)^2 stays exact in relative terms for |x| up to 100 and beyond.
__device__ __forceinline__ LogitTerms logit_terms(float xf, int t) {
    const double x = (double)xf;
    const double e = exp(-fabs(x));
    const double r = 1.0 / (1.0 + e);
    const double sp = x >= 0.0 ? r : e * r;  // sigmoid(x)
    const double sn = x >= 0.0 ? e * r : r;  // sigmoid(-x) = 1 - sigmoid(x)
    LogitTerms o;
    o.p = sp;
    o.q = t ? sn : sp;
    o.ce = fmax(x, 0.0) - x * (double)t + log1p(e);
    o.s = sp * sn;
    return o;
}

constexpr int LOSS_THREADS = 256;

__global__ void __launch_bounds__(LOSS_THREADS) mask_loss_stats_kernel(const float* __restrict__ logits, const unsigned char* __restrict__ gt,
                                                                       int C, int N, float* __restrict__ stats, int* __restrict__ counts) {
    pdl_prologue();
    const int zc = blockIdx.x, z = zc / C;
    const float* x = logits + (long long)zc * N;
    const unsigned char* g = gt + (long long)z * N;
    double f = 0.0, pt = 0.0, pp = 0.0;
    int ts = 0, in = 0, un = 0;
    for (int n = threadIdx.x; n < N; n += LOSS_THREADS) {
        const float xv = x[n];
        const int t = g[n] != 0;
        const LogitTerms a = logit_terms(xv, t);
        f += a.ce * a.q * a.q;
        pt += a.p * t;
        pp += a.p * a.p;
        ts += t;
        const int pr = xv > 0.0f;
        in += pr & t;
        un += pr | t;
    }
    __shared__ double sd[3][LOSS_THREADS / 32];
    __shared__ int si[3][LOSS_THREADS / 32];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    f = wsum_d(f), pt = wsum_d(pt), pp = wsum_d(pp);
    ts = wsum_i(ts), in = wsum_i(in), un = wsum_i(un);
    if (l == 0) sd[0][w] = f, sd[1][w] = pt, sd[2][w] = pp, si[0][w] = ts, si[1][w] = in, si[2][w] = un;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0, c = 0.0;
        int d = 0, e = 0, h = 0;
        for (int i = 0; i < LOSS_THREADS / 32; ++i) a += sd[0][i], b += sd[1][i], c += sd[2][i], d += si[0][i], e += si[1][i], h += si[2][i];
        stats[zc * 4 + 0] = (float)a;
        stats[zc * 4 + 1] = (float)b;
        stats[zc * 4 + 2] = (float)c;
        stats[zc * 4 + 3] = (float)d;
        counts[zc * 2 + 0] = e;
        counts[zc * 2 + 1] = h;
    }
}

__global__ void mask_loss_grad_kernel(const float* __restrict__ logits, const unsigned char* __restrict__ gt, int C, int N,
                                      const float* __restrict__ stats, const float* __restrict__ dloss, float* __restrict__ dlogits) {
    pdl_prologue();
    const int zc = blockIdx.y, z = zc / C;
    const float up = dloss[zc];
    const float* st = stats + zc * 4;
    const double A = 2.0 * st[1] + 1e-3, Bd = (double)st[2] + st[3] + 1e-3;
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) {
        const long long o = (long long)zc * N + n;
        if (up == 0.0f) {
            dlogits[o] = 0.0f;
            continue;
        }
        const int t = gt[(long long)z * N + n] != 0;
        const LogitTerms a = logit_terms(logits[o], t);
        // focal: ce q^2 with d ce = p - t and d q = (t ? -1 : 1) p (1 - p)
        const double dq = t ? -a.s : a.s;
        const double dfocal = (a.p - (double)t) * a.q * a.q + 2.0 * a.ce * a.q * dq;
        // 2 dice = 2 (1 - A / Bd): d / dp = 2 (2 A p / Bd^2 - 2 t / Bd)
        const double ddice = 2.0 * (2.0 * A * a.p / (Bd * Bd) - 2.0 * t / Bd) * a.s;
        dlogits[o] = (float)((double)up * (dfocal / (double)N + ddice));
    }
}

constexpr int INV_THREADS = 1024;

__global__ void __launch_bounds__(INV_THREADS) interp_inverse_kernel(const long long* __restrict__ idx, int N, int G,
                                                                     int* __restrict__ offsets, int* __restrict__ entries) {
    pdl_prologue();
    extern __shared__ int s_cnt[];  // [G] counts, then cursors
    __shared__ int s_warp[INV_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long* ib = idx + (long long)b * 3 * N;
    const int E = 3 * N;
    for (int g = tid; g < G; g += INV_THREADS) s_cnt[g] = 0;
    __syncthreads();
    for (int e = tid; e < E; e += INV_THREADS) {
        const long long g = ib[e];
        if (g >= 0 && g < G) atomicAdd(&s_cnt[g], 1);  // integer counts: order-independent
    }
    __syncthreads();
    // exclusive scan: thread t owns the contiguous segment [t * per, (t + 1) * per)
    const int per = (G + INV_THREADS - 1) / INV_THREADS;
    const int g0 = min(G, tid * per), g1 = min(G, g0 + per);
    int seg = 0;
    for (int g = g0; g < g1; ++g) seg += s_cnt[g];
    int incl = seg;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int v = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += y;
        }
        s_warp[lane] = v;
    }
    __syncthreads();
    int run = incl - seg + (warp ? s_warp[warp - 1] : 0);
    int* off = offsets + (long long)b * (G + 1);
    for (int g = g0; g < g1; ++g) {
        const int c = s_cnt[g];
        off[g] = run;
        s_cnt[g] = run;  // becomes the cursor
        run += c;
    }
    if (tid == INV_THREADS - 1) off[G] = s_warp[31];
    __syncthreads();
    // stable fill: chunks of INV_THREADS entries, warps in order, lanes of one patch ranked by lane
    int* eb = entries + (long long)b * E;
    for (int base = 0; base < E; base += INV_THREADS) {
        const int e = base + tid;
        long long gl = e < E ? ib[e] : -1;
        const int g = (gl >= 0 && gl < G) ? (int)gl : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, g);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        const int leader = __ffs(peers) - 1;
        for (int w = 0; w < INV_THREADS / 32; ++w) {
            if (warp == w) {
                const int at = g >= 0 ? s_cnt[g] : 0;
                __syncwarp();
                if (g >= 0) {
                    eb[at + rank] = e;
                    if (lane == leader) s_cnt[g] = at + __popc(peers);
                }
            }
            __syncthreads();
        }
    }
}

constexpr int HEAD_RB = 128;  // points per CTA of head_dp_kernel

__global__ void head_dp_kernel(const float* __restrict__ p, const float* __restrict__ dm, const float* __restrict__ hyper, int C, int N,
                               int D, __nv_bfloat16* __restrict__ dp_hi, long long dp_plane, long long ldp, float* __restrict__ part_h,
                               float* __restrict__ part_b) {
    pdl_prologue();
    __shared__ float s_dm[8][HEAD_RB];
    const int z = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x, d = threadIdx.x;
    const int n0 = chunk * HEAD_RB, cnt = min(HEAD_RB, N - n0);
    for (int i = threadIdx.x; i < C * HEAD_RB; i += blockDim.x) {
        const int c = i / HEAD_RB, j = i % HEAD_RB;
        s_dm[c][j] = j < cnt ? dm[((long long)z * C + c) * N + n0 + j] : 0.0f;
    }
    __syncthreads();
    float h[8], acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        h[c] = c < C ? hyper[((long long)z * C + c) * D + d] : 0.0f;
        acc[c] = 0.0f;
    }
    float accb = 0.0f;
    for (int j = 0; j < cnt; ++j) {
        const long long row = (long long)z * N + n0 + j;
        const float pv = p[row * D + d];
        float gs = 0.0f;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (c < C) gs = fmaf(s_dm[c][j], h[c], gs);
        const float u2 = gelu_erf(pv);
        const float dpv = gs * gelu_grad(pv);
        __nv_bfloat16 hi, lo;
        split_bf16(dpv, hi, lo);
        dp_hi[row * ldp + d] = hi;
        dp_hi[row * ldp + d + dp_plane] = lo;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (c < C) acc[c] = fmaf(s_dm[c][j], u2, acc[c]);
        accb += dpv;
    }
    const long long blk = (long long)z * nchunk + chunk;
    for (int c = 0; c < C; ++c) part_h[(blk * C + c) * D + d] = acc[c];
    part_b[blk * D + d] = accb;
}

constexpr int LNB_WARPS = 8;

template <int NV>
__global__ void __launch_bounds__(LNB_WARPS * 32)
interp_ln_gelu_bwd_kernel(const float* __restrict__ f, int Z, int rep, int G, int D, const long long* __restrict__ idx,
                          const float* __restrict__ w, int N, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                          float* __restrict__ du, float* __restrict__ part, int rb) {
    pdl_prologue();
    __shared__ float4 s_red[LNB_WARPS][2][NV * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long total = (long long)Z * N;
    const long long r0 = (long long)blockIdx.x * rb, r1 = min(total, r0 + rb);
    float4 ag[NV], ab[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) ag[i] = ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long pt = r0 + warp; pt < r1; pt += LNB_WARPS) {
        const int z = (int)(pt / N), n = (int)(pt % N);
        // the forward's arithmetic (interp_ln_gelu_kernel), value for value
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
        const float mean = wsum(s) / (float)D;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const float d0 = v[i].x - mean, d1 = v[i].y - mean, d2 = v[i].z - mean, d3 = v[i].w - mean;
            q += (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3);
        }
        const float rstd = rsqrtf(wsum(q) / (float)D + eps);
        // v becomes x_hat, and dx_hat = dh * gamma is kept in dx
        float4 dx[NV];
        float s1 = 0.f, s2 = 0.f;
        float* dur = du + pt * D;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = 4 * lane + 128 * i;
            const float4 g = *reinterpret_cast<const float4*>(gamma + c), b = *reinterpret_cast<const float4*>(beta + c);
            const float4 gu = *reinterpret_cast<const float4*>(dur + c);
            float4 xh, dh;
            xh.x = (v[i].x - mean) * rstd; xh.y = (v[i].y - mean) * rstd; xh.z = (v[i].z - mean) * rstd; xh.w = (v[i].w - mean) * rstd;
            dh.x = gu.x * gelu_grad(xh.x * g.x + b.x);
            dh.y = gu.y * gelu_grad(xh.y * g.y + b.y);
            dh.z = gu.z * gelu_grad(xh.z * g.z + b.z);
            dh.w = gu.w * gelu_grad(xh.w * g.w + b.w);
            ag[i].x = fmaf(dh.x, xh.x, ag[i].x); ag[i].y = fmaf(dh.y, xh.y, ag[i].y);
            ag[i].z = fmaf(dh.z, xh.z, ag[i].z); ag[i].w = fmaf(dh.w, xh.w, ag[i].w);
            ab[i].x += dh.x; ab[i].y += dh.y; ab[i].z += dh.z; ab[i].w += dh.w;
            dx[i] = make_float4(dh.x * g.x, dh.y * g.y, dh.z * g.z, dh.w * g.w);
            v[i] = xh;
            s1 += (dx[i].x + dx[i].y) + (dx[i].z + dx[i].w);
            s2 += (dx[i].x * xh.x + dx[i].y * xh.y) + (dx[i].z * xh.z + dx[i].w * xh.w);
        }
        const float m1 = wsum(s1) / (float)D, m2 = wsum(s2) / (float)D;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const int c = 4 * lane + 128 * i;
            float4 o;
            o.x = rstd * (dx[i].x - m1 - v[i].x * m2);
            o.y = rstd * (dx[i].y - m1 - v[i].y * m2);
            o.z = rstd * (dx[i].z - m1 - v[i].z * m2);
            o.w = rstd * (dx[i].w - m1 - v[i].w * m2);
            *reinterpret_cast<float4*>(dur + c) = o;
        }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        s_red[warp][0][i * 32 + lane] = ag[i];
        s_red[warp][1][i * 32 + lane] = ab[i];
    }
    __syncthreads();
    // column c = 4 * lane + 128 * i sits at float index 4 * (i * 32 + lane) + component
    float* out = part + (long long)blockIdx.x * 2 * D;
    for (int k = threadIdx.x; k < 2 * D; k += blockDim.x) {
        const int which = k / D, c = k % D;
        const int slot = (c % 128) / 4 + 32 * (c / 128), comp = c & 3;
        float acc = 0.f;
        for (int ww = 0; ww < LNB_WARPS; ++ww) acc += reinterpret_cast<const float*>(&s_red[ww][which][slot])[comp];
        out[k] = acc;
    }
}

template <int NV>
__global__ void __launch_bounds__(256)
interp_bwd_kernel(const float* __restrict__ dv, int Z, int rep, int G, int D, const int* __restrict__ offsets,
                  const int* __restrict__ entries, const float* __restrict__ w, int N, float* __restrict__ df) {
    pdl_prologue();
    const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * wpb + (threadIdx.x >> 5);
    if (item >= (long long)Z * G) return;
    const int z = (int)(item / G), g = (int)(item % G), b = z / rep;
    const int* off = offsets + (long long)b * (G + 1);
    const int* ent = entries + (long long)b * 3 * N;
    const float* wb = w + (long long)b * 3 * N;
    float4 acc[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int beg = off[g], end = off[g + 1];
    for (int j = beg; j < end; ++j) {
        const int e = ent[j];
        const float wt = wb[e];
        const float* row = dv + ((long long)z * N + e / 3) * D;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            const float4 x = *reinterpret_cast<const float4*>(row + 4 * lane + 128 * i);
            acc[i].x = fmaf(wt, x.x, acc[i].x); acc[i].y = fmaf(wt, x.y, acc[i].y);
            acc[i].z = fmaf(wt, x.z, acc[i].z); acc[i].w = fmaf(wt, x.w, acc[i].w);
        }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) *reinterpret_cast<float4*>(df + item * D + 4 * lane + 128 * i) = acc[i];
}

__global__ void sum_partials_kernel(const float* __restrict__ part, int nb, int S, long long n, float* __restrict__ out) {
    pdl_prologue();
    const long long total = (long long)nb * n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / n, k = i % n;
        const float* p = part + b * S * n + k;
        double acc = 0.0;
        for (int s = 0; s < S; ++s) acc += (double)p[(long long)s * n];
        out[i] = (float)acc;
    }
}

inline unsigned blocks_for(long long work, int per_block, long long max_blocks = 132 * 32) {
    long long b = (work + per_block - 1) / per_block;
    if (b < 1) b = 1;
    if (b > max_blocks) b = max_blocks;
    return (unsigned)b;
}

}  // namespace
}  // namespace psam

using namespace psam;

extern "C" int psam_mask_loss_stats(const float* logits, const unsigned char* gt, int Z, int C, int N, float* stats, int* counts,
                                    cudaStream_t stream) {
    if (!logits || !gt || !stats || !counts || Z <= 0 || C <= 0 || N <= 0 || (long long)Z * C > 2147483647LL) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(mask_loss_stats_kernel, dim3((unsigned)(Z * C)), dim3(LOSS_THREADS), (size_t)0, stream, logits, gt, C, N,
                               stats, counts));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_mask_loss_grad(const float* logits, const unsigned char* gt, int Z, int C, int N, const float* stats,
                                   const float* dloss, float* dlogits, cudaStream_t stream) {
    if (!logits || !gt || !stats || !dloss || !dlogits || Z <= 0 || C <= 0 || N <= 0 || (long long)Z * C > 65535) return PSAM_ERR_ARG;
    const dim3 grid(blocks_for(N, 256, 64), (unsigned)(Z * C));
    PSAM_CUDA_TRY(psam::launch(mask_loss_grad_kernel, grid, dim3(256), (size_t)0, stream, logits, gt, C, N, stats, dloss, dlogits));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_interp_inverse(const long long* idx, int B, int N, int G, int* offsets, int* entries, cudaStream_t stream) {
    if (!idx || !offsets || !entries || B <= 0 || N <= 0 || G <= 0 || G > 8192 || N > 700000000) return PSAM_ERR_ARG;
    const size_t smem = (size_t)G * sizeof(int);
    PSAM_CUDA_TRY(cudaFuncSetAttribute(interp_inverse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PSAM_CUDA_TRY(psam::launch(interp_inverse_kernel, dim3((unsigned)B), dim3(INV_THREADS), smem, stream, idx, N, G, offsets, entries));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_head_dp(const float* p, const float* dm, const float* hyper, int Z, int C, int N, int D, void* dp_hi,
                            long long dp_plane, long long ldp_s, float* part_hyper, float* part_b3, cudaStream_t stream) {
    if (!p || !dm || !hyper || !dp_hi || !part_hyper || !part_b3 || Z <= 0 || Z > 65535 || C <= 0 || C > 8 || N <= 0 || D <= 0 ||
        D > 1024 || D % 32 || ldp_s < D || dp_plane < 0)
        return PSAM_ERR_ARG;
    const dim3 grid((unsigned)((N + HEAD_RB - 1) / HEAD_RB), (unsigned)Z);
    PSAM_CUDA_TRY(psam::launch(head_dp_kernel, grid, dim3((unsigned)D), (size_t)0, stream, p, dm, hyper, C, N, D, (__nv_bfloat16*)dp_hi,
                               dp_plane, ldp_s, part_hyper, part_b3));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_head_dp_chunks(int N) { return N > 0 ? (N + HEAD_RB - 1) / HEAD_RB : 0; }

extern "C" int psam_interp_ln_gelu_backward(const float* f, int Z, int rep, int G, int D, const long long* idx, const float* w, int N,
                                            const float* gamma, const float* beta, float eps, float* du, float* part, int rows_per_block,
                                            cudaStream_t stream) {
    if (!f || !idx || !w || !gamma || !beta || !du || !part || Z <= 0 || rep <= 0 || G <= 0 || N <= 0 || D <= 0 || rows_per_block <= 0)
        return PSAM_ERR_ARG;
    if (D % 128 || D > 512) return PSAM_ERR_UNSUPPORTED;
    const long long blocks = ((long long)Z * N + rows_per_block - 1) / rows_per_block;
    if (blocks > 2147483647LL) return PSAM_ERR_ARG;
#define PSAM_LNB(NV) PSAM_CUDA_TRY(psam::launch(interp_ln_gelu_bwd_kernel<NV>, dim3((unsigned)blocks), dim3(LNB_WARPS * 32), (size_t)0, stream, \
                                                f, Z, rep, G, D, idx, w, N, gamma, beta, eps, du, part, rows_per_block))
    switch (D / 128) {
        case 1: PSAM_LNB(1); break;
        case 2: PSAM_LNB(2); break;
        case 4: PSAM_LNB(4); break;
        default: return PSAM_ERR_UNSUPPORTED;
    }
#undef PSAM_LNB
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_interp_backward(const float* dv, int Z, int rep, int G, int D, const int* offsets, const int* entries, const float* w,
                                    int N, float* df, cudaStream_t stream) {
    if (!dv || !offsets || !entries || !w || !df || Z <= 0 || rep <= 0 || G <= 0 || N <= 0 || D <= 0) return PSAM_ERR_ARG;
    if (D % 128 || D > 1024) return PSAM_ERR_UNSUPPORTED;
    const unsigned grid = (unsigned)(((long long)Z * G + 7) / 8);
#define PSAM_IB(NV) PSAM_CUDA_TRY(psam::launch(interp_bwd_kernel<NV>, dim3(grid), dim3(256), (size_t)0, stream, dv, Z, rep, G, D, offsets, \
                                               entries, w, N, df))
    switch (D / 128) {
        case 1: PSAM_IB(1); break;
        case 2: PSAM_IB(2); break;
        case 4: PSAM_IB(4); break;
        case 8: PSAM_IB(8); break;
        default: return PSAM_ERR_UNSUPPORTED;
    }
#undef PSAM_IB
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" int psam_sum_partials(const float* part, int nb, int S, long long n, float* out, cudaStream_t stream) {
    if (!part || !out || nb <= 0 || S <= 0 || n <= 0) return PSAM_ERR_ARG;
    PSAM_CUDA_TRY(psam::launch(sum_partials_kernel, dim3(blocks_for((long long)nb * n, 256)), dim3(256), (size_t)0, stream, part, nb, S, n, out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
