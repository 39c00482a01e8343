// Tensor-core GEMM for sm_90a: C[M,N] = A[M,K] * W[N,K]^T (+bias, activation, residual).
//
// Replaces every nn.Linear / bmm of the reference hot path that has enough rows to fill a 128-row
// MMA tile (PatchEncoder common.py:486-497, patch_proj/pos_embed/out_proj pc_encoder.py:99-116, the
// timm EVA block linears and attention products, output_upscaling mask_decoder.py:53-59).
//
// Numerics ("split-bf16"): the reference runs these contractions in fp32.  Operands are stored as two
// bf16 planes, x = hi + lo (relative residual <= 2^-17), and the product is accumulated in fp32 registers as
//        A_hi*W_hi + A_lo*W_hi + A_hi*W_lo                                   (passes = 3)
// which keeps ~16 mantissa bits per operand: end-to-end logit error ~2e-5 vs fp32, inside the
// 1e-3 abs / 1e-2 rel parity bound (a single bf16 pass, passes = 1, is ~1e-2 and fails it).
//
// Structure (one 128 x BN output tile per CTA, optional split-K over blockIdx.z):
//   warp 8   : TMA producer - 5-D tensor maps (k, row, plane, batch1, batch2), 128B-swizzled 3-D boxes of
//              64 bf16 x {128|BN} rows x {hi,lo}, 2-4 stage mbarrier ring
//   warps 0-7: two consumer warpgroups (rows 0-63 / 64-127 of the tile), wgmma m64nBNk16 from shared memory
//              into fp32 registers; one wgmma group stays in flight while the previous stage is released.
//              Epilogue: the accumulators are staged as an fp32 tile in the (then idle) stage memory, and each
//              warp takes 32-row x 32-column chunks of it, so every global access is a contiguous row segment:
//              bias/activation/residual, fp32 and/or split-bf16 stores (red.add for split-K)
// The output-tile width BN is 64, 128 or 256 (the wgmma N), chosen so the tile count fills the 132 SMs of an
// H100 in as few waves as possible.
#include <stdlib.h>

#include <cstdlib>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 288;  // two consumer warpgroups + one TMA warp
constexpr int GEMM_A_TILE = GEMM_BM * GEMM_BK * 2;  // bytes per plane of an A stage
// psam_gemm_out.variant bits.  GV_SCALAR_EPI forces the scalar epilogue; the other bits select kernels of other
// architectures and are accepted without effect, so callers built for them keep working.
constexpr int GV_SCALAR_EPI = 0x4;

struct GemmEpilogue {
    float* out_f32;            // may be null
    long long ldo;             // row stride of out_f32 / resid (elements)
    long long out_b1, out_b2;  // batch strides of out_f32 / resid
    __nv_bfloat16* out_hi;     // may be null; lo plane at out_hi + out_plane
    long long out_plane, ldo_s, outs_b1, outs_b2;
    const float* bias;   // [N] or null
    const float* resid;  // same geometry as out_f32, may alias it; null = none
    float alpha;         // scale applied to the accumulator before bias
    int act;
    int accumulate;  // 1: out_f32 += result via red.global.add (required for split_k > 1)
    int swiglu;      // 1: columns are (gate, value) pairs; out_f32[:, c/2] = silu(gate) * value
    float* gmax;     // optional: gmax[(row / group_rows) * ld_gmax + col] = max over the rows of a group (atomic, pre-filled with -inf)
    long long ld_gmax;
    int group_rows;  // multiple of 32
    const float* rd_w;   // optional fused row-dot: rd_out[z, c, n] += sum_col act(x[z*rd_rows + n, col]) * rd_w[z, c, col]
    float* rd_out;       // (pre-zeroed; the hyper-network mask product of the decoder), rd_rows % 32 == 0, rd_c <= 8
    int rd_rows, rd_c;
    float* stats_out;        // SwiGLU + split output: stats_out[row] += (sum, sum of squares) of the fp32 products of the row
    const float* ln_stats;   // LayerNorm folded into THIS GEMM: A holds the un-normalised rows, W is pre-scaled by gamma;
    const float* ln_c;       //   out = rstd * (acc - mean * ln_c[n]) + bias[n]  (bias = W beta + b), stats = (sum, sum sq) per row
    float ln_inv_h, ln_eps;
    int vec4;  // host-verified: every output / bias / residual row is 16-byte (split planes: 8-byte) addressable in 4-column steps
};

struct GemmShape {
    int M, N, K;
    int nb1, nb2;  // batch extents (blockIdx.z = ((b2 * nb1) + b1) * split_k + split)
    int split_k;
    int passes;  // 1 or 3
    int bn;      // output-tile width (64, 128 or 256)
};

template <int BN, int STAGES>
struct GemmSmem {
    static constexpr int B_TILE = BN * GEMM_BK * 2;  // bytes per plane
    static constexpr int STAGE = 2 * GEMM_A_TILE + 2 * B_TILE;
    static constexpr int PITCH = BN + 4;              // floats per row of the staged output tile
    static constexpr int EPI = GEMM_BM * PITCH * 4;   // the staged tile reuses the stage memory
    static constexpr int TOTAL = (STAGES * STAGE > EPI ? STAGES * STAGE : EPI) + 1024;  // + alignment slack
    static_assert(TOTAL <= 232448, "shared memory of one H100 SM");
};

// ---- epilogue row loops, specialised at compile time (runtime flags inside the loop cost ~10 uniform
//      branches per row and made the epilogue the slowest part of small-K GEMMs) -------------------------
template <int ACT, bool RES, bool ACC>
__device__ __forceinline__ void epi_rows_f32(const float* __restrict__ stg, int pitch, int lane, int row0, int M, int col,
                                             bool col_ok, float alpha, float bv, float* out, const float* res, long long ldo) {
    if (!col_ok) return;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) {
        const int row = row0 + r;
        if (row < M) {
            float x = fmaf(stg[r * pitch + lane], alpha, bv);
            if (RES) x += res[(long long)row * ldo + col];
            x = apply_act(x, ACT);
            if (ACC) atomicAdd(out + (long long)row * ldo + col, x);
            else out[(long long)row * ldo + col] = x;
        }
    }
}


// SwiGLU epilogue: W rows are interleaved (2i = gate_i, 2i+1 = value_i) so adjacent lanes hold a pair;
// out[row, col/2] = silu(acc_g + b_g) * (acc_x + b_x).  Halves the fc1 output traffic and removes the
// activation from the LayerNorm kernel that follows (timm SwiGLU: x = act(fc1_g(x)) * fc1_x(x)).
__device__ __forceinline__ void epi_rows_swiglu(const float* __restrict__ stg, int pitch, int lane, int row0, int M, int col,
                                                bool col_ok, float alpha, float bv, float* out, long long ldo) {
#pragma unroll 8
    for (int r = 0; r < 32; ++r) {
        const int row = row0 + r;
        const float x = fmaf(stg[r * pitch + lane], alpha, bv);
        const float other = __shfl_xor_sync(0xffffffffu, x, 1);
        if (row < M && col_ok && (lane & 1) == 0) out[(long long)row * ldo + (col >> 1)] = __fdividef(x, 1.0f + __expf(-x)) * other;
    }
}

template <int ACT, bool RES, bool F32>
__device__ __forceinline__ void epi_rows_split(const float* __restrict__ stg, int pitch, int lane, int row0, int M, int N, int col0,
                                               float alpha, const float* bias, float* out, const float* res, long long ldo,
                                               __nv_bfloat16* ohi, long long out_plane, long long ldo_s, bool vec_align) {
    // lanes 0..15 take row r, lanes 16..31 row r+1, two adjacent columns each
    const int half = lane >> 4, cpair = (lane & 15) * 2;
    const int c0 = col0 + cpair;
    const bool ok0 = c0 < N, ok1 = c0 + 1 < N;
    const float bv0 = (bias && ok0) ? bias[c0] : 0.f;
    const float bv1 = (bias && ok1) ? bias[c0 + 1] : 0.f;
    __nv_bfloat16* olo = ohi + out_plane;
    const bool vec_ok = vec_align && ok1;
#pragma unroll 4
    for (int r = 0; r < 32; r += 2) {
        const int row = row0 + r + half;
        if (row < M) {
            float x0 = fmaf(stg[(r + half) * pitch + cpair], alpha, bv0);
            float x1 = fmaf(stg[(r + half) * pitch + cpair + 1], alpha, bv1);
            if (RES) {
                if (ok0) x0 += res[(long long)row * ldo + c0];
                if (ok1) x1 += res[(long long)row * ldo + c0 + 1];
            }
            x0 = apply_act(x0, ACT);
            x1 = apply_act(x1, ACT);
            if (F32) {
                if (ok0) out[(long long)row * ldo + c0] = x0;
                if (ok1) out[(long long)row * ldo + c0 + 1] = x1;
            }
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(x0, h0, l0);
            split_bf16(x1, h1, l1);
            const long long o = (long long)row * ldo_s + c0;
            if (vec_ok) {
                *reinterpret_cast<uint32_t*>(ohi + o) = pack_bf16x2(h0, h1);
                *reinterpret_cast<uint32_t*>(olo + o) = pack_bf16x2(l0, l1);
            } else {
                if (ok0) ohi[o] = h0, olo[o] = l0;
                if (ok1) ohi[o + 1] = h1, olo[o + 1] = l1;
            }
        }
    }
}


__device__ __forceinline__ void atomic_max_f32(float* addr, float v) {
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// ---- vectorised epilogue (fast path) -------------------------------------------------------------------------------
// One 32-row x 32-column chunk of the staged fp32 tile per call: lane (rsub = lane/8, cg = lane%8) reads rows rsub,
// rsub+4, ... as float4 at columns 4*cg..4*cg+3, so every global instruction of the warp covers 4 rows x 128 contiguous
// bytes (8 LDS.128 + 8 STG.128, or 16 STG.64 for the split planes, per chunk instead of 32 + 32 scalar ones).
enum EpiMode { EPI_F32 = 0, EPI_ACC = 1, EPI_SPLIT = 2, EPI_SPLIT_F32 = 3, EPI_SWIGLU = 4, EPI_NONE = 5, EPI_SWIGLU_SPLIT = 6 };

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

template <int ACT, bool RES, int MODE>
__device__ __forceinline__ void epi_chunk_v4(const float* __restrict__ stg, int pitch, int lane, int row0, int M, int col0,
                                             const GemmEpilogue& ep, bool add_bias, float* out, const float* res,
                                             __nv_bfloat16* ohi) {
    const int cg = lane & 7, rsub = lane >> 3;
    const int col = col0 + cg * 4;
    const float4 b4 = add_bias ? ld4(ep.bias + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 c4 = ep.ln_stats ? ld4(ep.ln_c + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float alpha = ep.alpha;
    const float ninf = __int_as_float(0xff800000);
    float4 mx = make_float4(ninf, ninf, ninf, ninf);
    __nv_bfloat16* olo = ohi ? ohi + ep.out_plane : nullptr;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + rsub, row = row0 + rr;
        const bool ok = row < M;
        float4 x = ld4(stg + rr * pitch + cg * 4);
        // pre-activation: plain alpha*acc + bias, or the LayerNorm folded into this GEMM (A = un-normalised rows, W scaled by
        // gamma): rstd * (acc - mean * c[n]) + bias'[n] with the row statistics accumulated by the producer of A
        if (ep.ln_stats) {
            const float2 st = ok ? *reinterpret_cast<const float2*>(ep.ln_stats + 2 * (long long)row) : make_float2(0.f, 1.f);
            const float mean = st.x * ep.ln_inv_h;
            const float rstd = rsqrtf(fmaxf(fmaf(-mean, mean, st.y * ep.ln_inv_h), 0.f) + ep.ln_eps);
            const float ra = rstd * alpha, mr = add_bias ? -mean * rstd : 0.f;
            x.x = fmaf(x.x, ra, fmaf(mr, c4.x, b4.x)), x.y = fmaf(x.y, ra, fmaf(mr, c4.y, b4.y));
            x.z = fmaf(x.z, ra, fmaf(mr, c4.z, b4.z)), x.w = fmaf(x.w, ra, fmaf(mr, c4.w, b4.w));
        } else {
            x.x = fmaf(x.x, alpha, b4.x), x.y = fmaf(x.y, alpha, b4.y), x.z = fmaf(x.z, alpha, b4.z), x.w = fmaf(x.w, alpha, b4.w);
        }
        if (MODE == EPI_SWIGLU_SPLIT) {
            // product of the (gate, value) pairs -> split-bf16 planes + per-row (sum, sum of squares) for the LayerNorm that
            // the consuming GEMM applies algebraically (the reference normalises silu(g)*x before fc2, timm SwiGLU.norm)
            const float p0 = ok ? __fdividef(x.x, 1.0f + __expf(-x.x)) * x.y : 0.f;
            const float p1 = ok ? __fdividef(x.z, 1.0f + __expf(-x.z)) * x.w : 0.f;
            float s1 = p0 + p1, s2 = fmaf(p0, p0, p1 * p1);
#pragma unroll
            for (int o = 1; o <= 4; o <<= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (ok) {
                __nv_bfloat16 h0, l0, h1, l1;
                split_bf16(p0, h0, l0);
                split_bf16(p1, h1, l1);
                const long long o = (long long)row * ep.ldo_s + (col >> 1);
                *reinterpret_cast<uint32_t*>(ohi + o) = pack_bf16x2(h0, h1);
                *reinterpret_cast<uint32_t*>(olo + o) = pack_bf16x2(l0, l1);
                if (cg == 0 && ep.stats_out) {
                    atomicAdd(ep.stats_out + 2 * (long long)row, s1);
                    atomicAdd(ep.stats_out + 2 * (long long)row + 1, s2);
                }
            }
            continue;
        }
        if (ok && ep.gmax) mx.x = fmaxf(mx.x, x.x), mx.y = fmaxf(mx.y, x.y), mx.z = fmaxf(mx.z, x.z), mx.w = fmaxf(mx.w, x.w);
        if (MODE == EPI_NONE) continue;
        if (ok) {
            if (RES) {
                const float4 r4 = ld4(res + (long long)row * ep.ldo + col);
                x.x += r4.x, x.y += r4.y, x.z += r4.z, x.w += r4.w;
            }
            x.x = apply_act(x.x, ACT), x.y = apply_act(x.y, ACT), x.z = apply_act(x.z, ACT), x.w = apply_act(x.w, ACT);
            if (MODE == EPI_F32 || MODE == EPI_SPLIT_F32) *reinterpret_cast<float4*>(out + (long long)row * ep.ldo + col) = x;
            if (MODE == EPI_ACC) atomicAdd(reinterpret_cast<float4*>(out + (long long)row * ep.ldo + col), x);
            if (MODE == EPI_SWIGLU)
                *reinterpret_cast<float2*>(out + (long long)row * ep.ldo + (col >> 1)) =
                    make_float2(__fdividef(x.x, 1.0f + __expf(-x.x)) * x.y, __fdividef(x.z, 1.0f + __expf(-x.z)) * x.w);
            if (MODE == EPI_SPLIT || MODE == EPI_SPLIT_F32) {
                __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
                split_bf16(x.x, h0, l0);
                split_bf16(x.y, h1, l1);
                split_bf16(x.z, h2, l2);
                split_bf16(x.w, h3, l3);
                const long long o = (long long)row * ep.ldo_s + col;
                *reinterpret_cast<uint2*>(ohi + o) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
                *reinterpret_cast<uint2*>(olo + o) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
            }
        }
        if ((MODE == EPI_SPLIT || MODE == EPI_SPLIT_F32) && ep.stats_out) {
            // the rows this GEMM writes are the A operand of a LayerNorm-folded GEMM: accumulate their (sum, sum of squares)
            float s1 = ok ? (x.x + x.y) + (x.z + x.w) : 0.f;
            float s2 = ok ? fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, x.w * x.w))) : 0.f;
#pragma unroll
            for (int o = 1; o <= 4; o <<= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            }
            if (ok && cg == 0) {
                atomicAdd(ep.stats_out + 2 * (long long)row, s1);
                atomicAdd(ep.stats_out + 2 * (long long)row + 1, s2);
            }
        }
    }
    if (ep.gmax) {
        // rows of this chunk belong to one group: combine the 4 row sub-sets, then 8 lanes x 4 columns of atomics
#pragma unroll
        for (int o = 8; o <= 16; o <<= 1) {
            mx.x = fmaxf(mx.x, __shfl_xor_sync(0xffffffffu, mx.x, o));
            mx.y = fmaxf(mx.y, __shfl_xor_sync(0xffffffffu, mx.y, o));
            mx.z = fmaxf(mx.z, __shfl_xor_sync(0xffffffffu, mx.z, o));
            mx.w = fmaxf(mx.w, __shfl_xor_sync(0xffffffffu, mx.w, o));
        }
        if (rsub == 0 && row0 < M) {
            float* g = ep.gmax + (long long)(row0 / ep.group_rows) * ep.ld_gmax + col;
            atomic_max_f32(g, mx.x), atomic_max_f32(g + 1, mx.y), atomic_max_f32(g + 2, mx.z), atomic_max_f32(g + 3, mx.w);
        }
    }
}

template <int ACT>
__device__ __forceinline__ void epi_chunk_v4_dispatch(const float* stg, int pitch, int lane, int row0, int M, int col0,
                                                      const GemmEpilogue& ep, bool add_bias, float* out, const float* res,
                                                      __nv_bfloat16* ohi) {
#define PSAM_V4(R, MODE) epi_chunk_v4<ACT, R, MODE>(stg, pitch, lane, row0, M, col0, ep, add_bias, out, res, ohi)
    if (ep.swiglu && ohi) PSAM_V4(false, EPI_SWIGLU_SPLIT);
    else if (ep.swiglu) PSAM_V4(false, EPI_SWIGLU);
    else if (ep.accumulate) PSAM_V4(false, EPI_ACC);
    else if (ohi && out) { if (res) PSAM_V4(true, EPI_SPLIT_F32); else PSAM_V4(false, EPI_SPLIT_F32); }
    else if (ohi) { if (res) PSAM_V4(true, EPI_SPLIT); else PSAM_V4(false, EPI_SPLIT); }
    else if (out) { if (res) PSAM_V4(true, EPI_F32); else PSAM_V4(false, EPI_F32); }
    else PSAM_V4(false, EPI_NONE);
#undef PSAM_V4
}



// Epilogue of one 128 x BN tile from the staged fp32 accumulators `tile` (row pitch `pitch` floats).  Warp w of the
// eight consumer warps owns rows [32 (w % 4), +32) and the interleaved 32-column chunks c = w / 4, w / 4 + 2, ...
__device__ __forceinline__ void gemm_epilogue(const GemmShape& shape, const GemmEpilogue& ep, const float* tile, int pitch, int warp,
                                              int lane, int m_tile, int n_tile, int b1, int b2, int split, int BN) {
        const int quarter = warp & 3;
        const int row0 = m_tile * GEMM_BM + quarter * 32;
        const int ehalf = warp >> 2;
        const long long obase = (long long)b1 * ep.out_b1 + (long long)b2 * ep.out_b2;
        float* out = ep.out_f32 ? ep.out_f32 + obase : nullptr;
        const float* res = (ep.resid && !ep.accumulate) ? ep.resid + obase : nullptr;
        __nv_bfloat16* ohi = ep.out_hi ? ep.out_hi + (long long)b1 * ep.outs_b1 + (long long)b2 * ep.outs_b2 : nullptr;
        const bool add_bias = ep.bias && split == 0;
        const int nchunks = BN / 32;
#pragma unroll 1
        for (int c = ehalf; c < nchunks; c += 2) {
            const int col0 = n_tile * BN + c * 32;
            if (col0 >= shape.N) break;
            const float* stg = tile + quarter * 32 * pitch + c * 32;
            if (ep.rd_out) {
                // fused "masks = hyper_in @ upscaled^T" (mask_decoder.py:176): thread = row, the activated row chunk is
                // dotted with the rd_c hyper vectors and accumulated with one atomic per (row, c); the 32768 x 256
                // upscaled embedding is never written
                const int row = row0 + lane;
                const int zz = row0 / ep.rd_rows;
                const float* wz = ep.rd_w + (long long)zz * ep.rd_c * shape.N;
                float accd[8];
#pragma unroll
                for (int cc = 0; cc < 8; ++cc) accd[cc] = 0.f;
#pragma unroll
                for (int t = 0; t < 32; ++t) {
                    const int cidx = col0 + t;
                    if (cidx < shape.N) {
                        const float x = apply_act(fmaf(stg[lane * pitch + t], ep.alpha, add_bias ? ep.bias[cidx] : 0.f), ep.act);
#pragma unroll
                        for (int cc = 0; cc < 8; ++cc)
                            if (cc < ep.rd_c) accd[cc] = fmaf(x, wz[cc * shape.N + cidx], accd[cc]);
                    }
                }
                if (row < shape.M) {
                    float* o = ep.rd_out + (long long)zz * ep.rd_c * ep.rd_rows + (row - zz * ep.rd_rows);
#pragma unroll
                    for (int cc = 0; cc < 8; ++cc)
                        if (cc < ep.rd_c) atomicAdd(o + (long long)cc * ep.rd_rows, accd[cc]);
                }
                continue;
            }
            if (ep.vec4 && col0 + 32 <= shape.N) {
                if (ep.swiglu || ep.accumulate || ep.act == ACT_NONE)
                    epi_chunk_v4_dispatch<ACT_NONE>(stg, pitch, lane, row0, shape.M, col0, ep, add_bias, out, res, ohi);
                else if (ep.act == ACT_GELU) epi_chunk_v4_dispatch<ACT_GELU>(stg, pitch, lane, row0, shape.M, col0, ep, add_bias, out, res, ohi);
                else epi_chunk_v4_dispatch<ACT_RELU>(stg, pitch, lane, row0, shape.M, col0, ep, add_bias, out, res, ohi);
                continue;
            }
            const int col = col0 + lane;
            const bool col_ok = col < shape.N;
            if (ep.gmax) {
                // fused max-pool over the rows of a group (torch.max(x, dim=-2) of the mini-PointNet): the 32 rows of
                // this warp belong to one group; one atomic per column replaces a full write + re-read of x
                const float bvm = (add_bias && col_ok) ? ep.bias[col] : 0.f;
                float m = __int_as_float(0xff800000);
#pragma unroll 8
                for (int r = 0; r < 32; ++r)
                    if (row0 + r < shape.M) m = fmaxf(m, fmaf(stg[r * pitch + lane], ep.alpha, bvm));
                if (col_ok && row0 < shape.M) atomic_max_f32(ep.gmax + (long long)(row0 / ep.group_rows) * ep.ld_gmax + col, m);
                if (out == nullptr && ohi == nullptr) continue;
            }
            if (ohi == nullptr) {
                const float bv = (add_bias && col_ok) ? ep.bias[col] : 0.f;
#define PSAM_EPI_F32(A, R, C) epi_rows_f32<A, R, C>(stg, pitch, lane, row0, shape.M, col, col_ok, ep.alpha, bv, out, res, ep.ldo)
                if (ep.swiglu) epi_rows_swiglu(stg, pitch, lane, row0, shape.M, col, col_ok, ep.alpha, bv, out, ep.ldo);
                else if (ep.accumulate) PSAM_EPI_F32(ACT_NONE, false, true);
                else if (res) {
                    if (ep.act == ACT_NONE) PSAM_EPI_F32(ACT_NONE, true, false);
                    else if (ep.act == ACT_GELU) PSAM_EPI_F32(ACT_GELU, true, false);
                    else PSAM_EPI_F32(ACT_RELU, true, false);
                } else {
                    if (ep.act == ACT_NONE) PSAM_EPI_F32(ACT_NONE, false, false);
                    else if (ep.act == ACT_GELU) PSAM_EPI_F32(ACT_GELU, false, false);
                    else PSAM_EPI_F32(ACT_RELU, false, false);
                }
#undef PSAM_EPI_F32
            } else {
                const float* bias = add_bias ? ep.bias : nullptr;
                const bool va = ((ep.ldo_s | ep.out_plane | ep.outs_b1 | ep.outs_b2) & 1) == 0;
#define PSAM_EPI_SP(A, R, F) epi_rows_split<A, R, F>(stg, pitch, lane, row0, shape.M, shape.N, col0, ep.alpha, bias, out, res, ep.ldo, ohi, ep.out_plane, ep.ldo_s, va)
#define PSAM_EPI_SP_ACT(R, F)                                   \
    if (ep.act == ACT_NONE) PSAM_EPI_SP(ACT_NONE, R, F);        \
    else if (ep.act == ACT_GELU) PSAM_EPI_SP(ACT_GELU, R, F);   \
    else PSAM_EPI_SP(ACT_RELU, R, F)
                if (res) {
                    if (out) { PSAM_EPI_SP_ACT(true, true); } else { PSAM_EPI_SP_ACT(true, false); }
                } else {
                    if (out) { PSAM_EPI_SP_ACT(false, true); } else { PSAM_EPI_SP_ACT(false, false); }
                }
#undef PSAM_EPI_SP_ACT
#undef PSAM_EPI_SP
            }
        }
}

// Named barrier of the 256 consumer threads (the TMA warp does not take part).
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// One k-block of the split-bf16 product into the warpgroup's 64 x BN accumulator: 4 k-steps per pass.
template <int BN>
__device__ __forceinline__ void gemm_kblock(float (&acc)[BN / 2], uint32_t a_hi_addr, uint32_t a_lo_addr, uint32_t b_hi_addr,
                                            uint32_t b_lo_addr, bool lo_pass) {
    const uint64_t a_hi = gmma_desc_k(a_hi_addr), b_hi = gmma_desc_k(b_hi_addr);
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, a_hi + 2 * k, b_hi + 2 * k, 1u);
    if (lo_pass) {
        const uint64_t a_lo = gmma_desc_k(a_lo_addr), b_lo = gmma_desc_k(b_lo_addr);
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
    }
}

// Accumulator fragment of wgmma m64nN (thread = lane of warp w of the warpgroup): register i holds row
// 16 w + lane / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (lane % 4) + i % 2.
template <int BN>
__device__ __forceinline__ void stage_acc(float* tile, int pitch, int row_base, int lane, const float (&acc)[BN / 2]) {
    const int r = row_base + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        *reinterpret_cast<float2*>(tile + r * pitch + 8 * j + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(tile + (r + 8) * pitch + 8 * j + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, const GemmShape shape,
                  const GemmEpilogue ep) {
    pdl_launch_dependents();
    using S = GemmSmem<BN, STAGES>;
    extern __shared__ unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t full_bar[STAGES];
    __shared__ __align__(8) uint64_t empty_bar[STAGES];

    const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
    unsigned char* smem_aligned = smem_dyn + (smem_base - smem_u32(smem_dyn));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tile = blockIdx.x, m_tile = blockIdx.y;
    const int z = blockIdx.z;
    const int split = z % shape.split_k;
    const int bz = z / shape.split_k;
    const int b1 = bz % shape.nb1, b2 = bz / shape.nb1;

    const int kb_total = (shape.K + GEMM_BK - 1) / GEMM_BK;
    const int kb_per = (kb_total + shape.split_k - 1) / shape.split_k;
    const int kb_begin = split * kb_per;
    const int num_kb = max(0, min(kb_total, kb_begin + kb_per) - kb_begin);
    const bool lo_pass = shape.passes == 3;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 2);  // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();  // everything above is independent of the previous kernel; its outputs are read only below

    if (warp == 8) {
        // ===================== TMA producer: the hi and lo planes of a tile arrive with ONE 3-D box =====================
        if (lane == 0) {
            const uint32_t stage_bytes = (lo_pass ? 2u : 1u) * (uint32_t)(GEMM_A_TILE + S::B_TILE);
            for (int i = 0; i < num_kb; ++i) {
                const int s = i % STAGES;
                mbar_wait(smem_u32(&empty_bar[s]), ((uint32_t)(i / STAGES) & 1u) ^ 1u);
                const uint32_t fb = smem_u32(&full_bar[s]);
                const uint32_t sa = smem_base + s * S::STAGE;
                const int k0 = (kb_begin + i) * GEMM_BK;
                mbar_arrive_expect_tx(fb, stage_bytes);
                tma_load_5d(sa, &tmap_a, fb, k0, m_tile * GEMM_BM, 0, b1, b2);
                tma_load_5d(sa + 2 * GEMM_A_TILE, &tmap_b, fb, k0, n_tile * BN, 0, b1, b2);
            }
        }
        return;
    }
    // ===================== consumer warpgroups =====================
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int i = 0; i < num_kb; ++i) {
        const int s = i % STAGES;
        mbar_wait(smem_u32(&full_bar[s]), (uint32_t)(i / STAGES) & 1u);
        const uint32_t sa = smem_base + s * S::STAGE + wg * (GEMM_A_TILE / 2);  // this warpgroup's 64 rows
        const uint32_t sb = smem_base + s * S::STAGE + 2 * GEMM_A_TILE;
        fence_acc(acc);
        wgmma_fence();
        gemm_kblock<BN>(acc, sa, sa + GEMM_A_TILE, sb, sb + S::B_TILE, lo_pass);
        wgmma_commit();
        wgmma_wait<1>();  // the k-block before this one has retired: release its stage
        fence_acc(acc);
        if (i > 0 && (warp & 3) == 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[(i - 1) % STAGES]));
    }
    wgmma_wait<0>();
    fence_acc(acc);
    consumers_sync();  // every wgmma of both warpgroups has read its stage: the stage memory becomes the output tile
    float* tile = reinterpret_cast<float*>(smem_aligned);
    stage_acc<BN>(tile, S::PITCH, wg * 64 + (warp & 3) * 16, lane, acc);
    consumers_sync();
    gemm_epilogue(shape, ep, tile, S::PITCH, warp, lane, m_tile, n_tile, b1, b2, split, BN);
}

// ---------------------------------------------------------------------------------------------
// Row-complete GEMM with LayerNorm + GELU in the epilogue (mini-PointNet conv2[0..2], pc_sam/model/common.py:491-495):
//     Y = GELU(LayerNorm(A W^T + gbias[row / group_rows]))  ->  split-bf16
// A CTA owns 128 rows (warpgroup g: rows 64 g .. 64 g + 63) and computes each row over the FULL output width N = 256 NH,
// so the row statistics never leave the warp (a warp holds 16 whole rows; the four lanes of a quad share a row) and the
// fp32 pre-activation never reaches memory.  K <= 128: the A tile (both k-blocks, hi + lo = 64 KB) stays in shared memory
// while W sits in one 128 KB buffer, 256 rows at a time.  The registers hold one 64 x 256 accumulator per warpgroup, so
//   NH = 1: W is loaded once per CTA and stays resident; each tile is one product, exact two-pass statistics in registers;
//   NH = 2: the halves are computed in the order 0, 1, 0 - half 0 for its statistics only, half 1 for its statistics and
//           output (the two halves' (mean, M2) combined as in Chan et al.), half 0 again for its output.
// Persistent over the m-tiles.  warps 0-7: consumers, warp 8: TMA.
// ---------------------------------------------------------------------------------------------
struct RowLnParams {
    int M, N, K, passes;
    const float* gbias;   // [M / group_rows, N] or null
    long long ld_gbias;
    int group_rows;
    const float* gamma;   // [N]
    const float* beta;    // [N]
    float eps;
    int act;
    __nv_bfloat16* out_hi;  // [M, ldo_s] hi plane, lo plane at + out_plane
    long long out_plane, ldo_s;
};

constexpr int RL_A_TILE = 128 * 64 * 2;                  // one plane of one k-block of A
constexpr int RL_W_TILE = 256 * 64 * 2;                  // one plane of one k-block of a W half
constexpr int RL_SMEM = 2 * 2 * RL_A_TILE + 2 * 2 * RL_W_TILE + 1024;  // A: 2 k-blocks x (hi, lo); W half: 2 k-blocks x (hi, lo)

__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_rowln_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w, const RowLnParams p) {
    pdl_launch_dependents();
    extern __shared__ unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t a_full, a_empty, w_full, w_empty;

    const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
    const uint32_t sA = smem_base, sW = smem_base + 4 * RL_A_TILE;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int MT = ceil_div(p.M, GEMM_BM);
    const int NH = p.N / 256;                      // 256-column halves of the row
    const int KB = ceil_div(p.K, 64);              // k-blocks (1 or 2)
    const bool lo_pass = p.passes == 3;
    const uint32_t planes = lo_pass ? 2u : 1u;
    const bool resident = NH == 1;                 // W loaded once
    const int steps = NH == 1 ? 1 : 3;             // W halves per tile: 0 | 0, 1, 0

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_w);
        mbar_init(smem_u32(&a_full), 1);
        mbar_init(smem_u32(&a_empty), 2);
        mbar_init(smem_u32(&w_full), 1);
        mbar_init(smem_u32(&w_empty), 2);
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp == 8) {
        if (lane == 0) {
            auto load_w = [&](int h) {
                mbar_arrive_expect_tx(smem_u32(&w_full), planes * (uint32_t)(KB * RL_W_TILE));
                for (int kb = 0; kb < KB; ++kb)  // one 3-D box per k-block: 64 x 256 rows x {hi, lo}
                    tma_load_5d(sW + kb * 2 * RL_W_TILE, &tmap_w, smem_u32(&w_full), kb * 64, h * 256, 0, 0, 0);
            };
            if (resident) load_w(0);
            uint32_t it = 0, wit = 0;
            for (int tile = blockIdx.x; tile < MT; tile += gridDim.x, ++it) {
                mbar_wait(smem_u32(&a_empty), (it & 1u) ^ 1u);
                mbar_arrive_expect_tx(smem_u32(&a_full), planes * (uint32_t)(KB * RL_A_TILE));
                for (int kb = 0; kb < KB; ++kb)
                    tma_load_5d(sA + kb * 2 * RL_A_TILE, &tmap_a, smem_u32(&a_full), kb * 64, tile * GEMM_BM, 0, 0, 0);
                if (!resident) {
                    for (int st = 0; st < steps; ++st, ++wit) {
                        mbar_wait(smem_u32(&w_empty), (wit & 1u) ^ 1u);
                        load_w(st == 1 ? 1 : 0);
                    }
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // first of this thread's two rows in the tile (second: + 8)
    const int cq = 2 * (lane & 3);
    const float inv_half = 1.0f / 256.0f;
    uint32_t it = 0, wit = 0;
    for (int tile = blockIdx.x; tile < MT; tile += gridDim.x, ++it) {
        mbar_wait(smem_u32(&a_full), it & 1u);
        int rows[2] = {tile * GEMM_BM + rw, tile * GEMM_BM + rw + 8};
        const float* gb[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) gb[q] = (p.gbias && rows[q] < p.M) ? p.gbias + (long long)(rows[q] / p.group_rows) * p.ld_gbias : nullptr;
        float mean0[2] = {0.f, 0.f}, m2_0[2] = {0.f, 0.f}, mean[2], rstd[2];
        for (int st = 0; st < steps; ++st) {
            const int h = st == 1 ? 1 : 0;
            if (!resident || it == 0) mbar_wait(smem_u32(&w_full), resident ? 0u : (wit & 1u));
            float acc[128];
#pragma unroll
            for (int i = 0; i < 128; ++i) acc[i] = 0.f;
            fence_acc(acc);
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < 2; ++kb) {
                if (kb == KB) break;
                const uint32_t sa = sA + kb * 2 * RL_A_TILE + wg * (RL_A_TILE / 2), sw = sW + kb * 2 * RL_W_TILE;
                gemm_kblock<256>(acc, sa, sa + RL_A_TILE, sw, sw + RL_W_TILE, lo_pass);
            }
            wgmma_commit();
            wgmma_wait<0>();
            fence_acc(acc);
            if (!resident) {
                ++wit;
                if ((warp & 3) == 0 && lane == 0) mbar_arrive(smem_u32(&w_empty));  // this W half may be overwritten
            }
            if (st == steps - 1 && (warp & 3) == 0 && lane == 0) mbar_arrive(smem_u32(&a_empty));  // the A tile too
            // pre-activation + group bias, then exact two-pass statistics of this half of the row
            const int c0 = h * 256;
            float s1[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < 32; ++j) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const float2 g2 = gb[q] ? *reinterpret_cast<const float2*>(gb[q] + c0 + 8 * j + cq) : make_float2(0.f, 0.f);
                    acc[4 * j + 2 * q] += g2.x;
                    acc[4 * j + 2 * q + 1] += g2.y;
                    s1[q] += acc[4 * j + 2 * q] + acc[4 * j + 2 * q + 1];
                }
            }
            float mh[2], m2h[2];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                mh[q] = quad_sum(s1[q]) * inv_half;
                float s2 = 0.f;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const float d0 = acc[4 * j + 2 * q] - mh[q], d1 = acc[4 * j + 2 * q + 1] - mh[q];
                    s2 = fmaf(d0, d0, fmaf(d1, d1, s2));
                }
                m2h[q] = quad_sum(s2);
            }
            if (st == 0 && steps == 3) {  // statistics of half 0 only; its output comes in step 2
#pragma unroll
                for (int q = 0; q < 2; ++q) mean0[q] = mh[q], m2_0[q] = m2h[q];
                continue;
            }
            if (st < 2) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    if (steps == 1) {
                        mean[q] = mh[q];
                        rstd[q] = rsqrtf(m2h[q] * inv_half + p.eps);
                    } else {
                        // two equal halves: M2 = M2_0 + M2_1 + n_half ((mean_0 - mean)^2 + (mean_1 - mean)^2)
                        mean[q] = 0.5f * (mean0[q] + mh[q]);
                        const float d0 = mean0[q] - mean[q], d1 = mh[q] - mean[q];
                        rstd[q] = rsqrtf((m2_0[q] + m2h[q] + 256.0f * (d0 * d0 + d1 * d1)) * (0.5f * inv_half) + p.eps);
                    }
                }
            }
            // normalise, activate, store both planes
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (rows[q] >= p.M) continue;
                __nv_bfloat16* ohi = p.out_hi + (long long)rows[q] * p.ldo_s + c0 + cq;
                __nv_bfloat16* olo = ohi + p.out_plane;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int col = c0 + 8 * j + cq;
                    const float2 ga = *reinterpret_cast<const float2*>(p.gamma + col);
                    const float2 be = *reinterpret_cast<const float2*>(p.beta + col);
                    const float y0 = apply_act(fmaf((acc[4 * j + 2 * q] - mean[q]) * rstd[q], ga.x, be.x), p.act);
                    const float y1 = apply_act(fmaf((acc[4 * j + 2 * q + 1] - mean[q]) * rstd[q], ga.y, be.y), p.act);
                    __nv_bfloat16 h0, l0, h1, l1;
                    split_bf16(y0, h0, l0);
                    split_bf16(y1, h1, l1);
                    *reinterpret_cast<uint32_t*>(ohi + 8 * j) = pack_bf16x2(h0, h1);
                    *reinterpret_cast<uint32_t*>(olo + 8 * j) = pack_bf16x2(l0, l1);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side: tensor maps through the driver entry point (no link-time libcuda dependency)
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    }
    return fn;
}

static int make_operand_map(CUtensorMap* map, const psam_operand* op, int box_rows, int box_planes = 1) {
    PFN_encodeTiled enc = get_encode();
    if (!enc) return PSAM_ERR_UNSUPPORTED;
    const int nb1 = op->nb1 > 0 ? op->nb1 : 1, nb2 = op->nb2 > 0 ? op->nb2 : 1;
    cuuint64_t dims[5] = {(cuuint64_t)op->k, (cuuint64_t)op->rows, 2, (cuuint64_t)nb1, (cuuint64_t)nb2};
    // strides of dims 1..4 in bytes (dim 0 is contiguous); degenerate dims still need a 16-byte multiple
    const long long ps = op->plane_stride > 0 ? op->plane_stride : op->row_stride * (long long)op->rows;
    const long long s1 = op->b1_stride > 0 ? op->b1_stride : 8, s2 = op->b2_stride > 0 ? op->b2_stride : 8;
    cuuint64_t strides[4] = {(cuuint64_t)op->row_stride * 2, (cuuint64_t)ps * 2, (cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
    for (int i = 0; i < 4; ++i)
        if (strides[i] % 16) return PSAM_ERR_ARG;
    if (((uintptr_t)op->hi) % 16) return PSAM_ERR_ARG;
    cuuint32_t box[5] = {(cuuint32_t)GEMM_BK, (cuuint32_t)box_rows, (cuuint32_t)box_planes, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(op->hi), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? PSAM_OK : (int)(1000 + r);
}

int make_operand_map_ext(CUtensorMap* map, const psam_operand* op, int box_rows, int box_planes) {
    return make_operand_map(map, op, box_rows, box_planes);
}

template <int BN, int STAGES>
static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, const GemmShape& sh, const GemmEpilogue& ep, cudaStream_t stream) {
    auto kern = gemm_wgmma_kernel<BN, STAGES>;
    using S = GemmSmem<BN, STAGES>;
    PSAM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    const dim3 grid((unsigned)ceil_div(sh.N, BN), (unsigned)ceil_div(sh.M, GEMM_BM), (unsigned)(sh.nb1 * sh.nb2 * sh.split_k));
    PSAM_CUDA_TRY(psam::launch(kern, grid, dim3(GEMM_THREADS), (size_t)S::TOTAL, stream, ma, mb, sh, ep));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

// Output-tile width: 64, 128 or 256 minimising (waves over the 132 SMs of an H100) x (per-CTA cost), where the per-CTA cost
// follows the operand bytes streamed per k-block.  The throughput policy (several clouds in flight share the SMs) minimises
// the total SM-time instead, which favours wide tiles (fewer operand bytes per flop).
static int choose_bn(int M, int N, int K, int batches, int split_k, bool throughput) {
    const int mt = ceil_div(M, GEMM_BM);
    const int kb = ceil_div(ceil_div(K, GEMM_BK), split_k);
    int best = 128;
    double best_cost = 1e30;
    for (int bn = 64; bn <= 256; bn *= 2) {
        if (bn > 64 && bn / 2 >= N) break;
        const long long tiles = (long long)ceil_div(N, bn) * mt * batches * split_k;
        const long long waves = (tiles + 131) / 132;
        const double per_cta = 6.0 * 256 + (double)kb * (128 + bn) + 0.35 * bn * 4;
        const double cost = throughput ? (double)tiles * per_cta : (double)waves * per_cta;
        if (cost < best_cost - 1e-9) best_cost = cost, best = bn;
    }
    return best;
}

}  // namespace psam

extern "C" int psam_gemm_bf16x3(const psam_operand* a, const psam_operand* w, const psam_gemm_out* o, int passes,
                                int split_k, cudaStream_t stream) {
    using namespace psam;
    if (!a || !w || !o || !a->hi || !w->hi) return PSAM_ERR_ARG;
    if (a->k != w->k || a->k <= 0 || a->rows <= 0 || w->rows <= 0) return PSAM_ERR_ARG;
    if (passes != 1 && passes != 3) return PSAM_ERR_ARG;
    if (split_k < 1) split_k = 1;
    if (split_k > 1 && !(o->accumulate && o->out_f32 && !o->out_hi && o->act == 0)) return PSAM_ERR_ARG;
    if (!o->out_f32 && !o->out_hi && !o->gmax && !o->rd_out) return PSAM_ERR_ARG;
    GemmShape sh;
    sh.M = a->rows, sh.N = w->rows, sh.K = a->k;
    sh.nb1 = a->nb1 > 0 ? a->nb1 : 1;
    sh.nb2 = a->nb2 > 0 ? a->nb2 : 1;
    if ((w->nb1 > 0 ? w->nb1 : 1) != sh.nb1 || (w->nb2 > 0 ? w->nb2 : 1) != sh.nb2) return PSAM_ERR_ARG;
    sh.split_k = split_k;
    sh.passes = passes;
    const int variant = o->variant;
    GemmEpilogue ep;
    ep.out_f32 = o->out_f32, ep.ldo = o->ldo, ep.out_b1 = o->out_b1, ep.out_b2 = o->out_b2;
    ep.out_hi = (__nv_bfloat16*)o->out_hi, ep.out_plane = o->out_plane, ep.ldo_s = o->ldo_s;
    ep.outs_b1 = o->outs_b1, ep.outs_b2 = o->outs_b2;
    ep.bias = o->bias, ep.resid = o->resid, ep.alpha = o->alpha, ep.act = o->act, ep.accumulate = o->accumulate;
    ep.swiglu = o->swiglu;
    ep.gmax = o->gmax, ep.ld_gmax = o->ld_gmax, ep.group_rows = o->group_rows;
    ep.rd_w = o->rd_w, ep.rd_out = o->rd_out, ep.rd_rows = o->rd_rows, ep.rd_c = o->rd_c;
    {
        auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
        auto a8 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; };
        const bool off = (variant & GV_SCALAR_EPI) != 0;
        bool ok = !off && !ep.rd_out && (!ep.bias || a16(ep.bias));
        if (ep.out_f32) ok = ok && a16(ep.out_f32) && ((ep.ldo | ep.out_b1 | ep.out_b2) & 3) == 0;
        if (ep.resid) ok = ok && a16(ep.resid);
        if (ep.out_hi) ok = ok && a8(ep.out_hi) && ((ep.ldo_s | ep.out_plane | ep.outs_b1 | ep.outs_b2) & 3) == 0;
        if (ep.gmax) ok = ok && ep.group_rows % 32 == 0;
        ep.vec4 = ok ? 1 : 0;
    }
    ep.stats_out = o->stats_out, ep.ln_stats = o->ln_stats, ep.ln_c = o->ln_c;
    ep.ln_inv_h = o->ln_h > 0 ? 1.0f / (float)o->ln_h : 0.f, ep.ln_eps = o->ln_eps;
    // the fused forms exist only in the vectorised epilogue: whole 32-column chunks, aligned rows
    if ((ep.swiglu && ep.out_hi) || ep.ln_stats || ep.stats_out) {
        if (!ep.vec4 || sh.N % 32 != 0 || sh.nb1 * sh.nb2 != 1) return PSAM_ERR_UNSUPPORTED;
        if (ep.ln_stats && (!ep.ln_c || o->ln_h <= 0 || ep.gmax || ep.rd_out || (ep.swiglu && !ep.out_hi) ||
                            (reinterpret_cast<uintptr_t>(ep.ln_c) & 15) || (reinterpret_cast<uintptr_t>(ep.ln_stats) & 7)))
            return PSAM_ERR_ARG;
        // row statistics of the OUTPUT: either of the SwiGLU products, or of the rows written as split-bf16 (one writer per
        // element: no split-K, no accumulate)
        if (ep.stats_out && !(ep.out_hi && (ep.swiglu || (split_k == 1 && !ep.accumulate)))) return PSAM_ERR_ARG;
        if (ep.stats_out && (reinterpret_cast<uintptr_t>(ep.stats_out) & 7)) return PSAM_ERR_ARG;
    }
    if (ep.rd_out && (!ep.rd_w || ep.rd_rows <= 0 || ep.rd_rows % 32 || ep.rd_c <= 0 || ep.rd_c > 8 || ep.accumulate || ep.resid || ep.swiglu ||
                      ep.gmax || ep.out_f32 || ep.out_hi || split_k != 1 || sh.nb1 * sh.nb2 != 1)) return PSAM_ERR_ARG;
    if (ep.gmax && (ep.group_rows <= 0 || ep.group_rows % 32 || ep.accumulate || ep.resid || ep.act || ep.swiglu || sh.nb1 * sh.nb2 != 1)) return PSAM_ERR_ARG;
    if (ep.swiglu && ((!ep.out_hi == !ep.out_f32) || ep.accumulate || ep.resid || ep.act || (sh.N & 1))) return PSAM_ERR_ARG;
    int bn = choose_bn(sh.M, sh.N, sh.K, sh.nb1 * sh.nb2, sh.split_k, o->tile_hint == 1);
    if (o->tile_hint >= 32 && o->tile_hint <= 256 && o->tile_hint % 32 == 0) bn = o->tile_hint <= 64 ? 64 : (o->tile_hint <= 128 ? 128 : 256);
    sh.bn = bn;
    CUtensorMap ma, mb;
    int rc = make_operand_map(&ma, a, GEMM_BM, passes == 3 ? 2 : 1);
    if (rc) return rc;
    rc = make_operand_map(&mb, w, bn, passes == 3 ? 2 : 1);
    if (rc) return rc;
    if (bn == 64) return launch_gemm<64, 4>(ma, mb, sh, ep, stream);
    if (bn == 128) return launch_gemm<128, 3>(ma, mb, sh, ep, stream);
    return launch_gemm<256, 2>(ma, mb, sh, ep, stream);
}

extern "C" int psam_gemm_rowln_bf16x3(const psam_operand* a, const psam_operand* w, const float* gbias, long long ld_gbias, int group_rows,
                                      const float* gamma, const float* beta, float eps, int act, void* out_hi, long long out_plane,
                                      long long ldo_s, int passes, cudaStream_t stream) {
    using namespace psam;
    if (!a || !w || !a->hi || !w->hi || !gamma || !beta || !out_hi) return PSAM_ERR_ARG;
    if (a->k != w->k || a->rows <= 0 || (passes != 1 && passes != 3)) return PSAM_ERR_ARG;
    if ((w->rows != 256 && w->rows != 512) || a->k <= 0 || a->k > 128) return PSAM_ERR_UNSUPPORTED;
    if ((a->nb1 > 1) || (a->nb2 > 1) || (w->nb1 > 1) || (w->nb2 > 1)) return PSAM_ERR_UNSUPPORTED;
    if (gbias && (group_rows <= 0 || (ld_gbias & 3) || (reinterpret_cast<uintptr_t>(gbias) & 15))) return PSAM_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) | reinterpret_cast<uintptr_t>(out_hi)) & 15) return PSAM_ERR_ARG;
    if ((ldo_s & 7) || (out_plane & 7) || ldo_s < w->rows) return PSAM_ERR_ARG;
    RowLnParams p;
    p.M = a->rows, p.N = w->rows, p.K = a->k, p.passes = passes;
    p.gbias = gbias, p.ld_gbias = ld_gbias, p.group_rows = group_rows > 0 ? group_rows : 1;
    p.gamma = gamma, p.beta = beta, p.eps = eps, p.act = act;
    p.out_hi = (__nv_bfloat16*)out_hi, p.out_plane = out_plane, p.ldo_s = ldo_s;
    CUtensorMap ma, mw;
    int rc = make_operand_map(&ma, a, GEMM_BM, passes == 3 ? 2 : 1);
    if (rc) return rc;
    rc = make_operand_map(&mw, w, 256, passes == 3 ? 2 : 1);
    if (rc) return rc;
    int nsm = 132, devid = 0;
    if (cudaGetDevice(&devid) == cudaSuccess) cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, devid);
    const int mt = ceil_div(p.M, GEMM_BM);
    const int per = ceil_div(mt, nsm);
    const int ctas = ceil_div(mt, per);
    PSAM_CUDA_TRY(cudaFuncSetAttribute(gemm_rowln_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RL_SMEM));
    PSAM_CUDA_TRY(psam::launch(gemm_rowln_kernel, dim3((unsigned)ctas), dim3(GEMM_THREADS), (size_t)RL_SMEM, stream, ma, mw, p));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
