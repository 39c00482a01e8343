// Fused multi-head self-attention for sm_90a (encoder blocks): O = softmax(Q K^T * scale) V.
//
// Replaces F.scaled_dot_product_attention inside timm's EvaAttention (called from
// pc_sam/model/pc_encoder.py:138-139 via block(x); rope=None, no mask) and the four unfused kernels of
// an unfused implementation (QK^T GEMM, softmax, V transpose, PV GEMM).
//
// One CTA per (cloud, head, 128-query tile); two consumer warpgroups of 64 query rows each and one TMA warp.
//   warp 8     TMA producer: the Q tile once, then 64-key K and V blocks through a 4-stage mbarrier ring
//              (each stage = one 64-row block, hi+lo planes, per 64-column chunk of the head)
//   warps 0-7  per warpgroup and key block j:
//                S_j = Q K_j^T with wgmma (split-bf16, 3 passes) into fp32 registers,
//                softmax in registers (the four lanes of a quad share a row),
//                P_j split into bf16 hi/lo registers that are DIRECTLY the A operand of the next wgmma (the accumulator
//                fragment of m64n64 is the A fragment of k16 steps), O += P_j V_j with V_j^T read from the row-major V
//                block as an MN-major shared-memory B operand (no transpose pass)
// Streaming form (psam_attention_bf16x3): running row maximum, O and the row sum rescaled when it grows.
// Two-pass form (psam_attention_bf16x3_twopass, dh = 64): a first sweep over the K blocks computes the exact row maximum;
// the second sweep exponentiates with it, so nothing is rescaled.
// Head dims 64 and 88 (EVA-giant): dh = 88 is loaded as two 64-column chunks, the second holding columns 64..87 and the
// zeros TMA fills in beyond the head's extent.
// Numerics follow the split-bf16 scheme of gemm_tc.cu (x ~= hi + lo, three MMA passes).
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {

constexpr int ATT_BQ = 128;        // queries per CTA
constexpr int ATT_BKEY = 64;       // keys per block
constexpr int ATT_STAGES = 4;
constexpr int ATT_THREADS = 288;   // two consumer warpgroups + one TMA warp
constexpr int ATT_Q_TILE = 128 * 64 * 2;   // one plane of a 64-column chunk of the Q tile
constexpr int ATT_KV_TILE = 64 * 64 * 2;   // one plane of a 64-column chunk of a K or V block

template <int NCH>
struct AttSmem {
    static constexpr int Q = NCH * 2 * ATT_Q_TILE;
    static constexpr int STAGE = NCH * 2 * ATT_KV_TILE;
    static constexpr int TOTAL = Q + ATT_STAGES * STAGE + 1024;
};

struct AttnParams {
    int L, H, B;
    float scale_log2e;  // softmax scale * log2(e)
    __nv_bfloat16* out_hi;
    long long out_plane, ldo, out_h, out_b;  // elements: plane offset, row stride, head / cloud strides
};

__device__ __forceinline__ float ex2f(float x) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
    return e;
}

__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

__device__ __forceinline__ uint32_t bf16x2_bits(float lo, float hi) {
    const __nv_bfloat162 h2 = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h2);
}

// S = Q K^T for this warpgroup's 64 rows and one 64-key block: NCH chunks x {Q_hi K_hi, Q_lo K_hi, Q_hi K_lo}.
template <int NCH, int KS_LAST>
__device__ __forceinline__ void att_scores(float (&s)[32], uint32_t sq, uint32_t sk) {
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.f;
    fence_acc(s);
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
            const uint64_t qd = gmma_desc_k(sq + ch * 2 * ATT_Q_TILE + (pass == 1 ? ATT_Q_TILE : 0));
            const uint64_t kd = gmma_desc_k(sk + ch * 2 * ATT_KV_TILE + (pass == 2 ? ATT_KV_TILE : 0));
#pragma unroll
            for (int k = 0; k < (ch == NCH - 1 ? KS_LAST : 4); ++k) wgmma_ss<64>(s, qd + 2 * k, kd + 2 * k, 1u);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s);
}

// Keys at or beyond L take no part: their scores become -inf.  Register i of the fragment holds key 8 (i / 4) + 2 (lane % 4) + i % 2.
__device__ __forceinline__ void att_mask(float (&s)[32], int key0, int L, int lane) {
    if (key0 + ATT_BKEY <= L) return;
#pragma unroll
    for (int i = 0; i < 32; ++i)
        if (key0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= L) s[i] = __int_as_float(0xff800000);
}

template <int DH, bool TWO_PASS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
    constexpr int NCH = DH <= 64 ? 1 : 2;                         // 64-column chunks of a head
    constexpr int KS_LAST = DH <= 64 ? 4 : (DH - 64 + 15) / 16;   // 16-wide k-steps of the last chunk that hold data
    using S = AttSmem<NCH>;
    pdl_launch_dependents();
    extern __shared__ unsigned char smem_dyn[];
    __shared__ __align__(8) uint64_t q_full, kv_full[ATT_STAGES], kv_empty[ATT_STAGES];

    const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
    const uint32_t sQ = smem_base;      // chunk ch: hi plane at sQ + ch * 2 * ATT_Q_TILE, lo plane ATT_Q_TILE further
    const uint32_t sKV = sQ + S::Q;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q_tile = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int nkb = (p.L + ATT_BKEY - 1) / ATT_BKEY;

    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tmap_q);
        tma_prefetch_desc(&tmap_k);
        tma_prefetch_desc(&tmap_v);
        mbar_init(smem_u32(&q_full), 1);
        for (int s = 0; s < ATT_STAGES; ++s) {
            mbar_init(smem_u32(&kv_full[s]), 1);
            mbar_init(smem_u32(&kv_empty[s]), 2);  // one arrival per consumer warpgroup
        }
        fence_mbar_init();
    }
    __syncthreads();
    pdl_wait();  // everything above is independent of the previous kernel; its outputs are read only below

    // Order in which the stage ring carries the blocks (the consumers take them in exactly this order):
    //   two-pass: K_0 .. K_{nkb-1}, then K_0 V_0 K_1 V_1 ...;   streaming: K_0 V_0 K_1 V_1 ...
    const int n_items = (TWO_PASS ? 3 : 2) * nkb;
    if (warp == 8) {
        if (lane == 0) {
            const uint32_t qb = smem_u32(&q_full);
            mbar_arrive_expect_tx(qb, (uint32_t)S::Q);
            for (int ch = 0; ch < NCH; ++ch)  // one 3-D box per 64-column chunk: 64 x 128 rows x {hi, lo}
                tma_load_5d(sQ + ch * 2 * ATT_Q_TILE, &tmap_q, qb, 64 * ch, q_tile * ATT_BQ, 0, h, b);
            for (int i = 0; i < n_items; ++i) {
                const int s = i % ATT_STAGES;
                mbar_wait(smem_u32(&kv_empty[s]), ((uint32_t)(i / ATT_STAGES) & 1u) ^ 1u);
                const uint32_t fb = smem_u32(&kv_full[s]);
                mbar_arrive_expect_tx(fb, (uint32_t)S::STAGE);
                const int i2 = TWO_PASS ? i - nkb : i;  // position in the K V K V ... sequence (< 0: first sweep)
                const bool is_v = i2 >= 0 && (i2 & 1);
                const int blk = i2 < 0 ? i : (i2 >> 1);
                for (int ch = 0; ch < NCH; ++ch)
                    tma_load_5d(sKV + s * S::STAGE + ch * 2 * ATT_KV_TILE, is_v ? &tmap_v : &tmap_k, fb, 64 * ch, blk * ATT_BKEY, 0, h, b);
            }
        }
        return;
    }

    // ===================== consumer warpgroup: 64 query rows =====================
    const int wg = warp >> 2;
    const bool leader = (warp & 3) == 0 && lane == 0;  // releases stages for the warpgroup
    const uint32_t sq = sQ + wg * (ATT_Q_TILE / 2);
    const float c = p.scale_log2e;
    mbar_wait(smem_u32(&q_full), 0);
    int item = 0;
    auto acquire = [&]() {
        const int s = item % ATT_STAGES;
        mbar_wait(smem_u32(&kv_full[s]), (uint32_t)(item / ATT_STAGES) & 1u);
        return sKV + s * S::STAGE;
    };
    auto release = [&]() {
        if (leader) mbar_arrive(smem_u32(&kv_empty[item % ATT_STAGES]));
        ++item;
    };

    float m[2] = {__int_as_float(0xff800000), __int_as_float(0xff800000)};  // running maxima of the thread's two rows
    float s[32];
    if (TWO_PASS) {
        for (int j = 0; j < nkb; ++j) {
            att_scores<NCH, KS_LAST>(s, sq, acquire());
            release();
            att_mask(s, j * ATT_BKEY, p.L, lane);
#pragma unroll
            for (int i = 0; i < 32; ++i) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], s[i]);
        }
        m[0] = quad_max(m[0]);
        m[1] = quad_max(m[1]);
    }
    float o[NCH][32];
#pragma unroll
    for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
        for (int i = 0; i < 32; ++i) o[ch][i] = 0.f;
    float l[2] = {0.f, 0.f};  // partial row sums (this thread's columns)
    for (int j = 0; j < nkb; ++j) {
        att_scores<NCH, KS_LAST>(s, sq, acquire());
        release();
        att_mask(s, j * ATT_BKEY, p.L, lane);
        if (!TWO_PASS) {
            float mb[2] = {m[0], m[1]};
#pragma unroll
            for (int i = 0; i < 32; ++i) mb[(i >> 1) & 1] = fmaxf(mb[(i >> 1) & 1], s[i]);
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                mb[q] = quad_max(mb[q]);  // finite: every block holds at least one key < L
                const float f = ex2f((m[q] - mb[q]) * c);  // first block: m = -inf -> f = 0
                l[q] *= f;
#pragma unroll
                for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        if (((i >> 1) & 1) == q) o[ch][i] *= f;
                m[q] = mb[q];
            }
        }
        // P = exp2(S c - m c) split into bf16 hi / lo: k-step kk (16 keys) uses registers 8 kk .. 8 kk + 7
        uint32_t ph[4][4], pl[4][4];
        const float nm[2] = {-m[0] * c, -m[1] * c};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int i = 8 * kk + 2 * r, q = r & 1;
                const float e0 = ex2f(fmaf(s[i], c, nm[q])), e1 = ex2f(fmaf(s[i + 1], c, nm[q]));
                l[q] += e0 + e1;
                ph[kk][r] = bf16x2_bits(e0, e1);
                const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ph[kk][r]));
                pl[kk][r] = bf16x2_bits(e0 - hf.x, e1 - hf.y);
            }
        }
        const uint32_t sv = acquire();
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) fence_acc(o[ch]);
        wgmma_fence();
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
            const uint64_t v_hi = gmma_desc_mn64(sv + ch * 2 * ATT_KV_TILE), v_lo = gmma_desc_mn64(sv + ch * 2 * ATT_KV_TILE + ATT_KV_TILE);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {  // V: 16 rows = 2048 B further per k-step
                wgmma_rs_tb<64>(o[ch], ph[kk], v_hi + (uint64_t)(kk * (2048 >> 4)));
                wgmma_rs_tb<64>(o[ch], pl[kk], v_hi + (uint64_t)(kk * (2048 >> 4)));
                wgmma_rs_tb<64>(o[ch], ph[kk], v_lo + (uint64_t)(kk * (2048 >> 4)));
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) fence_acc(o[ch]);
        release();
    }
    // ---- epilogue: O / rowsum -> split-bf16 [B*L, H*dh] ----
    const int rbase = q_tile * ATT_BQ + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        float lq = l[q] + __shfl_xor_sync(0xffffffffu, l[q], 1);
        lq += __shfl_xor_sync(0xffffffffu, lq, 2);
        const float inv = 1.0f / lq;
        const int row = rbase + 8 * q;
        if (row >= p.L) continue;
        __nv_bfloat16* ohi = p.out_hi + (long long)b * p.out_b + (long long)h * p.out_h + (long long)row * p.ldo;
        __nv_bfloat16* olo = ohi + p.out_plane;
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const int col = ch * 64 + 8 * g + 2 * (lane & 3);
                if (col >= DH) continue;
                __nv_bfloat16 h0, l0, h1, l1;
                split_bf16(o[ch][4 * g + 2 * q] * inv, h0, l0);
                split_bf16(o[ch][4 * g + 2 * q + 1] * inv, h1, l1);
                *reinterpret_cast<uint32_t*>(ohi + col) = pack_bf16x2(h0, h1);
                *reinterpret_cast<uint32_t*>(olo + col) = pack_bf16x2(l0, l1);
            }
        }
    }
}

int make_operand_map_ext(CUtensorMap* map, const psam_operand* op, int box_rows, int box_planes);  // gemm_tc.cu

static int attention_setup(const psam_operand* q, const psam_operand* k, const psam_operand* v, void* out_hi, long long out_plane,
                           long long ldo, long long out_head_stride, long long out_cloud_stride, float scale, CUtensorMap* mq,
                           CUtensorMap* mk, CUtensorMap* mv, AttnParams* p, dim3* grid) {
    if (!q || !k || !v || !out_hi) return PSAM_ERR_ARG;
    const int L = q->rows, dh = q->k;
    const int H = q->nb1 > 0 ? q->nb1 : 1, B = q->nb2 > 0 ? q->nb2 : 1;
    if ((dh != 64 && dh != 88) || L <= 0) return PSAM_ERR_UNSUPPORTED;
    if (k->rows != L || v->rows != L || k->k != dh || v->k != dh) return PSAM_ERR_ARG;
    // K and V cover the same heads and clouds as Q (TMA would fill the missing ones with zeros)
    for (const psam_operand* x : {k, v})
        if ((x->nb1 > 0 ? x->nb1 : 1) != H || (x->nb2 > 0 ? x->nb2 : 1) != B) return PSAM_ERR_ARG;
    // the kernels subtract the maximum of the raw scores, which is the maximum of the scaled ones only for scale > 0
    if (!(scale > 0.f) || !isfinite(scale)) return PSAM_ERR_ARG;
    if ((ldo | out_plane | out_head_stride | out_cloud_stride) & 7) return PSAM_ERR_ARG;
    int rc = make_operand_map_ext(mq, q, ATT_BQ, 2);
    if (rc) return rc;
    rc = make_operand_map_ext(mk, k, ATT_BKEY, 2);
    if (rc) return rc;
    rc = make_operand_map_ext(mv, v, ATT_BKEY, 2);
    if (rc) return rc;
    p->L = L, p->H = H, p->B = B;
    p->scale_log2e = scale * 1.4426950408889634f;
    p->out_hi = (__nv_bfloat16*)out_hi;
    p->out_plane = out_plane, p->ldo = ldo, p->out_h = out_head_stride, p->out_b = out_cloud_stride;
    *grid = dim3((unsigned)ceil_div(L, ATT_BQ), (unsigned)H, (unsigned)B);
    return PSAM_OK;
}

template <int DH, bool TWO_PASS>
static int launch_attention(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttnParams& p, dim3 grid,
                            cudaStream_t stream) {
    auto kern = attention_wgmma_kernel<DH, TWO_PASS>;
    constexpr int smem = AttSmem<DH <= 64 ? 1 : 2>::TOTAL;
    PSAM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    PSAM_CUDA_TRY(psam::launch(kern, grid, dim3(ATT_THREADS), (size_t)smem, stream, mq, mk, mv, p));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

}  // namespace psam

extern "C" int psam_attention_bf16x3(const psam_operand* q, const psam_operand* k, const psam_operand* v, void* out_hi,
                                     long long out_plane, long long ldo, long long out_head_stride,
                                     long long out_cloud_stride, float scale, cudaStream_t stream) {
    using namespace psam;
    CUtensorMap mq, mk, mv;
    AttnParams p;
    dim3 grid;
    int rc = attention_setup(q, k, v, out_hi, out_plane, ldo, out_head_stride, out_cloud_stride, scale, &mq, &mk, &mv, &p, &grid);
    if (rc) return rc;
    if (q->k == 88) return launch_attention<88, false>(mq, mk, mv, p, grid, stream);
    return launch_attention<64, false>(mq, mk, mv, p, grid, stream);
}

extern "C" int psam_attention_bf16x3_twopass(const psam_operand* q, const psam_operand* k, const psam_operand* v, void* out_hi,
                                             long long out_plane, long long ldo, long long out_head_stride,
                                             long long out_cloud_stride, float scale, cudaStream_t stream) {
    using namespace psam;
    CUtensorMap mq, mk, mv;
    AttnParams p;
    dim3 grid;
    if (q && q->k != 64) return PSAM_ERR_UNSUPPORTED;  // the two-pass form covers dh = 64 only
    int rc = attention_setup(q, k, v, out_hi, out_plane, ldo, out_head_stride, out_cloud_stride, scale, &mq, &mk, &mv, &p, &grid);
    if (rc) return rc;
    return launch_attention<64, true>(mq, mk, mv, p, grid, stream);
}
