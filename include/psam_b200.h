/* psam_b200 - C ABI of the Point-SAM hot path on the H100 (sm_90a).
 *
 * This is the drop-in boundary.  In the reference the native boundary for this path is the pybind11
 * module torkit3d._C (third_party/torkit3d/torkit3d/csrc/torkit3d.cpp:10-23,
 * csrc/include/sample_farthest_points.h:6-8) plus the ATen/cuBLAS/apex kernels PyTorch dispatches to
 * from pc_sam/model/*.py.  Every entry point below names the reference interface it stands in for.
 *
 * Conventions: plain pointers and sizes only (no torch types); all pointers are DEVICE pointers unless
 * stated; tensors are contiguous row-major fp32 unless stated; no allocation inside (caller passes
 * outputs and workspace, `*_workspace_bytes` tells how much); no global mutable state, thread-safe,
 * work is enqueued on `stream` and nothing synchronises; return 0 on success, a negative PSAM_ERR_*
 * for bad arguments, a positive cudaError_t if a CUDA call failed (1000+CUresult for driver errors).
 *
 * Padded batches (the *_varlen entry points): B clouds of different sizes are held as [B, N_max, ...] with lengths [B]
 * (int32, DEVICE): cloud b's points are its rows n < lengths[b], later rows are padding that is never read.  Precondition:
 * 1 <= lengths[b] <= N_max (plus the call's own lower bound).  Kernels clamp each length into [0, N_max], so nothing past
 * N_max is read or written whatever lengths holds, but the results for an out-of-range length are unspecified.
 *
 * "split-bf16" operands: two bf16 planes [2][rows][row_stride] with x ~= hi + lo (|err| <= 2^-17 |x|);
 * plane 0 = hi, plane 1 = lo, lo plane `plane_stride` elements after the hi plane.
 */
#ifndef PSAM_B200_H
#define PSAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#define PSAM_ACT_NONE 0
#define PSAM_ACT_GELU 1
#define PSAM_ACT_RELU 2

/* ---- tokenizer ------------------------------------------------------------------------------ */

/* Farthest-point sampling + gather of the centres.
 * Replaces torkit3d._C.sample_farthest_points_cuda (sample_farthest_points_kernel.cu:106-165, called
 * from pc_sam/model/common.py:91) and batch_index_select (torkit3d/nn/functional.py:34-69, common.py:92).
 * xyz [B,N,3] -> idx_out [B,G] int64 (bit-exact with the reference kernel incl. tie-break),
 * centers_out [B,G,3].  Errors mirror the reference TORCH_CHECKs (:111-115): G<=0 or N<G -> PSAM_ERR_ARG.
 * workspace: psam_fps_workspace_bytes(B, N, G) bytes; it may be NULL when that is 0, and a NULL workspace where it is not
 * 0 -> PSAM_ERR_ARG.  Coordinates must be finite: NaN or inf coordinates are outside the contract. */
size_t psam_fps_workspace_bytes(int B, int N, int G);
int psam_fps_f32(const float* xyz, int B, int N, int G, long long* idx_out, float* centers_out, void* workspace,
                 cudaStream_t stream);
/* psam_fps_f32 on a padded batch: xyz [B, N_max, 3], lengths [B].  Cloud b samples among its
 * first lengths[b] points and its slots 0 .. min(G, lengths[b]) - 1 are bit-identical to psam_fps_f32 on that cloud alone
 * with G' = min(G, lengths[b]) (greedy FPS is prefix-consistent): the tie-break block size T is derived from lengths[b],
 * not from N_max.  Slots lengths[b] .. G-1 repeat sample 0 (index 0, centre xyz[b, 0]).  G may exceed N_max.  The cluster
 * plan and the workspace come from N_max (psam_fps_workspace_bytes(B, N_max, G)); the result does not depend on them.
 * Padded-batch rules as stated at the top of this header. */
int psam_fps_varlen_f32(const float* xyz, const int* lengths, int B, int N_max, int G, long long* idx_out, float* centers_out,
                        void* workspace, cudaStream_t stream);

/* K nearest keys of every query (exact, direct-difference squared distance, ties by lower index),
 * sorted by (distance, index).  Replaces knn_points = torch.cdist + torch.topk
 * (pc_sam/model/common.py:27-56; call sites :97 and :251).  query [B,Q,3], key [B,N,3] ->
 * idx_out [B,Q,K] int64, d2_out [B,Q,K] squared distances (may be NULL).  K <= 1024 and B <= 65535, else
 * PSAM_ERR_UNSUPPORTED.  Coordinates must be finite: NaN or inf coordinates are outside the contract. */
int psam_knn_f32(const float* query, const float* key, int B, int Q, int N, int K, long long* idx_out, float* d2_out,
                 cudaStream_t stream);
/* psam_knn_f32 on a padded batch: key [B, N_max, 3], lengths [B]; the keys of cloud b are its first lengths[b] rows, and
 * every query row's indices and distances equal psam_knn_f32 on the unpadded cloud bit for bit, ties included.  Query rows
 * are not limited (query [B, Q, 3]): the outputs of padded query rows are valid results for those points, and callers
 * ignore them.  Precondition: K <= lengths[b] (a length below K is treated as K).  K <= N_max.
 * Padded-batch rules as stated at the top of this header. */
int psam_knn_varlen_f32(const float* query, const float* key, const int* lengths, int B, int Q, int N_max, int K,
                        long long* idx_out, float* d2_out, cudaStream_t stream);

/* Group-feature gather: groups[b2,g,k,:] = [(xyz[b,idx]-centers[b,g])/radius, feats[b2,idx,0:C]], b=b2/rep.
 * Replaces the fancy-index gathers of KNNGrouper.forward (common.py:99-120) and
 * group_with_centers_and_knn (common.py:126-187).  radius<=0 means None.  feats [B*rep,N,C].
 * center_idx [B,G] (may be NULL) selects centralize_features=True (common.py:116-118, :181-185): C more channels
 * feats[b2,idx] - feats[b2,center_idx[b,g]] are appended (groups_out row = 3 + 2C floats).  N, G, K >= 1.
 * Rounding, exact: each coordinate is fp32(xyz - centre), times fp32(1 / radius) when radius > 0.  That product is what
 * torch computes on CUDA for `tensor / radius` with a Python-float radius (a CPU scalar divisor becomes a multiplication
 * by its fp32 reciprocal, as checked on an H100 with torch 2.11); it differs by 1 ulp from an fp32 division for about
 * 12 % of uniform values in [-1, 1] at radius 0.05 or 0.1.
 * Feature channels are copies, and the centralised ones fp32(f - f_centre). */
int psam_group_gather_f32(const float* xyz, const float* feats, const float* centers, const long long* knn_idx,
                          const long long* center_idx, int B, int rep, int N, int G, int K, int C, float radius,
                          float* groups_out, cudaStream_t stream);

/* Voronoi tokenizer features: out[b2,n,:] = [(xyz[b,n]-c)/max(|xyz[b,n]-c|,1e-8), |xyz[b,n]-c|, feats[b2,n,0:C]] with
 * c = centers[b, nn_idx[b,n]], b = b2/rep.  Replaces NNGrouper.forward / group_with_centers_and_nn
 * (common.py:190-236).  out fp32 [B*rep,N,4+C] and / or the split-bf16 copy y_hi (row pitch `pitch` >= 4+C, zero
 * padded) that feeds PatchEmbedNN.in_proj (pc_encoder.py:186) on the tensor cores.
 * Rounding: d = fp32(xyz - c) per axis, dist = sqrtf of the sum of squares, computed as one product and two fused
 * multiply-adds (three roundings in the sum, halved by the square root, plus the square root's own: relative error at
 * most 2.5 * 2^-24 against the exact norm of d; 2^-23 would not hold), and
 * each direction component is the fp32 quotient d / max(dist, 1e-8) - a division, as torch divides by a tensor.  The split
 * planes are hi = bf16(v), lo = bf16(v - hi) of those fp32 values.  pitch >= 4 + C whenever y_hi is given, and at least
 * one of out and y_hi, else PSAM_ERR_ARG. */
int psam_voronoi_features_f32(const float* xyz, const float* centers, const long long* nn_idx, const float* feats, int B,
                              int rep, int N, int G, int C, float* out, void* y_hi, long long y_plane, long long pitch,
                              cudaStream_t stream);

/* y[b, nn_idx[b,n], :] = max over the points of a Voronoi cell of x[b,n,:]; cells without a point are 0.
 * Replaces y.scatter_reduce_(1, nn_idx, x, "amax", include_self=False) on a zero tensor (pc_encoder.py:189-193), bit for
 * bit: the maximum is exact, and -0.0 orders below +0.0 and above every negative value (a cell holding -0.0 and negative
 * values gives -0.0).  NaN inputs are outside this contract.  x [B,N,D], y [B,G,D], D % 4 == 0. */
int psam_scatter_amax_f32(const float* x, const long long* nn_idx, int B, int N, int G, int D, float* y,
                          cudaStream_t stream);

/* 3 nearest centres per point and inverse-squared-distance weights.
 * Replaces compute_interp_weights (common.py:238-255).  idx_out [B,N,3] int64, w_out [B,N,3].  B <= 65535, else
 * PSAM_ERR_UNSUPPORTED. */
int psam_knn3_interp_f32(const float* xyz, const float* centers, int B, int N, int G, long long* idx_out, float* w_out,
                         cudaStream_t stream);

/* Nearest-neighbour squared distance (and index) of every query point to a key set; single cloud.
 * Replaces torkit3d chamfer_distance_forward (csrc/cuda/chamfer_distance_kernel.cu:10-151) as used by the
 * ground-truth prompt sampler (pc_sam/model/common.py:447-474): dist1/idx1 only.  idx_out may be NULL.
 * Ties go to the lower key index.  A key whose squared distance is NaN or not below 3.4e38 (a NaN or inf key) is never
 * chosen; a query with no such key (a NaN query, for one) gets (3.4e38, -1). */
int psam_nn_distance_f32(const float* query, const float* key, int n1, int n2, float* dist_out, long long* idx_out,
                         cudaStream_t stream);

/* Batched ground-truth prompt sampler: replaces the per-(cloud, mask) Python loops of sample_fixed_points /
 * sample_furthest_points_from_border (pc_sam/model/common.py:371-474) and their chamfer_distance calls with four launches
 * and no host synchronisation.  gt_masks [B*M, N] (0/1 bytes); prediction either as logits (mask = logit > 0,
 * common.py:392) or as 0/1 bytes (thresholded by the caller), or both NULL (first iteration: pred_logits is None).
 * from_error_region != 0: sample the point of (fn | fp) farthest from its complement (common.py:402-410);
 * == 0: the farther of the fn- and fp-region candidates, falling back to the ground-truth region (common.py:411-431).
 * Distances and tie-breaks equal the reference's (chamfer arithmetic, torch.argmax = lowest index).
 * Outputs: prompt_xyz_out [B*M, 3], prompt_label_out [B*M] (the ground-truth value at the sampled point), *status is
 * set to 1 if some mask had no valid candidate (the reference raises in torch.stack there); the caller zeroes it.
 * workspace: psam_border_prompt_workspace_bytes(B, M, N) bytes, 4-byte aligned (region counters, compacted foreground /
 * background index lists and per-point minima: the distance sweep costs |fg| x |bg| evaluations like the reference's
 * compacted chamfer call, spread over (fg block x background chunk) thread blocks). */
size_t psam_border_prompt_workspace_bytes(int B, int M, int N);
int psam_border_prompt_f32(const float* coords, const unsigned char* gt_masks, const float* pred_logits,
                           const unsigned char* pred_masks, int B, int M, int N, int from_error_region,
                           float* prompt_xyz_out, unsigned char* prompt_label_out, int* status, void* workspace,
                           cudaStream_t stream);

/* psam_border_prompt_f32 on a padded batch: coords [B, N_max, 3], lengths [B], gt_masks / pred_logits / pred_masks
 * [B*M, N_max].  Row i of (cloud b, mask m) takes part only when i < N_b = clamp(lengths[b], 0, N_max): rows at or past
 * N_b go on neither the foreground nor the background list.  For every (b, m) the prompt xyz and label are bit for bit
 * those psam_border_prompt_f32 returns on cloud b alone (its first N_b rows of coords, ground truth and prediction), and
 * *status is set exactly when one of those single-cloud calls would set it (N_b = 0 counts as a mask without a border),
 * whatever the padding rows hold.  Workspace: psam_border_prompt_workspace_bytes(B, M, N_max).  Refusals: those of
 * psam_border_prompt_f32, and PSAM_ERR_ARG for a NULL lengths. */
int psam_border_prompt_varlen_f32(const float* coords, const int* lengths, const unsigned char* gt_masks,
                                  const float* pred_logits, const unsigned char* pred_masks, int B, int M, int N_max,
                                  int from_error_region, float* prompt_xyz_out, unsigned char* prompt_label_out, int* status,
                                  void* workspace, cudaStream_t stream);

/* ---- dense contractions ---------------------------------------------------------------------- */

typedef struct {
    const void* hi;         /* bf16 hi plane, 16-byte aligned */
    long long plane_stride; /* elements from hi plane to lo plane (0: rows*row_stride) */
    int rows, k;            /* logical extents; k tail and row tail are zero-filled by TMA */
    long long row_stride;   /* elements, multiple of 8 */
    int nb1, nb2;           /* batch extents (0/1 = none) */
    long long b1_stride, b2_stride; /* elements, multiples of 8 */
} psam_operand;

typedef struct {
    float* out_f32;         /* optional fp32 output [.., M, ldo] */
    long long ldo, out_b1, out_b2;
    void* out_hi;           /* optional split-bf16 output (hi plane; lo at +out_plane elements).  Any bf16-aligned address:
                             * the vectorised epilogue runs when out_hi is 8-byte aligned and ldo_s, out_plane, outs_b1,
                             * outs_b2 are multiples of 4; otherwise the scalar one stores column pairs as 32-bit words
                             * only when out_hi is 4-byte aligned and those strides are even, and single bf16 otherwise */
    long long out_plane, ldo_s, outs_b1, outs_b2;
    const float* bias;      /* [N] or NULL */
    const float* resid;     /* fp32, geometry of out_f32 (may alias it) or NULL */
    float alpha;            /* accumulator scale (1.0f for a plain linear) */
    int act;                /* PSAM_ACT_* applied after bias/residual */
    int accumulate;         /* 1: out_f32 += alpha*acc (+bias) with red.add; required when split_k>1.  Needs out_f32, and
                             * out_hi == NULL, act == 0, resid NULL or == out_f32 (out_f32 is its own residual);
                             * PSAM_ERR_ARG otherwise */
    int swiglu;             /* 1: W rows interleaved (gate_i, value_i); out_f32[:, i] = silu(gate_i)*value_i (fp32 out only) */
    int tile_hint;          /* 0: tile width for lowest latency; 1: for lowest SM-time (several clouds in flight); 32..256: explicit
                               (a multiple of 32, rounded up to the tile widths the kernel has: 64, 128, 256) */
    float* gmax;            /* optional fused max-pool: gmax[(row / group_rows) * ld_gmax + col] = max over the group rows
                               (atomic; caller pre-fills with -inf; group_rows multiple of 32); replaces torch.max(x, dim=-2).
                               -0.0 orders below +0.0 and above every negative value; NaN values are outside this contract */
    long long ld_gmax;
    int group_rows;
    const float* rd_w;      /* optional fused row-dot (replaces masks = hyper_in @ upscaled^T, mask_decoder.py:176):        */
    float* rd_out;          /*   rd_out[z, c, n] += sum_col act(alpha*acc + bias)[z*rd_rows + n, col] * rd_w[z, c, col]    */
    int rd_rows, rd_c;      /*   rd_out pre-zeroed [Z, rd_c, rd_rows]; rd_rows % 32 == 0; rd_c <= 8; no other output allowed */
    float* stats_out;       /* stats_out[row] (2 floats, pre-zeroed) accumulates (sum, sum of squares) of the row this GEMM
                             * WRITES as split-bf16 - the statistics a LayerNorm-folded consumer GEMM needs: with swiglu +
                             * out_hi the SwiGLU products (timm SwiGLU.norm), otherwise (out_hi, split_k == 1, no
                             * accumulate) the final values after bias / residual / activation (norm1 / norm2 / fc_norm) */
    const float* ln_stats;  /* LayerNorm folded into this GEMM: A = the un-normalised rows, W pre-multiplied by gamma,
                             * ln_c[n] = sum_k gamma_k W[n,k], bias[n] = sum_k beta_k W[n,k] + b[n];
                             * out = act(alpha * rstd_row * (acc - mean_row * ln_c[n]) + bias[n] (+ resid)) with mean / rstd
                             * from ln_stats[row] = (sum, sum sq) over ln_h columns; bias may be NULL.  Works with every
                             * output form of the vectorised epilogue (fp32, split-bf16, SwiGLU pairs) and with accumulate /
                             * split_k (each split scales its partial sum; split 0 adds the mean term and the bias). */
    const float* ln_c;
    int ln_h;
    float ln_eps;
    int variant;            /* 0 = policy default.  0x4 forces the scalar epilogue (the library reads no environment
                             * variable); every other bit is accepted and has no effect on sm_90a */
} psam_gemm_out;

/* C[M,N] = A[M,K] * W[N,K]^T on the tensor cores (TMA-fed wgmma, fp32 register accumulators).
 * passes=3: split-bf16 emulation of the reference's fp32 nn.Linear / bmm; passes=1: hi planes only.
 * Replaces nn.Linear / F.linear / @ on the PatchEncoder, ViT blocks and upscaling MLP
 * (common.py:486-497, pc_encoder.py:99-116,136-143, timm EvaBlock, mask_decoder.py:53-59). */
int psam_gemm_bf16x3(const psam_operand* a, const psam_operand* w, const psam_gemm_out* out, int passes, int split_k,
                     cudaStream_t stream);

/* Row-complete GEMM with LayerNorm and activation in the epilogue:
 *   Y = act(LayerNorm(A W^T + gbias[row / group_rows])) as split-bf16, A [M,K<=128], W [N,K] with N = 256 or 512 (a CTA owns
 * 128 rows x the full width, so the row statistics stay in registers and the fp32 pre-activation never reaches memory).
 * Replaces conv2[0..2] of PatchEncoder (Linear on cat[max, x] = W_a max + W_b x, LayerNorm, GELU; common.py:491-495):
 * gbias carries W_a max + b per group.  gamma / beta [N]; out_hi [M, ldo_s] hi plane, lo plane out_plane elements further. */
int psam_gemm_rowln_bf16x3(const psam_operand* a, const psam_operand* w, const float* gbias, long long ld_gbias, int group_rows,
                           const float* gamma, const float* beta, float eps, int act, void* out_hi, long long out_plane,
                           long long ldo_s, int passes, cudaStream_t stream);

/* Fused encoder self-attention on tensor cores: out = softmax(Q K^T * scale) V per (cloud, head).
 * q/k/v are split-bf16 operand views [L rows x dh] with nb1 = heads, nb2 = clouds (typically three column windows of
 * the fused qkv activation).  dh == 64 or 88 (EVA-giant; the 88-wide head is handled as 64 + 24 columns, zero padded by
 * TMA), any L >= 1 (PSAM_ERR_UNSUPPORTED otherwise - the caller then uses
 * psam_gemm_bf16x3 + psam_softmax_split).  k and v must have q's rows, k, nb1 and nb2, and scale must be finite and > 0
 * (PSAM_ERR_ARG otherwise).  Key blocks are streamed once: S_j = Q K_j^T stays in registers, the running row
 * maximum rescales O and the row sum when it grows, and P_j (split-bf16, in registers) is the A operand of the PV wgmma.
 * Replaces F.scaled_dot_product_attention in timm EvaAttention (blocks called at pc_encoder.py:138-139). */
int psam_attention_bf16x3(const psam_operand* q, const psam_operand* k, const psam_operand* v, void* out_hi,
                          long long out_plane, long long ldo, long long out_head_stride, long long out_cloud_stride,
                          float scale, cudaStream_t stream);

/* Same contract for dh == 64, with an exact two-pass softmax: a first sweep over the key blocks computes the row maximum,
 * the second exponentiates with it (nothing is rescaled).  The tests cross-check the streaming form against it. */
int psam_attention_bf16x3_twopass(const psam_operand* q, const psam_operand* k, const psam_operand* v, void* out_hi,
                                  long long out_plane, long long ldo, long long out_head_stride,
                                  long long out_cloud_stride, float scale, cudaStream_t stream);

/* y = split-bf16(x (+ add)) with zero fill up to `pitch` (add may be NULL; same row stride as x). */
int psam_split_add_f32(const float* x, const float* add, long long ld, long long rows, int D, void* y_hi, long long y_plane,
                       long long ldy_s, long long pitch, cudaStream_t stream);

/* Small fp32 SIMT linear for the prompt decoder (rows < one MMA tile):
 * Y[z][M,N] = act((X[z] (+X2[z]))[M,K] * W[z][N,K]^T + b[z]) (+R[z]); strides in elements; any pointer
 * stride may be 0 to broadcast.  Replaces nn.Linear in transformer.py:199-202,239-253 and the MLP
 * heads mask_decoder.py:189-211. */
typedef struct {
    const float* x;  long long ldx, x_z;
    const float* x2; long long x2_z;      /* optional addend with the geometry of x */
    const float* w;  long long ldw, w_z;
    const float* b;  long long b_z;       /* optional */
    const float* r;  long long r_z;       /* optional residual with the geometry of y */
    float* y;        long long ldy, y_z;
    int M, N, K, Z, act;
} psam_linear_args;
int psam_linear_f32(const psam_linear_args* args, cudaStream_t stream);

/* ---- normalisation / activation / glue -------------------------------------------------------- */

/* y = LayerNorm(x (+ r) (+ gbias[row / group_rows])) * gamma + beta, optional GELU afterwards; writes
 * fp32 and/or split-bf16 (columns D..pitch of the split output are zero-filled).
 * Replaces apex FusedLayerNorm / nn.LayerNorm (+nn.GELU) (torch_utils.py:28-38, common.py:487-495,
 * transformer.py norms, timm norm1/norm2/fc_norm). */
typedef struct {
    const float* x; long long ldx;
    const float* r; long long ldr;            /* optional residual */
    const float* gbias; long long ld_gbias; int group_rows; /* optional per-group row addend */
    const float* gamma; const float* beta; float eps;
    int rows, D, act;
    float* y; long long ldy;                  /* optional */
    void* y_hi; long long y_plane, ldy_s, pitch; /* optional split output */
    int padded;                               /* 1: x rows (zeros), gamma, beta and outputs are valid up to roundup4(D) */
    int policy;                               /* 0: lowest latency (CTA per row for short token streams); 1: least SM-time
                                               * (warp per row, no block barriers) - used when several clouds are in flight */
    const float* post_add; long long ld_post; /* optional: a SECOND split-bf16 output y2 = split(y + post_add[row]) - the     */
    void* y2_hi; long long y2_plane, ldy2_s;  /* "keys + positional encoding" operand of the decoder's projections         */
} psam_ln_args;
int psam_layernorm_f32(const psam_ln_args* args, cudaStream_t stream);

/* SwiGLU with inner LayerNorm (timm SwiGLU, scale_mlp=True): h = silu(g)*x, y = LN(h); gx holds g in
 * columns [0,H) and x in columns [x_off, x_off+H).  Output split-bf16, zero padded to pitch. */
int psam_swiglu_ln(const float* gx, long long ld, long long x_off, int rows, int H, const float* gamma,
                   const float* beta, float eps, void* y_hi, long long y_plane, long long ldy_s, long long pitch,
                   cudaStream_t stream);

/* First layer of the mini-PointNet / positional MLP: y = act(LN?(x[rows,Cin] * W[Cout,Cin]^T + b)),
 * Cin <= 16, Cout in {32, 64, 128, 256, 512} (another multiple of 32 -> PSAM_ERR_UNSUPPORTED); split-bf16 output.  Replaces conv1[0..2] of PatchEncoder
 * (common.py:486-489) and pos_embed[0..1] (pc_encoder.py:102-104). */
int psam_small_in_linear(const float* x, int rows, int Cin, const float* W, const float* b, const float* gamma,
                         const float* beta, float eps, int use_ln, int act, int Cout, void* y_hi, long long y_plane,
                         long long ldy_s, cudaStream_t stream);

/* Max over the K rows of each group: x [groups*K, D] -> y [groups, D] fp32 (optional) and split-bf16
 * (optional).  Replaces torch.max(x, dim=-2) (common.py:501,505). */
int psam_group_max(const float* x, long long ldx, int groups, int K, int D, float* y, long long ldy, void* y_hi,
                   long long y_plane, long long ldy_s, cudaStream_t stream);

/* Row softmax of fp32 scores with scale, split-bf16 output (attention probabilities). */
int psam_softmax_split(const float* s, long long lds, long long rows, int L, float scale, void* p_hi,
                       long long p_plane, long long ldp, cudaStream_t stream);

/* Transposed copy of a split-bf16 matrix block per batch: dst[z][c][r] = src[z][r][c] (both planes). */
int psam_transpose_split(const void* src_hi, long long src_plane, long long src_ld, long long src_z1,
                         long long src_z2, void* dst_hi, long long dst_plane, long long dst_ld, long long dst_z1,
                         long long dst_z2, int rows, int cols, int nz1, int nz2, cudaStream_t stream);

/* Random-Fourier positional encoding (+ optional prompt-label embedding):
 * out[r,:] = [sin(2*pi*c@G), cos(2*pi*c@G)] (+ emb[label[r]]).  Also raises the out-of-range flag
 * (*bad_flag = 1) if any coordinate is outside [-1-1e-6, 1+1e-6] (prompt_encoder.py:44-46).
 * Replaces PositionEmbeddingRandom / PointEncoder (prompt_encoder.py:13-77). labels int32 or NULL. */
int psam_posenc_f32(const float* coords, long long rows, const float* gauss, int F, const int* labels,
                    const float* emb0, const float* emb1, float* out, int* bad_flag, cudaStream_t stream);

/* Multi-head softmax attention for short sequences (fp32, one warp per query):
 * O[z,i,h,:] = softmax(Q[z,i,h,:] . K[z,:,h,:]^T / sqrt(dh)) V[z,:,h,:].  Replaces
 * Attention.forward core (transformer.py:214-233).  dh in {8, 16, 32, 64} and Lk <= 12798 - 2*dh (the scores of four
 * queries stay in shared memory); otherwise PSAM_ERR_UNSUPPORTED. */
int psam_attention_f32(const float* q, const float* k, const float* v, float* o, int Z, int Lq, int Lk, int H, int dh,
                       long long ldq, long long ldk, long long ldv, long long ldo, cudaStream_t stream);

/* Mask-decoder glue (mask_decoder.py:126-139).  With T = 1 + n_mask_tokens + P, for z < Z, g < G, d < D:
 *   tokens[(z*T + t)*D + d] = iou_token[d]                                 (t = 0)
 *                           = mask_tokens[(t-1)*D + d]                     (1 <= t <= n_mask_tokens)
 *                           = sparse[(z*P + t-1-n_mask_tokens)*D + d]      (t > n_mask_tokens)
 *   src[(z*G + g)*D + d]    = pc_emb[((z/rep)*G + g)*D + d] + dense[z*dense_z + g*dense_g + d]   (one fp32 add)
 * i.e. tokens = cat(iou_token, mask_tokens, sparse[z]) and src = repeat_interleave(pc_emb, rep) + dense.  The engine
 * passes dense in three forms: the no-mask embedding [D] broadcast to every (z, g) (dense_z = dense_g = 0), one map per
 * prompt [Z,G,D] (dense_z = G*D, dense_g = D), and one map for all prompts [1,G,D] (dense_z = 0, dense_g = D).
 * sparse may be NULL when P == 0. */
int psam_decoder_prepare(const float* iou_token, const float* mask_tokens, int n_mask_tokens, const float* sparse,
                         int P, const float* pc_emb, const float* dense, long long dense_z, long long dense_g, int Z,
                         int rep, int G, int D, float* tokens, float* src, cudaStream_t stream);

/* 3-NN feature upsampling fused with LayerNorm + GELU: y[z*N+n,:] = GELU(LN(sum_k w[b,n,k]*f[z,idx[b,n,k],:])),
 * b = z/rep; split-bf16 output.  Replaces interpolate_features (common.py:258-274) + output_upscaling[1..2]
 * (mask_decoder.py:55-56) after output_upscaling[0] has been applied to the patch features. */
int psam_interp_ln_gelu(const float* f, int Z, int rep, int G, int D, const long long* idx, const float* w, int N,
                        const float* gamma, const float* beta, float eps, void* y_hi, long long y_plane,
                        long long ldy_s, cudaStream_t stream);

/* psam_interp_ln_gelu with a per-cloud row addend before the LayerNorm:
 * y[z*N+n,:] = GELU(LN(sum_k w[b,n,k]*f[z,idx[b,n,k],:] + addend[b,n,:])), b = z/rep, addend fp32 [B,N,D].
 * Replaces the first stage of MaskDecoderHier's upscaling (mask_decoder.py:322-323): interpolate_features to the level-1
 * centres, cat with the tokenizer's level-1 embeddings, output_upscaling2[0..2], where output_upscaling2[0] has been split
 * into its interpolated half (applied to the patch features, f) and its embedding half (applied once per cloud, addend). */
int psam_interp_add_ln_gelu(const float* f, int Z, int rep, int G, int D, const long long* idx, const float* w, int N,
                            const float* addend, const float* gamma, const float* beta, float eps, void* y_hi,
                            long long y_plane, long long ldy_s, cudaStream_t stream);

/* masks[z,c,n] = sum_d hyper[z,c,d] * u[z*N+n,d]  (mask_decoder.py:176). */
int psam_mask_dot(const float* u, long long ldu, const float* hyper, int Z, int C, int N, int D, float* masks,
                  cudaStream_t stream);

/* out[i] = a[i] + b[(((i / chunk) / rep) * chunk + i % chunk) % b_period]  (repeat_interleave-style broadcast,
 * pc_sam/model/common.py:277-284) */
int psam_add_bcast_f32(const float* a, const float* b, long long n, long long chunk, long long rep, long long b_period,
                       float* out, cudaStream_t stream);

/* fp32 [rows,D] (row stride ld) -> split-bf16 planes (weight packing, activations entering a GEMM) */
int psam_split_f32(const float* x, long long ld, long long rows, int D, void* y_hi, long long y_plane,
                   long long ldy_s, long long pitch, cudaStream_t stream);

/* ---- automatic mask generation ("segment everything") ------------------------------------------ */

/* Candidate extraction of a batch of multimask decoder outputs.  Stands in for the filtering stage of segment-anything's
 * SamAutomaticMaskGenerator._process_batch (predicted-IoU filter, stability score, binarisation), restated for point
 * clouds; the caller loops over prompt batches and gives every batch its own `base`.
 * logits [Z, C, N] fp32, iou_preds [Z, C] fp32.  Each logit row is read once (128-bit loads when N % 4 == 0 and the
 * pointer is 16-byte aligned).  Candidate slot s = base + z*C + c receives
 *   bits[s*W .. s*W+W)  the bit-packed mask logit > mask_threshold (point n = bit n%32 of word n/32; words past N zero),
 *   area[s]             the number of set bits (int32),
 *   stability[s]        fp32(count(logit > hi)) / fp32(count(logit > lo)) with IEEE division (0/0 = NaN), where
 *                       hi = mask_threshold + stability_offset and lo = mask_threshold - stability_offset in fp32,
 *   score[s]            iou_preds[z, c] if the candidate survives, -inf if it does not.
 * A candidate survives when all of these hold (SAM's comparisons):
 *   iou > pred_iou_thresh          (only when pred_iou_thresh > 0; a NaN IoU never survives),
 *   stability >= stability_thresh  (only when stability_thresh > 0),
 *   area >= min_area, and area >= 1 (an empty mask is never kept).
 * W >= ceil(N/32).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_candidates_f32(const float* logits, const float* iou_preds, int Z, int C, int N, float mask_threshold,
                             float stability_offset, float pred_iou_thresh, float stability_thresh, int min_area,
                             long long base, int W, uint32_t* bits, int* area, float* stability, float* score,
                             cudaStream_t stream);
/* The same for B clouds in one launch: logits [B * Zc, C, N] and iou_preds [B * Zc, C], where rows b * Zc .. b * Zc + Zc - 1
 * belong to cloud b (the mask decoder's layout for B encoded clouds).  Row z = b * Zc + j, output c goes to slot
 *   b * cloud_stride + base + j * C + c,
 * with the same rules and the same fp32 arithmetic, so every cloud's slots equal psam_mask_candidates_f32 on its own rows.
 * psam_mask_candidates_f32 is the case B = 1, Zc = Z.  B >= 1, Zc >= 1, B * Zc * C < 2^31, and for B > 1
 * cloud_stride >= base + Zc * C (the clouds' blocks do not overlap).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_candidates_batched_f32(const float* logits, const float* iou_preds, int B, int Zc, int C, int N,
                                     float mask_threshold, float stability_offset, float pred_iou_thresh, float stability_thresh,
                                     int min_area, long long base, long long cloud_stride, int W, uint32_t* bits, int* area,
                                     float* stability, float* score, cudaStream_t stream);
/* psam_mask_candidates_batched_f32 on a padded batch: rows have N_max logits (the row stride), of which cloud b's first
 * lengths[b] are its points.  Only those are counted and packed (bits past lengths[b] are 0, so psam_mask_nms_batched stays
 * exact with W = ceil(N_max/32)), and the slots of prompts j >= min(P, lengths[b]) (prompt j owns slots j * C .. j * C + C-1
 * of the cloud's block, counted from the block start, base included) score -inf.  Every cloud's other slots equal
 * psam_mask_candidates_f32 on its own unpadded rows.  P >= 0; the other rules are psam_mask_candidates_batched_f32's.
 * Padded-batch rules as stated at the top of this header. */
int psam_mask_candidates_varlen_f32(const float* logits, const float* iou_preds, const int* lengths, int B, int Zc, int C,
                                    int N_max, int P, float mask_threshold, float stability_offset, float pred_iou_thresh,
                                    float stability_thresh, int min_area, long long base, long long cloud_stride, int W,
                                    uint32_t* bits, int* area, float* stability, float* score, cudaStream_t stream);

/* Greedy mask-IoU non-maximum suppression over K <= 16384 candidate slots of W words each (the output of
 * psam_mask_candidates_f32).  Stands in for the duplicate-removal stage of SamAutomaticMaskGenerator._process_batch /
 * _process_crop (batched_nms on boxes), here on the masks themselves.
 * Candidates are ordered by (score descending, slot index ascending); -inf scores are dropped.  NaN scores are dropped
 * like -inf, and -0.0 ranks equal to +0.0 (the lower slot goes first).  Walking that order, a
 * candidate is kept unless an earlier kept one overlaps it with
 *   fp32(inter) / fp32(area_i + area_j - inter) > nms_thresh,   inter = popcount(bits_i & bits_j),
 * so the result is exact and bit-reproducible.  Three launches (order, pairwise suppression bits, greedy scan) and no
 * host synchronisation: the number of valid candidates stays on the device.
 * Outputs: keep[0 .. *keep_count) = the kept slot indices in score order (keep holds K ints), *keep_count (device int32).
 * bits / area / score may be NULL when K == 0.  workspace: psam_mask_nms_workspace_bytes(K, W) bytes, 16-byte aligned. */
size_t psam_mask_nms_workspace_bytes(int K, int W);
int psam_mask_nms(const uint32_t* bits, const int* area, const float* score, int K, int W, float nms_thresh, int* keep,
                  int* keep_count, void* workspace, cudaStream_t stream);
/* psam_mask_nms on B clouds of K candidate slots each, in the same three launches: bits [B, K, W], area / score [B, K];
 * keep [B, K] holds each cloud's kept slot indices (within the cloud, 0 .. K-1) in score order, keep_count [B] their counts.
 * Each cloud's result equals psam_mask_nms on its own slice: the order, the tie-break and the IoU arithmetic are the same.
 * The order and scan kernels run one CTA per cloud; the pairwise tiles past a cloud's own valid count exit at once.
 * workspace: psam_mask_nms_batched_workspace_bytes(B, K, W) = B * psam_mask_nms_workspace_bytes(K, W) bytes, 16-byte aligned:
 * per cloud a K x ceil(K/64) matrix of 64-bit suppression words plus the order (1.2 MB at K = 3072, about 34 MB at
 * K = 16383).  psam_mask_nms is the case B = 1.  1 <= B <= 65535 (0 bytes outside), 0 <= K <= 16384.
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_mask_nms_batched_workspace_bytes(int B, int K, int W);
int psam_mask_nms_batched(const uint32_t* bits, const int* area, const float* score, int B, int K, int W, float nms_thresh,
                          int* keep, int* keep_count, void* workspace, cudaStream_t stream);

/* Small-region post-processing of the kept masks: segment-anything's SamAutomaticMaskGenerator.postprocess_small_regions /
 * remove_small_regions (min_mask_region_area), restated for a point cloud of N points.
 * Connectivity: nbr [N, k1] int64 is the cloud's kNN graph (psam_knn_f32(xyz, xyz, k1); the generator uses
 * k1 = min(9, N), the analogue of 8-connectivity).  {i, j} is an edge when j = nbr[i, t] for some t and i != j (undirected);
 * an entry outside 0..N-1 is no edge.  Only edges with both ends in the working set count (the induced subgraph).
 * For every kept rank p < *keep_count (read on the device), on the mask m = bits[keep[p]]:
 *   1. holes:   working set = the points n < N outside m; every component of fewer than min_area points joins m.
 *               changed_h = at least one did.
 *   2. islands: working set = m (after step 1).  If some component has fewer than min_area points (changed_i), m keeps
 *               its components of >= min_area points, or, when none reaches min_area, only the largest one (on equal
 *               sizes the one whose smallest point index is lowest).
 * Outputs by rank p (so they feed psam_mask_nms directly): bits_out[p*W .. p*W+W) the new mask (bits past N and words past
 * ceil(N/32) zero), area_out[p] its point count, score_out[p] = 1 if neither step changed the mask, 0 otherwise (SAM's
 * rescoring); ranks p >= *keep_count get score_out[p] = -inf and nothing else.  A non-empty mask stays non-empty.
 * The result is exact and independent of scheduling: every decision is made on exact integer counts of unique components.
 * bits [K', W] (W >= ceil(N/32)) and keep [K] are the outputs of psam_mask_candidates_f32 / psam_mask_nms, K <= 16384,
 * 1 <= N <= 1048576, 1 <= k1 <= N, min_area >= 1.  bits / keep / outputs may be NULL when K == 0.
 * workspace: psam_mask_regions_workspace_bytes(K, N) bytes, 16-byte aligned.  Labels of up to 49152 points live in shared
 * memory (16 bytes); beyond that the workspace holds one 4N-byte label slice per CTA, min(K, 132, 24 MiB / 4N) slices
 * (at least one), rounded up to 16 bytes.
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_mask_regions_workspace_bytes(int K, int N);
int psam_mask_regions(const uint32_t* bits, int K, int W, int N, const int* keep, const int* keep_count, const long long* nbr,
                      int k1, int min_area, uint32_t* bits_out, int* area_out, float* score_out, void* workspace,
                      cudaStream_t stream);
/* psam_mask_regions on B clouds of N points in one launch of persistent CTAs over the B * K (cloud, rank) items.  Cloud b's
 * candidate masks start at bits + b * cloud_slots * W (its keep entries index them), its kNN graph is nbr[b] of nbr
 * [B, N, k1], its keep list keep[b] of keep [B, K] and its count keep_count[b]; its outputs are row b of bits_out [B, K, W],
 * area_out [B, K] and score_out [B, K] (score -inf past the cloud's count).  Each cloud's result equals psam_mask_regions
 * on its own slice.  The label slices of the workspace form are shared by all items of the launch, so the workspace does not
 * grow with B beyond its cap: psam_mask_regions_batched_workspace_bytes(B, K, N) is psam_mask_regions_workspace_bytes' formula
 * with min(B * K, 132, 24 MiB / 4N) slices.  psam_mask_regions is the case B = 1 (cloud_slots unused).  B >= 1,
 * cloud_slots >= 1 when B > 1.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_mask_regions_batched_workspace_bytes(int B, int K, int N);
int psam_mask_regions_batched(const uint32_t* bits, long long cloud_slots, int B, int K, int W, int N, const int* keep,
                              const int* keep_count, const long long* nbr, int k1, int min_area, uint32_t* bits_out,
                              int* area_out, float* score_out, void* workspace, cudaStream_t stream);
/* psam_mask_regions_batched on a padded batch: cloud b's working sets (holes, then islands) hold only its points
 * n < lengths[b], so padding never forms a component; nbr [B, N_max, k1] is psam_knn_varlen_f32's graph (the generator uses
 * k1 = min(9, lengths[b]) for every cloud).  Each cloud's outputs equal psam_mask_regions on its own cloud; bits past
 * lengths[b] are 0.  Workspace: psam_mask_regions_batched_workspace_bytes(B, K, N_max).
 * Padded-batch rules as stated at the top of this header. */
int psam_mask_regions_varlen(const uint32_t* bits, long long cloud_slots, const int* lengths, int B, int K, int W, int N_max,
                             const int* keep, const int* keep_count, const long long* nbr, int k1, int min_area,
                             uint32_t* bits_out, int* area_out, float* score_out, void* workspace, cudaStream_t stream);

/* ---- crop layers of automatic mask generation (SAM's crop_n_layers) ------------------------------ */
/* Layout.  Layer 0 is the whole cloud.  Layer i >= 1 splits every axis a of the cloud's axis-aligned bounding box
 * [lo_a, hi_a] into n = 2^i crops.  Everything is fp32, every operation rounded on its own (no contraction), in this order:
 *   lo_a = min_n xyz[n, a], hi_a = max_n xyz[n, a]          (exact; NaN coordinates are ignored, and an axis with
 *                                                              nothing but NaN gives lo_a = +inf, hi_a = -inf; -0.0
 *                                                              orders below +0.0, so lo_a = -0.0 when the axis's smallest
 *                                                              value is zero and one of its zeros is -0.0, and hi_a = +0.0
 *                                                              when its largest is zero and one of its zeros is +0.0)
 *   L_a  = hi_a - lo_a
 *   o_a  = ((r * L_a) * 2) / n                                r = overlap_ratio
 *   s_a  = (L_a + o_a * (n - 1)) / n
 *   crop j of the axis: [lo_a + j * (s_a - o_a), lo_a + j * (s_a - o_a) + s_a], except that the last crop's upper bound is
 *   exactly hi_a (layer 0: [lo_a + 0 * (L_a - o_a), hi_a]).
 * Crops are numbered layer by layer (layer 0 first), and within layer i as (jx * n + jy) * n + jz, so there are
 * psam_crop_total(n_layers) = sum_{i <= n_layers} 8^i of them.  boxes[t*6 .. t*6+6) = (x0, y0, z0, x1, y1, z1).
 * Point n is in crop t when x0 <= x <= x1, y0 <= y <= y1 and z0 <= z <= z1 (closed; a NaN coordinate is in no crop).
 * counts[t] = the number of points in crop t, or -1 when an earlier crop of the same layer has an identical box (a
 * duplicate; it happens on zero-extent axes).
 * 1 <= N, 0 <= n_layers <= 3, 0 <= overlap_ratio < 1.  Two launches (one CTA for the box and the layout, then a grid for
 * the counts).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_crop_total(int n_layers); /* 0 when n_layers is outside 0..3 */
int psam_crop_layout_f32(const float* xyz, int N, int n_layers, float overlap_ratio, float* boxes, int* counts,
                         cudaStream_t stream);

/* Crop gather: the crop cloud of crop `crop` (0 <= crop < n_crops) of psam_crop_layout_f32's boxes, whose n_out points
 * (its count) come out in ascending global index:
 *   idx_out[k]       the global index of the crop's k-th point (int32),
 *   xyz_out[k*3+a]   (p_a - c_a) / scale, where c_a = (x0_a + x1_a) * 0.5 is the box midpoint and scale = sqrt(max_k d2_k),
 *                    d2 = (dx*dx + dy*dy) + dz*dz with dx = p_x - c_x etc.; every coordinate is 0 when scale is 0, and
 *                    |xyz_out| <= 1 otherwise (IEEE division and square root),
 *   rgb_out[k*3+a]   rgb unchanged,
 *   edge[k/32] bit k%32   the point is within m_a = edge_margin * L_a (L_a = x1_a - x0_a of crop 0, the bounding box) of an
 *                    interior face of the crop: (x0_a != lo_a and p_a - x0_a <= m_a) or (x1_a != hi_a and x1_a - p_a <= m_a)
 *                    on some axis a; words up to ceil(n_out / 32) are written (bits past n_out zero).
 * The compaction is stable and the same on every run.  Two launches.  workspace: psam_crop_gather_workspace_bytes(N)
 * bytes, 16-byte aligned.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_crop_gather_workspace_bytes(int N);
int psam_crop_gather_f32(const float* xyz, const float* rgb, int N, const float* boxes, int crop, int n_crops, float edge_margin,
                         int n_out, int* idx_out, float* xyz_out, float* rgb_out, uint32_t* edge, void* workspace,
                         cudaStream_t stream);

/* Edge filter (SAM's is_box_near_crop_edge, on masks): score[k] = -inf for every candidate k < K whose mask bits[k*W ..)
 * shares a point with edge[0 .. W) (the crop's edge bitset).  Run between psam_mask_candidates_f32 and psam_mask_nms.
 * bits / edge / score may be NULL when K == 0.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_crop_edge_filter(const uint32_t* bits, int K, int W, const uint32_t* edge, float* score, cudaStream_t stream);

/* Uncrop: append a crop's kept masks to the global set.  For every kept rank p < *keep_count (read on the device), with
 * s = keep[p], z = s / slots and d = *offset_in + p < capacity:
 *   gbits[d*Wg .. d*Wg+Wg)  the mask bits[s*W ..) of the crop's n points lifted to the cloud's N points (local point k is
 *                           global point idx[k]; every other bit zero),
 *   garea[d] = area[s], giou[d] = score[s], gstab[d] = stability[s], gprompt[d] = idx[prompt_index[z]] (int64),
 *   gslot[d] = s - z * slots, gcrop[d] = crop, gscore[d] = layer_score.
 * *offset_out = *offset_in + *keep_count (offset_out must not alias offset_in: the caller keeps one entry per crop), and
 * *overflow = 1 when that exceeds capacity; ranks at or past capacity are not written.
 * 1 <= n <= N, W >= ceil(n/32), Wg >= ceil(N/32), 1 <= capacity <= 16384, K >= 1 = the length of keep.
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_crop_uncrop(const uint32_t* bits, const int* area, const float* score, const float* stability, int K, int W,
                     const int* keep, const int* keep_count, const int* idx, int n, const long long* prompt_index, int slots,
                     int crop, float layer_score, int N, int Wg, int capacity, const int* offset_in, int* offset_out,
                     uint32_t* gbits, int* garea, float* giou, float* gstab, long long* gprompt, int* gslot, int* gcrop,
                     float* gscore, int* overflow, cudaStream_t stream);

/* Crop layers on a batch of B clouds.  Each entry point below gives every cloud (or crop) the result of its single-cloud
 * counterpart above bit for bit; the single-cloud entry points are the case B = 1 of the same kernels.
 *
 * Batched layout: psam_crop_layout_f32 on each cloud of xyz [B, N_max, 3]: boxes [B, T, 6] and counts [B, T] with
 * T = psam_crop_total(n_layers).  lengths [B] (device int32, NULL: every cloud has N_max points): cloud b is its first
 * clamp(lengths[b], 0, N_max) rows; the rows past it are never read, so they touch neither its bounding box nor any count
 * whatever they hold (NaN included).  1 <= B <= 65535.  Two launches.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_crop_layout_batched_f32(const float* xyz, const int* lengths, int B, int N_max, int n_layers, float overlap_ratio,
                                 float* boxes, int* counts, cudaStream_t stream);
/* Batched gather: P (cloud, crop) pairs of the batched layout into one padded batch of crop clouds.  pairs [3, P] (device
 * int32): row 0 the clouds (0 .. B-1), row 1 the crops (0 .. n_crops-1), row 2 the counts (the layout's count of that crop,
 * 0 .. n_max).  xyz / rgb [B, N_max, 3] and lengths as for the layout; boxes [B, n_crops, 6].  Outputs: idx_out [P, n_max],
 * xyz_out / rgb_out [P, n_max, 3] and edge [P, ceil(n_max / 32)]; row p's first counts[p] entries equal
 * psam_crop_gather_f32(cloud's points, crop, n_out = counts[p]) bit for bit (same stable compaction, the edge margin from
 * the cloud's own bounding box), its later rows are 0 and its edge bits past counts[p] are 0.  A pair outside these ranges
 * gathers nothing (all its rows 0).  1 <= P <= 65535, 1 <= n_max <= N_max.  Two launches.  workspace:
 * psam_crop_gather_batched_workspace_bytes(P, N_max) bytes, 16-byte aligned.  Bad arguments -> PSAM_ERR_ARG before any CUDA
 * call. */
size_t psam_crop_gather_batched_workspace_bytes(int P, int N_max);
int psam_crop_gather_batched_f32(const float* xyz, const float* rgb, const int* lengths, int B, int N_max, const float* boxes,
                                 int n_crops, const int* pairs, int P, int n_max, float edge_margin, int* idx_out, float* xyz_out,
                                 float* rgb_out, uint32_t* edge, void* workspace, cudaStream_t stream);
/* Batched edge filter: psam_crop_edge_filter on each crop t < T of bits [T, K, W], edge [T, W] and score [T, K], one launch.
 * 1 <= T <= 65535; bits / edge / score may be NULL when K == 0.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_crop_edge_filter_batched(const uint32_t* bits, int T, int K, int W, const uint32_t* edge, float* score,
                                  cudaStream_t stream);
/* Batched uncrop: psam_crop_uncrop for R crop runs of B clouds in one launch.  runs[R] (device memory) describes each run
 * with the arguments of psam_crop_uncrop (its candidates, keep list of K entries, kept count, crop point indices idx of its
 * n points, prompt indices, slots, crop number and layer score), its cloud, and the cloud's capacity (<= cloud_rows).
 * The runs of one cloud are consecutive and in that cloud's crop order; `first` is the index of its cloud's first run and
 * `last` is 1 for its cloud's last run.  Run r's masks go to cloud c's rows of gbits [B, cloud_rows, Wg] and of the per-mask
 * outputs [B, cloud_rows], starting at the exclusive prefix (in run order) of the kept counts of the cloud's earlier runs,
 * computed on the device: the result equals psam_crop_uncrop over the cloud's runs in order.  The cloud's last run writes
 * lifted[c] (the total kept count) and overflow[c] (1 when that exceeds the capacity, else 0); no other CTA writes them.
 * Every cloud needs at least one run.  1 <= R <= 65535, K_max >= every run's K, Wg >= ceil(N_max / 32) with every run's
 * idx < N_max, 1 <= cloud_rows <= 16384.  Bad arguments -> PSAM_ERR_ARG before any CUDA call.
 * psam_crop_run_bytes() = sizeof(psam_crop_run), for bindings that lay the table out themselves. */
typedef struct psam_crop_run {
    const uint32_t* bits;           /* [K', W] candidates */
    const int* area;
    const float* score;
    const float* stability;
    const int* keep;                /* [K] kept slots */
    const int* keep_count;          /* [1] */
    const int* idx;                 /* [n] the crop's point indices in its cloud */
    const long long* prompt_index;  /* crop-local prompt indices */
    int K, W, n, slots, crop, cloud, first, last;
    float layer_score;
    int capacity;
} psam_crop_run;
size_t psam_crop_run_bytes(void);
int psam_crop_uncrop_batched(const psam_crop_run* runs, int R, int K_max, int B, int N_max, int Wg, int cloud_rows, uint32_t* gbits,
                             int* garea, float* giou, float* gstab, long long* gprompt, int* gslot, int* gcrop, float* gscore,
                             int* lifted, int* overflow, cudaStream_t stream);

/* ---- meshes and dense clouds ---------------------------------------------------------------------- */
/* Area-weighted surface sampling of a triangle mesh: vertices [V, 3] fp32, faces [F, 3] int32 -> S samples xyz_out [S, 3],
 * rgb_out [S, 3] and face_out [S] (int32, the face each sample lies on).  Everything is fp32, every operation rounded on its
 * own (no contraction), in this order, unless stated otherwise:
 *   weight  e1 = b - a, e2 = c - a (a, b, c = the face's vertices), n = (e1y*e2z - e1z*e2y, e1z*e2x - e1x*e2z,
 *           e1x*e2y - e1y*e2x), A2 = sqrt((nx*nx + ny*ny) + nz*nz) (twice the area).  A face with an index outside [0, V),
 *           or whose A2 is not finite or <= 0, has weight 0 (a "bad" face).  With A2max in [2^(E-1), 2^E) the largest A2 of
 *           the good faces, the weight is the integer q_f = floor(A2_f * 2^(32 - E)) (computed in fp64, where it is exact),
 *           so q_f <= 2^32 - 1, and a face smaller than 2^-32 of the largest has weight 0 and is never sampled.
 *   cdf     cdf[f] = q_0 + ... + q_f, an exact uint64 prefix sum; total = cdf[F - 1].
 *   hash    h_j(s) = splitmix64 finaliser of seed + (3*s + j + 1) * 0x9E3779B97F4A7C15 (mod 2^64), streams j = 0, 1, 2 of
 *           sample s: z ^= z >> 30, z *= 0xBF58476D1CE4E5B9, z ^= z >> 27, z *= 0x94D049BB133111EB, z ^= z >> 31.  There is no
 *           generator state, so the samples do not depend on the launch configuration.
 *   face    u = mulhi64(h_0, total) (the high 64 bits of the 128-bit product); the face is the smallest f with cdf[f] > u, so
 *           a face is chosen with probability q_f / total and a weight-0 face never.
 *   point   r1 = (h_1 >> 40) * 2^-24, r2 = (h_2 >> 40) * 2^-24 (exact), v = sqrt(r1), w = (1 - v, v * (1 - r2), v * r2);
 *           p = (w0 * a + w1 * b) + w2 * c, then each axis clamped to [min, max] of the three vertices' coordinates (so the
 *           samples of a mesh inside [-1, 1] stay inside it): min(max(p, min(min(a, b), c)), max(max(a, b), c)), where
 *           min and max ignore a NaN operand and order -0.0 below +0.0 (so a p of either sign of zero inside the box is
 *           kept as it is).
 *   colour  with texture [tex_h, tex_w, tex_c] uint8 (tex_c = 3 or 4) and uv [V, 2]: (tu, tv) = the uv interpolated like p
 *           (not clamped), texel x = floor(tu * tex_w + 0.5), y = floor((1 - tv) * tex_h + 0.5), each clamped into the image
 *           (a NaN gives 0); the colour is its first three channels / 255.  Otherwise with vertex_colors [V, 3]: interpolated
 *           and clamped like p.  With neither: 0.5.  texture and vertex_colors are exclusive; uv goes with texture.
 * stats (device int64 [3]): stats[0] = total weight, stats[1] = bad faces, stats[2] = faces with an index outside [0, V)
 * (counted among the bad faces).  When the total weight is 0 every sample gets face -1, xyz 0 and rgb 0.
 * Five launches (areas, three for the scan, samples) and two memsets, no host synchronisation.  1 <= V, 1 <= F < 2^31,
 * 1 <= S.  workspace: psam_mesh_sample_workspace_bytes(F) bytes, 16-byte aligned.  Bad arguments -> PSAM_ERR_ARG before any
 * CUDA call. */
size_t psam_mesh_sample_workspace_bytes(int F);
int psam_mesh_sample_f32(const float* vertices, int V, const int* faces, int F, int S, unsigned long long seed,
                         const float* vertex_colors, const float* uv, const unsigned char* texture, int tex_h, int tex_w, int tex_c,
                         float* xyz_out, float* rgb_out, int* face_out, long long* stats, void* workspace, cudaStream_t stream);

/* centers[f] = ((a + b) + c) / 3 per axis in fp32 (IEEE division), NaN for a face with an index outside [0, V): the query
 * points that carry masks to faces (psam_nn_distance_f32 gives such a query no nearest sample, index -1).
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mesh_face_centers_f32(const float* vertices, int V, const int* faces, int F, float* centers, cudaStream_t stream);

/* Mask lifting: masks over S points carried to M other points through their nearest point.  bits [K, Ws] (bit-packed as in
 * psam_mask_candidates_f32, Ws >= ceil(S/32)), nearest [M] int64 -> bits_out [K, Wm] (Wm >= ceil(M/32)): bit t of row k is
 * bit nearest[t] of row k of bits; an entry outside [0, S) reads as 0, and bits past M and words past ceil(M/32) are 0.
 * area_out[k] = the number of set bits of row k of bits_out (exact).  Two launches: one warp per 4 output words, each lane
 * holding its nearest index across all K rows, then one warp per row for the areas.  K = 0 is a no-op (pointers may be
 * NULL).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_lift(const uint32_t* bits, int K, int Ws, int S, const long long* nearest, int M, int Wm, uint32_t* bits_out,
                   int* area_out, cudaStream_t stream);

/* Part labels: labels[n] = the row k of bits [K, W] (W >= ceil(N/32)) that contains point n with the smallest priority[k]
 * (int32), ties to the lower k; -1 when no row contains it.  With priority = area the smallest mask containing a point wins,
 * which is the order in which segment-anything's show_anns paints (largest first, so the smallest ends on top).  K = 0 gives
 * -1 everywhere.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_label_map(const uint32_t* bits, int K, int W, const int* priority, int N, int* labels, cudaStream_t stream);

/* ---- dense scans ---------------------------------------------------------------------------------- */
/* Exact nearest key on a uniform grid: query [n1, 3], key [n2, 3] -> dist_out [n1] fp32 and idx_out [n1] int64 (may be NULL),
 * bit for bit what psam_nn_distance_f32 writes for every input:
 *   d(j) = fma(dz, dz, fma(dy, dy, dx * dx)) with dx = key_x - query_x etc. (each step rounded once);
 *   the result is the lexicographic minimum of (d(j), j) over the keys with d(j) < 3.4e38f, or (3.4e38f, -1) when there is
 *   none: so a query with a non-finite coordinate, or whose every distance overflows or is NaN, gets index -1, and a key with
 *   a non-finite coordinate is never chosen.  Candidates are compared as (d, j) pairs, so the order of the visits is free.
 * Evaluation order (each call builds the grid afresh over the finite keys, a counting sort):
 *   box      klo_a / hi_a = min / max of the finite keys' coordinates (exact), F = the number of finite keys, and a
 *            1024-bin histogram of them on each axis over [klo_a, hi_a].
 *   grid     its box on axis a runs from lo_a = max(klo_a, b5 - w / 10) to min(hi_a, b95 + w / 10), where b5 is the lower edge
 *            of the bin holding the key of rank F / 20, b95 the upper edge of the bin holding rank F - 1 - F / 20 and
 *            w = b95 - b5, so far outliers do not stretch it; T = min(F, 2^22) target cells; cubic cells of side h, with
 *            dims_a = min(floor(ext_a / h) + 1, 2^21) cells on axis a (ext_a = the box's extent, fp64) and h the (fp64
 *            bisection) smallest found with dims_x dims_y dims_z <= T; one cell of side 1 when every ext_a is 0.  Keys
 *            outside the box land in its border cells (the clamp below).  The box, h and the dims decide only the speed.
 *   cell     c_a(p) = clamp(floor((p_a - lo_a) * (1 / h)), 0, dims_a - 1) in fp64, cell id (c_x dims_y + c_y) dims_z + c_z;
 *            a histogram (the rank of a key in its cell comes from the counting atomic), an exclusive scan of the counts
 *            and a scatter of (x, y, z, j) into cell order (the order inside a cell is free).
 *   search   every query visits the rings r = 0, 1, ... of cells at Chebyshev index distance r from its clamped cell c(q),
 *            each grid row along z as one contiguous run, and after ring r stops when a lower bound LB on the squared
 *            distance to every key in an unvisited cell satisfies LB' = LB (1 - 2^-20) - 2^-140 > best d (fp64 compare),
 *            or LB' >= 3.4e38, or no cell is left.
 * The lower bound and its margin.  Unvisited cells lie beyond one of the six faces of the visited block (cells c(q)_a - r ..
 * c(q)_a + r); for the face on axis a at f = lo_a + k h, LB = max(t^2, o_a^2) + sum_{b != a} o_b^2, where o_b = the distance
 * from q_b to [klo_b, hi_b] (every finite key lies in that box) and t = max(|q_a - f| - s_a, 0) on the face's far side.
 * The slop s_a = 2^-40 (|lo_a| + |klo_a| + |hi_a| + |q_a| + (dims_a + 1) h) covers the fp64 rounding of the cell coordinates
 * and of f: a key in cell k >= 1 has (p_a - lo_a)(1 + e1)(1 / h)(1 + e2) >= k with |e1|, |e2| <= 2^-53, so p_a >= f - 2^-50 k h,
 * and likewise below.  The clamp into the border cells only moves a key into a cell on the same side of every face, so
 * the bound holds for clamped keys too.  Then, for every unvisited key, its true squared distance D >= LB up to the relative fp64
 * rounding of LB (a few 2^-53).  Its computed d is five roundings away from D: the subtractions (exact when the result is
 * subnormal, else relative error <= 2^-24), the product and the two fmas (relative error <= 2^-24, or absolute <= 2^-150
 * where the result is subnormal).  Every step is monotone, so d >= D (1 - 2^-24)^5 - 3 * 2^-150 >= D (1 - 2^-21) - 2^-148;
 * a step that overflows gives inf, which is still >= that bound.  Hence d >= LB' for every unvisited key, and LB' > best d
 * means no unvisited key can win (nor tie with a lower index); LB' >= 3.4e38 means none can be accepted.  A query far
 * outside the keys' box is answered exactly, by visiting more rings.
 * Launches: box, box histograms, setup (one thread), cell histogram, one to three for the scan, scatter, queries (one
 * thread per query, an outward ring search) - up to nine launches after one memset, no host synchronisation.
 * 1 <= n1 <= 2^31 - 1, 1 <= n2 <= 2^31 - 1.  workspace: psam_nn_grid_workspace_bytes(n2), about 12.4 KB + 4 (C + 1) +
 * 8 ceil((C + 1) / 1024) + 24 n2 bytes (each part rounded up to 16 bytes) with C = min(n2, 2^22) cells, 16-byte aligned.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_nn_grid_workspace_bytes(int n2);
int psam_nn_grid_f32(const float* query, int n1, const float* key, int n2, float* dist_out, long long* idx_out, void* workspace,
                     cudaStream_t stream);

/* Voxel subsample of P points xyz [P, 3] (normalised coordinates, fp32) to at most S of them.  A point with a non-finite
 * coordinate is invalid and takes part in nothing.  For a valid point, per axis a:
 *   q_a = clamp(floor(fl(x_a + 1) * 2^20), 0, 2^21 - 1)   (fp32 add, exact multiply, clamp in float, then integer)
 *   level L = 0..21: cell k_a = q_a >> (21 - L), key = (k_x << 42) | (k_y << 21) | k_z,
 *   e = sum_a (2 q_a + 1 - (2 k_a + 1) 2^(21 - L))^2 (exact int64: the squared distance to the cell centre, in units of
 *   2^-21 / 2).
 * n_L = the number of distinct occupied cells at level L (non-decreasing in L).  L* = the smallest L with n_L >= S, or 21.
 * Each occupied cell at L* has one representative, the point of smallest (e, index).  When n_L* > S only the S
 * representatives of smallest (h(key), key) are kept, h(key) = the splitmix64 finaliser of psam_mesh_sample_f32 applied to
 * seed + (key + 1) * 0x9E3779B97F4A7C15 (mod 2^64); h is a bijection of the key, so the order is the order of h.
 * Outputs: idx_out [S] int64 = the kept point indices in ascending order, then -1; stats (device int64 [4]) = (valid points,
 * L*, n_L*, kept = min(S, n_L*)).
 * Method: the level-21 keys; a binary search for L* over 0..21 (five steps, each counting the distinct cells of one level in
 * an open-addressing hash set of 2^ceil(log2(2 P)) slots); the set of level L* with each cell's smallest e (atomicMin) and
 * then its smallest index among the points with that e; the S-th smallest h by an 8-pass radix select; a flag per kept point
 * and a stable compaction.  The result does not depend on the schedule.  34 launches and 10 memsets, no host
 * synchronisation.  1 <= P <= 2^31 - 1, S >= 1.  workspace: psam_voxel_subsample_workspace_bytes(P) bytes, about
 * 25 P + 20 * 2^ceil(log2(2 P)) (0.9 GB at P = 10^7), 16-byte aligned.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
size_t psam_voxel_subsample_workspace_bytes(int P);
int psam_voxel_subsample_f32(const float* xyz, int P, int S, unsigned long long seed, long long* idx_out, long long* stats,
                             void* workspace, cudaStream_t stream);

/* ---- decoder fine-tuning (csrc/train.cu) ------------------------------------------------------------------------------
 * Training of mask_decoder on a frozen encoder: the reference's mask loss (pc_sam/model/loss.py:58-158) and the backward of
 * the per-point mask head (mask_decoder.py:146-176).  No float atomics: every output is bitwise reproducible run to run. */

/* Per (row z, mask c) statistics of compute_mask_loss over logits [Z,C,N] fp32 and gt [Z,N] (bytes, nonzero = inside):
 * stats[z,c,:] = (sum_n focal, sum_n p t, sum_n p^2, sum_n t) with p = sigmoid(logit), focal = torchvision's
 * sigmoid_focal_loss(alpha=-1, gamma=2) = BCE-with-logits * (1 - p_t)^2; counts[z,c,:] = (|pred & gt|, |pred | gt|) with
 * pred = logit > 0 (compute_iou).  Every element and sum in fp64, stored as fp32 / int32.  One CTA per (z, c).
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_loss_stats(const float* logits, const unsigned char* gt, int Z, int C, int N, float* stats, int* counts,
                         cudaStream_t stream);

/* dlogits[z,c,n] = dloss[z,c] * d(focal_mean + 2 dice)[z,c] / dlogit[z,c,n], dice = 1 - (2 sum p t + 1e-3) / (sum p^2 + sum t
 * + 1e-3), from psam_mask_loss_stats' stats.  A (z, c) with dloss == 0 (a mask the criterion did not select) is written as
 * zeros without evaluating its terms.  Z * C <= 65535.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_mask_loss_grad(const float* logits, const unsigned char* gt, int Z, int C, int N, const float* stats, const float* dloss,
                        float* dlogits, cudaStream_t stream);

/* Inverse of the 3-NN interpolation index idx [B,N,3] (int64, values in [0, G); psam_knn3_interp_f32): per cloud b,
 * offsets[b, g] .. offsets[b, g+1] (int32 [B, G+1]) delimit the entries e = n * 3 + k with idx[b,n,k] == g in entries
 * (int32 [B, 3N]), in ascending e.  One CTA per cloud; a stable counting sort.  G <= 8192.  Bad arguments -> PSAM_ERR_ARG
 * before any CUDA call. */
int psam_interp_inverse(const long long* idx, int B, int N, int G, int* offsets, int* entries, cudaStream_t stream);

/* Head backward, elementwise part.  p [Z*N, D] = output_upscaling[3] pre-activation (fp32), dm [Z,C,N] the gradient of the
 * masks, hyper [Z,C,D]:  dp[z*N+n, d] = GELU'(p) * sum_c dm[z,c,n] hyper[z,c,d] as split-bf16 (row stride ldp_s, lo plane
 * dp_plane elements after the hi plane), and partial sums over chunks of 128 points (K = psam_head_dp_chunks(N) chunks):
 * part_hyper [Z, K, C, D] of dm * GELU(p) (-> dhyper) and part_b3 [Z, K, D] of dp (-> the bias gradient); psam_sum_partials
 * finishes both.  C <= 8, D a multiple of 32 <= 1024, Z <= 65535.  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_head_dp(const float* p, const float* dm, const float* hyper, int Z, int C, int N, int D, void* dp_hi, long long dp_plane,
                 long long ldp_s, float* part_hyper, float* part_b3, cudaStream_t stream);
int psam_head_dp_chunks(int N);

/* Backward of psam_interp_ln_gelu: du [Z*N, D] holds dL/dy on entry and dL/dv on return (in place), v = the interpolated
 * row before the LayerNorm; the interpolation and LayerNorm are recomputed with the forward's arithmetic.  part
 * [ceil(Z*N / rows_per_block), 2, D] receives per-CTA partial sums of dgamma (row 0) and dbeta (row 1), each CTA covering
 * rows_per_block consecutive rows; psam_sum_partials finishes them.  D in {128, 256, 512} (PSAM_ERR_UNSUPPORTED otherwise).
 * Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_interp_ln_gelu_backward(const float* f, int Z, int rep, int G, int D, const long long* idx, const float* w, int N,
                                 const float* gamma, const float* beta, float eps, float* du, float* part, int rows_per_block,
                                 cudaStream_t stream);

/* Backward of the 3-NN interpolation (interpolate_features, common.py:258-274) as a gather: df[z*G+g, :] = sum over the
 * entries e of patch g of cloud b = z / rep (psam_interp_inverse, in its order) of w[b, e] * dv[z*N + e/3, :].  D a multiple of
 * 128 <= 1024 (PSAM_ERR_UNSUPPORTED otherwise).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_interp_backward(const float* dv, int Z, int rep, int G, int D, const int* offsets, const int* entries, const float* w, int N,
                         float* df, cudaStream_t stream);

/* out[b*n + i] = sum_{s < S} part[(b*S + s)*n + i], in order s = 0, 1, ... with an fp64 accumulator: the fixed-order finish of
 * every partial-sum buffer above (and of split-K GEMM partials).  Bad arguments -> PSAM_ERR_ARG before any CUDA call. */
int psam_sum_partials(const float* part, int nb, int S, long long n, float* out, cudaStream_t stream);

const char* psam_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PSAM_B200_H */
