// Farthest-point sampling for sm_90a.
//
// Replaces torkit3d's sample_farthest_points_cuda
// (third_party/torkit3d/torkit3d/csrc/cuda/sample_farthest_points_kernel.cu:8-165) and the
// batch_index_select of the centres that follows it (pc_sam/model/common.py:91-92).
//
// Design: one thread-block CLUSTER per cloud.  The cloud (xyz + running min-distance) lives in the
// registers of the cluster's threads for the whole kernel, so an iteration touches no global memory.
// Per iteration every warp reduces its candidates with redux.sync into one 20-byte record (max-distance
// bits, tie-break priority, xyz of the candidate) and pushes it straight into the shared memory of EVERY
// CTA of the cluster with st.async (DSMEM store that completes transaction bytes on the receiver's
// mbarrier - data and signal in a single hop).  All threads then wait on their local mbarrier and reduce
// the C x 8 records.  No __syncthreads, no barrier.cluster and no second reduction stage inside the loop
// (round 1 combined the warps of a CTA through shared memory first: one block barrier plus a serial
// warp-0 stage per iteration, 0.77 us/iteration at N = 32768).
//
// Bit-exactness: squared distance is fmaf(dz,dz,fmaf(dy,dy,dx*dx)) with d = p_j - p_sel, and among
// equal maxima the winner is the lexicographic minimum of (bitrev(j mod T), j div T), T = the
// reference's block size for this N; if the maximum is 0 the previous index
// is repeated.  Independent of how points are distributed over threads here.
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace psam {

constexpr int FPS_THREADS = 256;
constexpr int FPS_WARPS = FPS_THREADS / 32;
constexpr int FPS_MAX_CLUSTER = 16;
constexpr int FPS_MAX_SLOTS = FPS_MAX_CLUSTER * FPS_WARPS;

__device__ __forceinline__ uint32_t fps_prio(uint32_t j, uint32_t tmask, int log2T) {
    // smaller is better: bit-reversed (j mod T) in the top log2T bits, (j div T) below.
    return __brev(j & tmask) | (j >> log2T);
}

// log2 of the reference's block size T for a cloud of N points: the smallest power of two >= N capped at 512, and 32 below
// 64 (utils.h:13-19, :153-161).  T decides which of several equal maxima wins, so a padded cloud derives it from its own length.
__host__ __device__ __forceinline__ int fps_log2T(int N) {
    int T = 1;
    while (T < N && T < 512) T *= 2;
    if (T < 64) T = 32;
    int l = 0;
    while ((1 << l) < T) ++l;
    return l;
}

__device__ __forceinline__ float fps_sqdist(float x, float y, float z, float cx, float cy, float cz) {
    const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy), dz = __fsub_rn(z, cz);
    return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}

// PPT > 0: register-resident points (PPT per thread).  PPT == 0: streaming fallback for clouds that
// exceed the register capacity of a cluster; min-distance then lives in the global workspace `ws`.
// VARLEN: cloud b is the first lengths[b] of its Ns rows (clamped to [1, Ns]); it derives its own log2T, runs
// min(G, lengths[b]) greedy steps and fills the remaining slots with sample 0.  Otherwise every cloud has Ns points.
template <int PPT, bool VARLEN>
__global__ void __launch_bounds__(FPS_THREADS, 1)
fps_cluster_kernel(const float* __restrict__ xyz, int Ns, int G, int log2T_all, const int* __restrict__ lengths,
                   long long* __restrict__ idx_out, float* __restrict__ centers_out, float* __restrict__ ws) {
    pdl_prologue();
    __shared__ __align__(16) uint4 slot_a[2][FPS_MAX_SLOTS];  // records received from every warp of the cluster {bits, prio, x, y}
    __shared__ float slot_z[2][FPS_MAX_SLOTS];
    __shared__ __align__(8) uint64_t mbar[2];
    extern __shared__ float spts[];  // PPT > 0: this CTA's points, [slot][thread][xyz] - the winning lane fetches its candidate by index

    const uint32_t C = cluster_nctarank();
    const uint32_t rank = cluster_ctarank();
    const int cloud = blockIdx.x / C;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = VARLEN ? min(max(lengths[cloud], 1), Ns) : Ns;
    const int log2T = VARLEN ? fps_log2T(N) : log2T_all;
    const int Gs = VARLEN ? min(G, N) : G;  // greedy steps; slots Gs .. G-1 repeat sample 0
    const uint32_t tmask = (1u << log2T) - 1u;
    const uint32_t qmask = (1u << (32 - log2T)) - 1u;
    const int stride = (int)C * FPS_THREADS;
    const int gt = (int)rank * FPS_THREADS + tid;
    const uint32_t tx_bytes = C * FPS_WARPS * 20u;  // every warp of every peer (incl. this CTA) delivers 16 + 4 bytes per iteration
    // When the thread stride is a multiple of T, (j mod T) is the same for every point of a thread and (j div T) grows with the
    // slot: the tie-break priority is prio0 + slot * kprio, i.e. among equal maxima of ONE thread the lowest slot wins.  The
    // per-iteration tie scan then needs no priority arithmetic at all (it was ~45 % of the loop's instructions).
    const bool linear_prio = (stride & (int)tmask) == 0;
    const uint32_t prio0 = fps_prio((uint32_t)gt, tmask, log2T);
    const uint32_t kprio = (uint32_t)stride >> log2T;

    xyz += (size_t)cloud * Ns * 3;
    idx_out += (size_t)cloud * G;
    centers_out += (size_t)cloud * G * 3;
    float* md_g = (PPT == 0) ? ws + (size_t)cloud * Ns : nullptr;

    if (tid == 0) {
        mbar_init(smem_u32(&mbar[0]), 1);
        mbar_init(smem_u32(&mbar[1]), 1);
        fence_mbar_init();
        mbar_arrive_expect_tx(smem_u32(&mbar[0]), tx_bytes);  // armed for iterations 2 and 1
        mbar_arrive_expect_tx(smem_u32(&mbar[1]), tx_bytes);
    }

    float px[PPT > 0 ? PPT : 1], py[PPT > 0 ? PPT : 1], pz[PPT > 0 ? PPT : 1], md[PPT > 0 ? PPT : 1];
    if constexpr (PPT > 0) {
#pragma unroll
        for (int s = 0; s < PPT; ++s) {
            const int j = s * stride + gt;
            if (j < N) {
                px[s] = xyz[(size_t)j * 3 + 0];
                py[s] = xyz[(size_t)j * 3 + 1];
                pz[s] = xyz[(size_t)j * 3 + 2];
                md[s] = __int_as_float(0x7f800000);  // +inf
            } else {
                px[s] = py[s] = pz[s] = 0.0f;
                md[s] = 0.0f;  // never a candidate unless everything is 0 (then the result is ignored)
            }
            spts[(s * FPS_THREADS + tid) * 3 + 0] = px[s];
            spts[(s * FPS_THREADS + tid) * 3 + 1] = py[s];
            spts[(s * FPS_THREADS + tid) * 3 + 2] = pz[s];
        }
    } else {
        for (int j = gt; j < N; j += stride) md_g[j] = __int_as_float(0x7f800000);
    }

    float cx = xyz[0], cy = xyz[1], cz = xyz[2];
    uint32_t sel = 0;
    if (rank == 0 && tid == 0) {
        idx_out[0] = 0;
        centers_out[0] = cx;
        centers_out[1] = cy;
        centers_out[2] = cz;
        if constexpr (VARLEN) {
            for (int it = Gs; it < G; ++it) {
                idx_out[it] = 0;
                centers_out[it * 3 + 0] = cx;
                centers_out[it * 3 + 1] = cy;
                centers_out[it * 3 + 2] = cz;
            }
        }
    }
    cluster_sync_all();  // barriers initialised and armed everywhere before the first remote store

    for (int it = 1; it < Gs; ++it) {
        const int p = it & 1;
        // ---- 1. update min-distances, per-thread maximum -------------------------------------
        float best = 0.0f;
        uint32_t myprio = 0xFFFFFFFFu;
        float wx = 0.f, wy = 0.f, wz = 0.f;
        if constexpr (PPT > 0) {
#pragma unroll
            for (int s = 0; s < PPT; ++s) {
                const float d = fps_sqdist(px[s], py[s], pz[s], cx, cy, cz);
                md[s] = fminf(md[s], d);
                best = fmaxf(best, md[s]);
            }
        } else {
            for (int j = gt; j < N; j += stride) {
                const float x = xyz[(size_t)j * 3], y = xyz[(size_t)j * 3 + 1], z = xyz[(size_t)j * 3 + 2];
                const float m = fminf(md_g[j], fps_sqdist(x, y, z, cx, cy, cz));
                md_g[j] = m;
                const uint32_t pr = fps_prio((uint32_t)j, tmask, log2T);
                if (m > best || (m == best && pr < myprio)) {
                    best = m;
                    myprio = pr;
                    wx = x, wy = y, wz = z;
                }
            }
        }
        // ---- 2. warp candidate: max distance, then min priority ------------------------------
        const uint32_t bestbits = __float_as_uint(best);
        const uint32_t wmax = __reduce_max_sync(0xffffffffu, bestbits);
        if constexpr (PPT > 0) {
            if (linear_prio) {
                int bs = PPT;  // lowest slot holding the warp maximum (PPT = none)
#pragma unroll
                for (int s = PPT - 1; s >= 0; --s)
                    if (__float_as_uint(md[s]) == wmax) bs = s;
                if (bs < PPT) {
                    myprio = prio0 + (uint32_t)bs * kprio;
                    const float* c = spts + (bs * FPS_THREADS + tid) * 3;  // own data: written by this thread before the loop
                    wx = c[0], wy = c[1], wz = c[2];
                }
            } else if (bestbits == wmax) {
#pragma unroll
                for (int s = 0; s < PPT; ++s) {
                    const uint32_t pr = fps_prio((uint32_t)(s * stride + gt), tmask, log2T);
                    if (__float_as_uint(md[s]) == wmax && pr < myprio) {
                        myprio = pr;
                        wx = px[s], wy = py[s], wz = pz[s];
                    }
                }
            }
        } else {
            if (bestbits != wmax) myprio = 0xFFFFFFFFu;
        }
        const uint32_t wprio = __reduce_min_sync(0xffffffffu, myprio);
        // ---- 3. every warp pushes ITS record straight into every CTA of the cluster (lane c serves peer c): no
        //         shared-memory staging, no __syncthreads, no second reduction stage on the critical path ----------
        {
            const int src = __ffs(__ballot_sync(0xffffffffu, myprio == wprio && bestbits == wmax)) - 1;  // exactly one lane
            const uint32_t ox = __shfl_sync(0xffffffffu, __float_as_uint(wx), src);
            const uint32_t oy = __shfl_sync(0xffffffffu, __float_as_uint(wy), src);
            const uint32_t oz = __shfl_sync(0xffffffffu, __float_as_uint(wz), src);
            if ((uint32_t)lane < C) {
                const int slot = (int)rank * FPS_WARPS + warp;
                const uint32_t ra = mapa_shared(smem_u32(&slot_a[p][slot]), lane);
                const uint32_t rz = mapa_shared(smem_u32(&slot_z[p][slot]), lane);
                const uint32_t rb = mapa_shared(smem_u32(&mbar[p]), lane);
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];"
                             ::"r"(ra), "r"(wmax), "r"(wprio), "r"(ox), "r"(oy), "r"(rb) : "memory");
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];"
                             ::"r"(rz), "r"(oz), "r"(rb) : "memory");
            }
        }
        // ---- 4. wait for the C x 8 records of this iteration, re-arm the barrier for iteration it+2 ----
        {
            const uint32_t bar = smem_u32(&mbar[p]);
            const uint32_t parity = ((uint32_t)(it - 1) >> 1) & 1u;
            // the records arrive through st.async + complete_tx: the phase completion itself orders them before this
            // wait returns (as for TMA writes); a cluster-scope acquire would add an L1 invalidation (CCTL.IVALL, 19 % of
            // the kernel's stall samples in profiles/r02) to every iteration
            mbar_wait(bar, parity);
            if (tid == 0) mbar_arrive_expect_tx(bar, tx_bytes);
        }
        // ---- 5. reduce the records (every warp redundantly; lane l folds records l, l+32, ...) ------
        uint4 a = make_uint4(0u, 0xFFFFFFFFu, 0u, 0u);
        float z = 0.f;
        for (int r = lane; r < (int)C * FPS_WARPS; r += 32) {
            const uint4 b4 = slot_a[p][r];
            if (b4.x > a.x || (b4.x == a.x && b4.y < a.y)) {
                a = b4;
                z = slot_z[p][r];
            }
        }
        const uint32_t fmax = __reduce_max_sync(0xffffffffu, a.x);
        const uint32_t fprio = __reduce_min_sync(0xffffffffu, a.x == fmax ? a.y : 0xFFFFFFFFu);
        const int fo = __ffs(__ballot_sync(0xffffffffu, a.x == fmax && a.y == fprio)) - 1;
        const float nx = __uint_as_float(__shfl_sync(0xffffffffu, a.z, fo));
        const float ny = __uint_as_float(__shfl_sync(0xffffffffu, a.w, fo));
        const float nz = __shfl_sync(0xffffffffu, z, fo);
        if (fmax != 0u) {  // max == 0: every remaining point coincides with a selected one -> repeat
            cx = nx, cy = ny, cz = nz;
            sel = ((fprio & qmask) << log2T) | (__brev(fprio & ~qmask));
        }
        if (rank == 0 && tid == 0) {
            idx_out[it] = (long long)sel;
            centers_out[it * 3 + 0] = cx;
            centers_out[it * 3 + 1] = cy;
            centers_out[it * 3 + 2] = cz;
        }
    }
    cluster_sync_all();  // no CTA may exit while peers can still write into its shared memory
}

template <int PPT, bool VARLEN>
static int launch_fps(const float* xyz, int B, int N, int G, int log2T, const int* lengths, long long* idx, float* centers,
                      float* ws, int cluster, cudaStream_t stream, bool probe_only = false) {
    auto kern = fps_cluster_kernel<PPT, VARLEN>;
    if (cluster > 8) PSAM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(B * cluster));
    cfg.blockDim = dim3(FPS_THREADS);
    cfg.dynamicSmemBytes = (size_t)PPT * FPS_THREADS * 3 * sizeof(float);
    if (cfg.dynamicSmemBytes > 32 * 1024)  // static + dynamic beyond the 48 KB default needs the opt-in
        PSAM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.dynamicSmemBytes));
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 2 : 1;
    if (probe_only) {  // can a cluster of this size be co-scheduled at all on this device?
        int n = 0;
        cfg.numAttrs = 1;
        if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
            cudaGetLastError();
            return PSAM_ERR_UNSUPPORTED;
        }
        return n > 0 ? PSAM_OK : PSAM_ERR_UNSUPPORTED;
    }
    PSAM_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, xyz, N, G, log2T, lengths, idx, centers, ws));
    return PSAM_OK;
}

static void fps_plan(int N, int max_cluster, int* cluster, int* ppt) {
    // Prefer the largest cluster (least work per SM), then the smallest PPT that holds the cloud.
    int c = max_cluster > 8 && N > 8 * FPS_THREADS * 32 ? max_cluster : (max_cluster > 8 ? 8 : max_cluster);
    while (c > 1 && (c / 2) * FPS_THREADS >= N) c /= 2;
    long long per_thread = ceil_div_ll(N, (long long)c * FPS_THREADS);
    int p = 1;
    while (p < per_thread) p *= 2;
    *cluster = c;
    *ppt = (p <= 32) ? p : 0;
}

// 16-CTA clusters are "non-portable": probed once per process, used only for clouds that do not fit 8 CTAs' registers.
static int fps_max_cluster() {
    static int v = 0;
    if (v == 0) v = launch_fps<32, false>(nullptr, 1, 1, 1, 5, nullptr, nullptr, nullptr, nullptr, 16, 0, true) == PSAM_OK ? 16 : 8;
    return v;
}

}  // namespace psam

extern "C" size_t psam_fps_workspace_bytes(int B, int N, int G) {
    (void)G;
    // conservative: the 16-CTA register-resident plan may be unavailable on the device, so every cloud beyond the
    // 8-CTA capacity gets a workspace (used only by the streaming fallback)
    int cluster, ppt;
    psam::fps_plan(N, 8, &cluster, &ppt);
    return ppt == 0 ? (size_t)B * N * sizeof(float) : 0;
}

namespace psam {

// Shared by psam_fps_f32 (lengths == nullptr) and psam_fps_varlen_f32: the cluster size and points per thread come from N.
template <bool VARLEN>
static int fps_dispatch(const float* xyz, int B, int N, int G, const int* lengths, long long* idx_out, float* centers_out,
                        void* workspace, cudaStream_t stream) {
    const int log2T = fps_log2T(N);
    int cluster, ppt;
    fps_plan(N, N > 8 * FPS_THREADS * 32 ? fps_max_cluster() : 8, &cluster, &ppt);
    if (ppt == 0) cluster = fps_max_cluster();  // streaming fallback: spread the cloud over as many SMs as possible
    if (ppt == 0 && !workspace) return PSAM_ERR_ARG;
    float* ws = (float*)workspace;
    switch (ppt) {
        case 1: return launch_fps<1, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        case 2: return launch_fps<2, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        case 4: return launch_fps<4, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        case 8: return launch_fps<8, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        case 16: return launch_fps<16, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        case 32: return launch_fps<32, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
        default: return launch_fps<0, VARLEN>(xyz, B, N, G, log2T, lengths, idx_out, centers_out, ws, cluster, stream);
    }
}

}  // namespace psam

extern "C" int psam_fps_f32(const float* xyz, int B, int N, int G, long long* idx_out, float* centers_out,
                            void* workspace, cudaStream_t stream) {
    if (!xyz || !idx_out || !centers_out || B <= 0 || N <= 0 || G <= 0 || G > N) return PSAM_ERR_ARG;
    return psam::fps_dispatch<false>(xyz, B, N, G, nullptr, idx_out, centers_out, workspace, stream);
}

extern "C" int psam_fps_varlen_f32(const float* xyz, const int* lengths, int B, int N_max, int G, long long* idx_out,
                                   float* centers_out, void* workspace, cudaStream_t stream) {
    if (!xyz || !lengths || !idx_out || !centers_out || B <= 0 || N_max <= 0 || G <= 0) return PSAM_ERR_ARG;
    return psam::fps_dispatch<true>(xyz, B, N_max, G, lengths, idx_out, centers_out, workspace, stream);
}
