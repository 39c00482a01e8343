// Dense scans: an exact nearest-key search on a uniform grid, and a deterministic voxel subsample.  The semantics, the
// stopping rule's rounding margin and the workspace layouts are stated in include/psam_b200.h.
//
// Grid nearest search (psam_nn_grid_f32):
//   nn_box_kernel      one thread per key: the box of the finite keys (atomicMax on order-preserving bit patterns) and
//                      their count; nn_boxhist_kernel their histogram on each axis.
//   nn_setup_kernel    one thread: the grid's box (from the histogram's 5 % and 95 % quantiles), cell size h and
//                      extents (bisection in fp64 on the cell count).
//   nn_hist_kernel     one thread per key: its cell, and its rank in the cell from the counting atomic.
//   nn_scan_*          exclusive prefix sum of the cell counts (block scans, one CTA over the block totals, offsets).
//   nn_scatter_kernel  one thread per key: (x, y, z, index) to its slot of the cell-sorted array.
//   nn_query_kernel    one thread per query: rings of cells outward from its cell, each ring's rows along z read as one
//                      contiguous run, until the lower bound of every unvisited cell exceeds the best distance.
// Voxel subsample (psam_voxel_subsample_f32):
//   vox_quant_kernel   one thread per point: validity and the level-21 cell key.
//   vox_count_kernel   x5, with vox_step_kernel: binary search for L* over the levels, each step counting the distinct
//                      cells of one level in a fresh open-addressing hash set.
//   vox_insert_kernel  the hash set of level L*, each cell's smallest e (atomicMin), then vox_rep_kernel its smallest
//                      index among the points with that e.
//   vox_list_kernel    the occupied slots as (h(key), representative) pairs.
//   vox_hist_kernel    x8, with vox_pick_kernel: radix select of the S-th smallest h, 8 bits per pass.
//   vox_mark_kernel    flags the kept representatives; vox_flag_scan_kernel / vox_compact_kernel write them in
//                      ascending order.
#include <math.h>
#include "psam_common.cuh"
#include "../../include/psam_b200.h"

namespace {

constexpr int kThreads = 256;
constexpr int kScan = 1024;
constexpr long long kMaxCells = 1ll << 22;
constexpr float kNoDist = 3.4e38f;  // psam_nn_distance_f32's "no key" distance: a candidate must be below it
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kBoxBins = 1024;  // histogram bins per axis for the grid's box

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// ------------------------------------------------------------------------------------------------------------------
// grid nearest search
// ------------------------------------------------------------------------------------------------------------------
struct Grid {
    double lo[3], hi[3], klo[3], h, inv_h;  // grid origin, the keys' maximum and minimum (exact), cell side
    int dims[3];
    int cells;  // 0: no finite key
};

struct NnHeader {            // zeroed by one memset together with the cell counts
    unsigned lo_enc[3];      // ~enc(min): the maximum of ~enc is the minimum
    unsigned hi_enc[3];
    unsigned nfin;
    unsigned pad;
    Grid g;
    unsigned hist[3][kBoxBins];  // per axis: the finite keys in each of kBoxBins equal bins of [min, max]
};
constexpr size_t kNnHeader = (sizeof(NnHeader) + 15) & ~(size_t)15;
static_assert(sizeof(NnHeader) <= kNnHeader, "header");

// order-preserving map of a float to an unsigned (for finite values: a < b iff enc(a) < enc(b))
__device__ __forceinline__ unsigned enc_f(float f) {
    const unsigned b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_f(unsigned e) { return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e); }

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

long long nn_cell_cap(int n2) { return n2 < kMaxCells ? (long long)(n2 > 0 ? n2 : 1) : kMaxCells; }

__global__ void __launch_bounds__(kThreads) nn_box_kernel(const float* __restrict__ key, int n2, NnHeader* __restrict__ hd) {
    psam::pdl_prologue();
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    unsigned lo[3] = {0u, 0u, 0u}, hi[3] = {0u, 0u, 0u};
    bool fin = false;
    if (j < n2) {
        const float x = key[j * 3], y = key[j * 3 + 1], z = key[j * 3 + 2];
        fin = finite3(x, y, z);
        if (fin) {
            const float p[3] = {x, y, z};
#pragma unroll
            for (int a = 0; a < 3; ++a) lo[a] = ~enc_f(p[a]), hi[a] = enc_f(p[a]);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = __reduce_max_sync(0xffffffffu, lo[a]);
        hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
    }
    const unsigned nf = __reduce_add_sync(0xffffffffu, fin ? 1u : 0u);
    if ((threadIdx.x & 31) == 0 && nf) {
#pragma unroll
        for (int a = 0; a < 3; ++a) atomicMax(&hd->lo_enc[a], lo[a]), atomicMax(&hd->hi_enc[a], hi[a]);
        atomicAdd(&hd->nfin, nf);
    }
}

__global__ void __launch_bounds__(kThreads) nn_boxhist_kernel(const float* __restrict__ key, int n2, NnHeader* __restrict__ hd) {
    psam::pdl_prologue();
    __shared__ unsigned sh[3][kBoxBins];
    for (int t = threadIdx.x; t < 3 * kBoxBins; t += kThreads) sh[t / kBoxBins][t % kBoxBins] = 0;
    __syncthreads();
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j < n2) {
        const float x = key[j * 3], y = key[j * 3 + 1], z = key[j * 3 + 2];
        if (finite3(x, y, z)) {
            const float p[3] = {x, y, z};
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                const double lo = (double)dec_f(~hd->lo_enc[a]), ext = (double)dec_f(hd->hi_enc[a]) - lo;
                const double b = ext > 0.0 ? floor(((double)p[a] - lo) * (kBoxBins / ext)) : 0.0;
                atomicAdd(&sh[a][(int)fmin(fmax(b, 0.0), kBoxBins - 1.0)], 1u);
            }
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 3 * kBoxBins; t += kThreads)
        if (sh[t / kBoxBins][t % kBoxBins]) atomicAdd(&hd->hist[t / kBoxBins][t % kBoxBins], sh[t / kBoxBins][t % kBoxBins]);
}

// the bin of the histogram that holds the key of 0-based rank r
__device__ __forceinline__ int hist_bin(const unsigned* h, unsigned r) {
    unsigned c = 0;
    int b = 0;
    for (; b < kBoxBins - 1 && c + h[b] <= r; ++b) c += h[b];
    return b;
}

__device__ __forceinline__ double grid_cells(const double* ext, double h) {
    double c = 1.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) c *= fmin(floor(ext[a] / h) + 1.0, 2097152.0);
    return c;
}

__global__ void nn_setup_kernel(NnHeader* __restrict__ hd, long long cap) {
    psam::pdl_prologue();
    Grid& g = hd->g;
    if (hd->nfin == 0) {
        g.cells = 0;
        return;
    }
    // The grid spans the 5 % - 95 % quantiles of the keys on each axis (to histogram-bin precision), widened by 10 % of that
    // width and clipped to the keys' box: far outliers would otherwise crowd the rest into a handful of cells.  Keys outside
    // it are clamped into the border cells, which keeps every face bound of the search valid (see the header), so the grid
    // decides the speed, never the result.
    double ext[3], emax = 0.0;
    const unsigned F = hd->nfin;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        g.klo[a] = (double)dec_f(~hd->lo_enc[a]);
        g.hi[a] = (double)dec_f(hd->hi_enc[a]);
        const double bw = (g.hi[a] - g.klo[a]) / kBoxBins;
        const double qlo = g.klo[a] + hist_bin(hd->hist[a], F / 20) * bw;
        const double qhi = g.klo[a] + (hist_bin(hd->hist[a], F - 1 - F / 20) + 1) * bw;
        const double glo = fmax(g.klo[a], qlo - 0.1 * (qhi - qlo)), ghi = fmin(g.hi[a], qhi + 0.1 * (qhi - qlo));
        g.lo[a] = glo;
        ext[a] = ghi - glo;
        emax = fmax(emax, ext[a]);
    }
    const double T = (double)min((long long)hd->nfin, cap);  // target cell count: about one finite key per cell
    double h = 1.0;
    if (emax > 0.0) {
        double a = emax / (T + 1.0), b = 2.0 * emax;  // cells(a) > T >= 1 = cells(b)
        for (int it = 0; it < 80; ++it) {
            const double m = 0.5 * (a + b);
            if (grid_cells(ext, m) <= T) b = m;
            else a = m;
        }
        h = b;
    }
    long long cells = 1;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        g.dims[a] = emax > 0.0 ? (int)fmin(floor(ext[a] / h) + 1.0, 2097152.0) : 1;
        cells *= g.dims[a];
    }
    g.h = h;
    g.inv_h = 1.0 / h;
    g.cells = (int)cells;
}

// the cell coordinate of p on axis a: floor((p - lo) * inv_h) in fp64, clamped into the grid
__device__ __forceinline__ int cell_coord(const Grid& g, int a, float p) {
    const double t = floor(((double)p - g.lo[a]) * g.inv_h);
    return (int)fmin(fmax(t, 0.0), (double)(g.dims[a] - 1));
}

__device__ __forceinline__ int cell_id(const Grid& g, int cx, int cy, int cz) { return (cx * g.dims[1] + cy) * g.dims[2] + cz; }

__global__ void __launch_bounds__(kThreads) nn_hist_kernel(const float* __restrict__ key, int n2, const NnHeader* __restrict__ hd,
                                                           unsigned* __restrict__ count, unsigned* __restrict__ kcell,
                                                           unsigned* __restrict__ krank) {
    psam::pdl_prologue();
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j >= n2) return;
    const Grid g = hd->g;
    const float x = key[j * 3], y = key[j * 3 + 1], z = key[j * 3 + 2];
    if (g.cells == 0 || !finite3(x, y, z)) {
        kcell[j] = 0xffffffffu;
        return;
    }
    const int c = cell_id(g, cell_coord(g, 0, x), cell_coord(g, 1, y), cell_coord(g, 2, z));
    kcell[j] = (unsigned)c;
    krank[j] = atomicAdd(count + c, 1u);
}

__global__ void __launch_bounds__(kScan) nn_scan_block_kernel(unsigned* __restrict__ count, int n, unsigned long long* __restrict__ bsum) {
    psam::pdl_prologue();
    __shared__ unsigned long long sw[32];
    const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
    const unsigned v = i < n ? count[i] : 0u;
    unsigned long long total;
    const unsigned long long x = psam::block_scan_u64<kScan>(v, sw, total);
    if (i < n) count[i] = (unsigned)(x - v);  // exclusive within the block
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScan) nn_scan_sums_kernel(unsigned long long* __restrict__ bsum, int nb) {
    psam::pdl_prologue();
    psam::scan_block_sums<kScan>(bsum, nb, nullptr);
}

__global__ void __launch_bounds__(kScan) nn_scan_add_kernel(unsigned* __restrict__ start, int n, const unsigned long long* __restrict__ bsum) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
    if (blockIdx.x && i < n) start[i] += (unsigned)bsum[blockIdx.x];
}

__global__ void __launch_bounds__(kThreads) nn_scatter_kernel(const float* __restrict__ key, int n2, const unsigned* __restrict__ start,
                                                              const unsigned* __restrict__ kcell, const unsigned* __restrict__ krank,
                                                              float4* __restrict__ sorted) {
    psam::pdl_prologue();
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j >= n2) return;
    const unsigned c = kcell[j];
    if (c == 0xffffffffu) return;
    sorted[start[c] + krank[j]] = make_float4(key[j * 3], key[j * 3 + 1], key[j * 3 + 2], __int_as_float((int)j));
}

// (d, j) is a better candidate than (bd, bj) when d < kNoDist and (d, j) < (bd, bj) lexicographically
__device__ __forceinline__ void nn_visit(const float4* __restrict__ sorted, unsigned s, unsigned e, float qx, float qy, float qz,
                                         float& bd, int& bj) {
#pragma unroll 1
    for (unsigned t = s; t < e; ++t) {
        const float4 k = __ldg(sorted + t);
        const float d = psam::sqdist3(k.x, k.y, k.z, qx, qy, qz);
        const int j = __float_as_int(k.w);
        if (d < kNoDist && (d < bd || (d == bd && j < bj))) bd = d, bj = j;
    }
}

// One axis of a query: its cell c, the squared distance o2 from its coordinate q to the keys' interval (a lower bound for
// every key), and below = q - lo - slop, above = lo - q - slop, so that the gap to the face at lo + k h, less the rounding
// slop of the header, is below - k h or above + k h.
struct Axis {
    double below, above, o2;
    int c, dims;
};

__device__ __forceinline__ Axis make_axis(const Grid& g, int a, float q) {
    Axis x;
    const double qa = (double)q;
    x.dims = g.dims[a];
    x.c = cell_coord(g, a, q);
    const double o = fmax(fmax(g.klo[a] - qa, qa - g.hi[a]), 0.0);
    x.o2 = o * o;
    const double slop = 0x1p-40 * (fabs(g.lo[a]) + fabs(g.klo[a]) + fabs(g.hi[a]) + fabs(qa) + g.h * (x.dims + 1.0));
    x.below = (qa - g.lo[a]) - slop;
    x.above = (g.lo[a] - qa) - slop;
    return x;
}

// lower bound over the unvisited cells beyond the two faces of the visited block (cells c - r .. c + r) on this axis; `rest`
// is the other axes' o2
__device__ __forceinline__ double side_bound(const Axis& x, int r, double h, double rest, double lb) {
    if (x.c - r - 1 >= 0) {
        const double t = fmax(x.below - (double)(x.c - r) * h, 0.0);
        lb = fmin(lb, fmax(t * t, x.o2) + rest);
    }
    if (x.c + r + 1 < x.dims) {
        const double t = fmax(x.above + (double)(x.c + r + 1) * h, 0.0);
        lb = fmin(lb, fmax(t * t, x.o2) + rest);
    }
    return lb;
}

__global__ void __launch_bounds__(kThreads, 2) nn_query_kernel(const float* __restrict__ query, int n1, const NnHeader* __restrict__ hd,
                                                            const unsigned* __restrict__ start, const float4* __restrict__ sorted,
                                                            float* __restrict__ dist, long long* __restrict__ idx) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n1) return;
    const float qx = query[i * 3], qy = query[i * 3 + 1], qz = query[i * 3 + 2];
    float bd = kNoDist;
    int bj = -1;
    const int cells = hd->g.cells;
    if (cells > 0 && finite3(qx, qy, qz)) {
        const Grid& g = hd->g;
        const Axis ax = make_axis(g, 0, qx), ay = make_axis(g, 1, qy), az = make_axis(g, 2, qz);
        const double h = g.h;
        const int dy = ay.dims, dz = az.dims;
        for (int r = 0;; ++r) {
            const int x0 = max(ax.c - r, 0), x1 = min(ax.c + r, ax.dims - 1);
            const int y0 = max(ay.c - r, 0), y1 = min(ay.c + r, dy - 1);
            const int z0 = max(az.c - r, 0), z1 = min(az.c + r, dz - 1);
#pragma unroll 1
            for (int cx = x0; cx <= x1; ++cx)
#pragma unroll 1
                for (int cy = y0; cy <= y1; ++cy) {
                    const int row = (cx * dy + cy) * dz;
                    if (abs(cx - ax.c) == r || abs(cy - ay.c) == r) {  // the whole z run of the ring box
                        nn_visit(sorted, __ldg(start + row + z0), __ldg(start + row + z1 + 1), qx, qy, qz, bd, bj);
                    } else {  // only the ring's two z faces
                        if (az.c - r >= 0) nn_visit(sorted, __ldg(start + row + az.c - r), __ldg(start + row + az.c - r + 1), qx, qy, qz, bd, bj);
                        if (r > 0 && az.c + r < dz)
                            nn_visit(sorted, __ldg(start + row + az.c + r), __ldg(start + row + az.c + r + 1), qx, qy, qz, bd, bj);
                    }
                }
            // lower bound on the squared distance to any key outside the cells visited so far (see the header)
            double lb = side_bound(ax, r, h, ay.o2 + az.o2, INFINITY);
            lb = side_bound(ay, r, h, ax.o2 + az.o2, lb);
            lb = side_bound(az, r, h, ax.o2 + ay.o2, lb);
            if (lb == INFINITY) break;  // every cell visited
            const double lbd = lb * (1.0 - 0x1p-20) - 0x1p-140;
            if (lbd > (double)bd || lbd >= (double)kNoDist) break;
        }
    }
    dist[i] = bd;
    if (idx) idx[i] = bj;
}

// workspace of psam_nn_grid_f32: [header with the histograms, 12.4 KB][start: cap + 1 uint32][chunk sums][kcell: n2][krank: n2][sorted: n2 float4]
struct NnLayout {
    size_t start, bsum, kcell, krank, sorted, total;
    long long cap;
    int nb;
};

NnLayout nn_layout(int n2) {
    NnLayout L;
    L.cap = nn_cell_cap(n2);
    L.nb = (int)psam::ceil_div_ll(L.cap + 1, kScan);
    L.start = kNnHeader;
    L.bsum = L.start + align16((size_t)(L.cap + 1) * 4);
    L.kcell = L.bsum + align16((size_t)L.nb * 8);
    L.krank = L.kcell + align16((size_t)n2 * 4);
    L.sorted = L.krank + align16((size_t)n2 * 4);
    L.total = L.sorted + (size_t)n2 * 16;
    return L;
}

// ------------------------------------------------------------------------------------------------------------------
// voxel subsample
// ------------------------------------------------------------------------------------------------------------------
struct VoxState {                // zeroed by a memset
    unsigned long long valid;    // valid points
    unsigned long long cnt;      // distinct cells found by the current pass
    unsigned long long nlist;    // representatives listed
    unsigned long long prefix;   // radix select: the high digits of the threshold chosen so far
    unsigned long long krem;     // radix select: the rank still to find below the prefix
    int lo, hi;                  // binary search over the levels
};
constexpr size_t kVoxState = 256;

__device__ __forceinline__ unsigned long long splitmix(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__device__ __forceinline__ unsigned long long level_key(unsigned long long k21, int L) {
    const int s = 21 - L;
    const unsigned long long m = (1ull << 21) - 1;
    return (((k21 >> 42) >> s) << 42) | ((((k21 >> 21) & m) >> s) << 21) | ((k21 & m) >> s);
}

__device__ __forceinline__ long long cell_e(unsigned long long k21, int L) {
    const int s = 21 - L;
    long long e = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const long long q = (long long)((k21 >> (42 - 21 * a)) & ((1ull << 21) - 1));
        const long long d = 2 * q + 1 - (2 * (q >> s) + 1) * (1ll << s);
        e += d * d;
    }
    return e;
}

// the slot of `key` in an open-addressing set (linear probing, kEmpty = free); is_new: this call inserted it
__device__ __forceinline__ unsigned long long set_insert(unsigned long long* table, unsigned long long mask, unsigned long long key, bool& is_new) {
    unsigned long long s = splitmix(key) & mask;
    is_new = false;
    for (;;) {
        const unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(table + s);
        if (cur == key) return s;
        if (cur == kEmpty) {
            const unsigned long long prev = atomicCAS(table + s, kEmpty, key);
            if (prev == kEmpty) {
                is_new = true;
                return s;
            }
            if (prev == key) return s;
        }
        s = (s + 1) & mask;
    }
}

__device__ __forceinline__ float quant(float x) {
    const float t = floorf(__fmul_rn(__fadd_rn(x, 1.0f), 1048576.0f));
    return fminf(fmaxf(t, 0.0f), 2097151.0f);
}

__global__ void __launch_bounds__(kThreads) vox_quant_kernel(const float* __restrict__ xyz, int P, unsigned long long* __restrict__ k21,
                                                             VoxState* __restrict__ st) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool ok = false;
    if (i < P) {
        const float x = xyz[i * 3], y = xyz[i * 3 + 1], z = xyz[i * 3 + 2];
        ok = finite3(x, y, z);
        k21[i] = ok ? ((unsigned long long)quant(x) << 42) | ((unsigned long long)quant(y) << 21) | (unsigned long long)quant(z) : kEmpty;
    }
    const int n = __syncthreads_count(ok);
    if (threadIdx.x == 0) {
        if (n) atomicAdd(&st->valid, (unsigned long long)n);
        if (blockIdx.x == 0) st->hi = 21;
    }
}

// one step of the binary search: counts the distinct cells of level (lo + hi) / 2 (nothing once lo == hi)
__global__ void __launch_bounds__(kThreads) vox_count_kernel(const unsigned long long* __restrict__ k21, int P, unsigned long long* table,
                                                             unsigned long long mask, VoxState* __restrict__ st) {
    psam::pdl_prologue();
    const int lo = st->lo, hi = st->hi;
    if (lo == hi) return;
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool is_new = false;
    if (i < P && k21[i] != kEmpty) set_insert(table, mask, level_key(k21[i], (lo + hi) >> 1), is_new);
    const int n = __syncthreads_count(is_new);
    if (threadIdx.x == 0 && n) atomicAdd(&st->cnt, (unsigned long long)n);
}

__global__ void vox_step_kernel(VoxState* __restrict__ st, int S) {
    psam::pdl_prologue();
    if (st->lo < st->hi) {
        const int mid = (st->lo + st->hi) >> 1;
        if (st->cnt >= (unsigned long long)S) st->hi = mid;
        else st->lo = mid + 1;
    }
    st->cnt = 0;
}

// the set of level L* (= lo once the search is done): each point's slot, and the smallest e of each cell
__global__ void __launch_bounds__(kThreads) vox_insert_kernel(const unsigned long long* __restrict__ k21, int P, unsigned long long* table,
                                                              unsigned long long mask, unsigned* __restrict__ pslot,
                                                              unsigned long long* __restrict__ rep_e, VoxState* __restrict__ st) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool is_new = false;
    if (i < P && k21[i] != kEmpty) {
        const int L = st->lo;
        const unsigned long long s = set_insert(table, mask, level_key(k21[i], L), is_new);
        pslot[i] = (unsigned)s;
        atomicMin(rep_e + s, (unsigned long long)cell_e(k21[i], L));
    }
    const int n = __syncthreads_count(is_new);
    if (threadIdx.x == 0 && n) atomicAdd(&st->cnt, (unsigned long long)n);
}

__global__ void __launch_bounds__(kThreads) vox_rep_kernel(const unsigned long long* __restrict__ k21, int P, const unsigned* __restrict__ pslot,
                                                           const unsigned long long* __restrict__ rep_e, unsigned* __restrict__ rep_i,
                                                           const VoxState* __restrict__ st) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= P || k21[i] == kEmpty) return;
    const unsigned s = pslot[i];
    if ((unsigned long long)cell_e(k21[i], st->lo) == rep_e[s]) atomicMin(rep_i + s, (unsigned)i);
}

__global__ void __launch_bounds__(kThreads) vox_list_kernel(const unsigned long long* __restrict__ table, unsigned long long cap,
                                                            const unsigned* __restrict__ rep_i, unsigned long long seed,
                                                            unsigned long long* __restrict__ lh, unsigned* __restrict__ li,
                                                            VoxState* __restrict__ st) {
    psam::pdl_prologue();
    const unsigned long long s = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
    if (s >= cap) return;
    const unsigned long long key = table[s];
    if (key == kEmpty) return;
    const unsigned long long t = atomicAdd(&st->nlist, 1ull);
    lh[t] = splitmix(seed + (key + 1ull) * 0x9E3779B97F4A7C15ull);
    li[t] = rep_i[s];
}

// radix select, pass `pass` (0 = the top 8 bits): histogram of the next digit among the hashes that match the prefix
__global__ void __launch_bounds__(kThreads) vox_hist_kernel(const unsigned long long* __restrict__ lh, int S, int pass,
                                                            unsigned* __restrict__ hist, const VoxState* __restrict__ st) {
    psam::pdl_prologue();
    __shared__ unsigned sh[256];
    const unsigned long long n = st->nlist;
    if (n <= (unsigned long long)S) return;  // every representative is kept
    const long long base = (long long)blockIdx.x * kThreads;
    if ((unsigned long long)base >= n) return;
    sh[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long t = base + threadIdx.x;
    const int shift = 56 - 8 * pass;
    if (t < n) {
        const unsigned long long h = lh[t];
        if (pass == 0 || (h >> (shift + 8)) == (st->prefix >> (shift + 8))) atomicAdd(&sh[(h >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(hist + threadIdx.x, sh[threadIdx.x]);
}

__global__ void vox_pick_kernel(int S, int pass, unsigned* __restrict__ hist, VoxState* __restrict__ st) {
    psam::pdl_prologue();
    if (st->nlist <= (unsigned long long)S) return;
    unsigned long long k = pass == 0 ? (unsigned long long)S : st->krem;  // 1-based rank among the prefix's hashes
    const int shift = 56 - 8 * pass;
    unsigned long long c = 0;
    int d = 0;
    for (; d < 255 && c + hist[d] < k; ++d) c += hist[d];
    st->prefix = (pass == 0 ? 0ull : st->prefix) | ((unsigned long long)d << shift);
    st->krem = k - c;
    for (int b = 0; b < 256; ++b) hist[b] = 0;
}

__global__ void __launch_bounds__(kThreads) vox_mark_kernel(const unsigned long long* __restrict__ lh, const unsigned* __restrict__ li,
                                                            int S, unsigned char* __restrict__ flag, const VoxState* __restrict__ st,
                                                            long long* __restrict__ stats) {
    psam::pdl_prologue();
    const unsigned long long n = st->nlist;
    const unsigned long long t = (unsigned long long)blockIdx.x * kThreads + threadIdx.x;
    if (t == 0) {
        stats[0] = (long long)st->valid;
        stats[1] = st->lo;
        stats[2] = (long long)n;
        stats[3] = (long long)(n < (unsigned long long)S ? n : (unsigned long long)S);
    }
    if (t >= n) return;
    if (n <= (unsigned long long)S || lh[t] <= st->prefix) flag[li[t]] = 1;
}

__global__ void __launch_bounds__(kScan) vox_flag_scan_kernel(const unsigned char* __restrict__ flag, int P, unsigned long long* __restrict__ bsum) {
    psam::pdl_prologue();
    const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
    const int n = __syncthreads_count(i < P && flag[i]);
    if (threadIdx.x == 0) bsum[blockIdx.x] = (unsigned long long)n;
}

__global__ void __launch_bounds__(kScan) vox_compact_kernel(const unsigned char* __restrict__ flag, int P, const unsigned long long* __restrict__ bsum,
                                                            int S, long long* __restrict__ idx_out) {
    psam::pdl_prologue();
    __shared__ unsigned long long sw[32];
    const long long i = (long long)blockIdx.x * kScan + threadIdx.x;
    const unsigned f = i < P && flag[i] ? 1u : 0u;
    unsigned long long total;
    const unsigned long long x = psam::block_scan_u64<kScan>(f, sw, total);
    const unsigned long long pos = bsum[blockIdx.x] + x - 1;
    if (f && pos < (unsigned long long)S) idx_out[pos] = i;
}

// workspace of psam_voxel_subsample_f32: [state 256 B][k21: P uint64][table: cap uint64][rep_e: cap uint64][rep_i: cap uint32]
// [pslot: P uint32][list hashes: P uint64][list indices: P uint32][flags: P bytes][chunk sums][histogram: 256 uint32]
struct VoxLayout {
    size_t k21, table, rep_e, rep_i, pslot, lh, li, flag, bsum, hist, total;
    unsigned long long cap;
    int nb;
};

VoxLayout vox_layout(int P) {
    VoxLayout L;
    L.cap = 64;
    while (L.cap < 2ull * (unsigned long long)P) L.cap <<= 1;
    L.nb = psam::ceil_div(P, kScan);
    L.k21 = kVoxState;
    L.table = L.k21 + (size_t)P * 8;
    L.rep_e = L.table + L.cap * 8;
    L.rep_i = L.rep_e + L.cap * 8;
    L.pslot = L.rep_i + align16(L.cap * 4);
    L.lh = L.pslot + align16((size_t)P * 4);
    L.li = L.lh + (size_t)P * 8;
    L.flag = L.li + align16((size_t)P * 4);
    L.bsum = L.flag + align16((size_t)P);
    L.hist = L.bsum + align16((size_t)L.nb * 8);
    L.total = L.hist + 1024;
    return L;
}

}  // namespace

extern "C" size_t psam_nn_grid_workspace_bytes(int n2) {
    if (n2 <= 0) return 0;
    return nn_layout(n2).total;
}

extern "C" int psam_nn_grid_f32(const float* query, int n1, const float* key, int n2, float* dist_out, long long* idx_out,
                                void* workspace, cudaStream_t stream) {
    if (!query || !key || !dist_out || !workspace || n1 <= 0 || n2 <= 0) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    const NnLayout L = nn_layout(n2);
    char* ws = static_cast<char*>(workspace);
    NnHeader* hd = reinterpret_cast<NnHeader*>(ws);
    unsigned* start = reinterpret_cast<unsigned*>(ws + L.start);
    unsigned long long* bsum = reinterpret_cast<unsigned long long*>(ws + L.bsum);
    unsigned* kcell = reinterpret_cast<unsigned*>(ws + L.kcell);
    unsigned* krank = reinterpret_cast<unsigned*>(ws + L.krank);
    float4* sorted = reinterpret_cast<float4*>(ws + L.sorted);
    const unsigned kb = (unsigned)psam::ceil_div(n2, kThreads);
    PSAM_CUDA_TRY(cudaMemsetAsync(ws, 0, L.start + (size_t)(L.cap + 1) * 4, stream));
    PSAM_CUDA_TRY(psam::launch(nn_box_kernel, dim3(kb), dim3(kThreads), (size_t)0, stream, key, n2, hd));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(nn_boxhist_kernel, dim3(kb), dim3(kThreads), (size_t)0, stream, key, n2, hd));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(nn_setup_kernel, dim3(1), dim3(1), (size_t)0, stream, hd, L.cap));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(nn_hist_kernel, dim3(kb), dim3(kThreads), (size_t)0, stream, key, n2, (const NnHeader*)hd, start, kcell, krank));
    PSAM_LAUNCH_CHECK();
    const int nc = (int)(L.cap + 1);  // start[cells] = the finite keys: the scan covers the whole capacity
    PSAM_CUDA_TRY(psam::launch(nn_scan_block_kernel, dim3(L.nb), dim3(kScan), (size_t)0, stream, start, nc, bsum));
    PSAM_LAUNCH_CHECK();
    if (L.nb > 1) {
        PSAM_CUDA_TRY(psam::launch(nn_scan_sums_kernel, dim3(1), dim3(kScan), (size_t)0, stream, bsum, L.nb));
        PSAM_LAUNCH_CHECK();
        PSAM_CUDA_TRY(psam::launch(nn_scan_add_kernel, dim3(L.nb), dim3(kScan), (size_t)0, stream, start, nc, (const unsigned long long*)bsum));
        PSAM_LAUNCH_CHECK();
    }
    PSAM_CUDA_TRY(psam::launch(nn_scatter_kernel, dim3(kb), dim3(kThreads), (size_t)0, stream, key, n2, (const unsigned*)start,
                               (const unsigned*)kcell, (const unsigned*)krank, sorted));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(nn_query_kernel, dim3((unsigned)psam::ceil_div_ll(n1, kThreads)), dim3(kThreads), (size_t)0, stream, query,
                               n1, (const NnHeader*)hd, (const unsigned*)start, (const float4*)sorted, dist_out, idx_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}

extern "C" size_t psam_voxel_subsample_workspace_bytes(int P) {
    if (P <= 0) return 0;
    return vox_layout(P).total;
}

extern "C" int psam_voxel_subsample_f32(const float* xyz, int P, int S, unsigned long long seed, long long* idx_out, long long* stats,
                                        void* workspace, cudaStream_t stream) {
    if (!xyz || !idx_out || !stats || !workspace || P <= 0 || S <= 0) return PSAM_ERR_ARG;
    if (reinterpret_cast<uintptr_t>(workspace) & 15) return PSAM_ERR_ARG;
    const VoxLayout L = vox_layout(P);
    char* ws = static_cast<char*>(workspace);
    VoxState* st = reinterpret_cast<VoxState*>(ws);
    unsigned long long* k21 = reinterpret_cast<unsigned long long*>(ws + L.k21);
    unsigned long long* table = reinterpret_cast<unsigned long long*>(ws + L.table);
    unsigned long long* rep_e = reinterpret_cast<unsigned long long*>(ws + L.rep_e);
    unsigned* rep_i = reinterpret_cast<unsigned*>(ws + L.rep_i);
    unsigned* pslot = reinterpret_cast<unsigned*>(ws + L.pslot);
    unsigned long long* lh = reinterpret_cast<unsigned long long*>(ws + L.lh);
    unsigned* li = reinterpret_cast<unsigned*>(ws + L.li);
    unsigned char* flag = reinterpret_cast<unsigned char*>(ws + L.flag);
    unsigned long long* bsum = reinterpret_cast<unsigned long long*>(ws + L.bsum);
    unsigned* hist = reinterpret_cast<unsigned*>(ws + L.hist);
    const unsigned long long mask = L.cap - 1;
    const dim3 pb((unsigned)psam::ceil_div(P, kThreads)), tb(kThreads);
    PSAM_CUDA_TRY(cudaMemsetAsync(st, 0, kVoxState, stream));
    PSAM_CUDA_TRY(cudaMemsetAsync(hist, 0, 1024, stream));
    PSAM_CUDA_TRY(cudaMemsetAsync(flag, 0, (size_t)P, stream));
    PSAM_CUDA_TRY(cudaMemsetAsync(idx_out, 0xff, (size_t)S * 8, stream));
    PSAM_CUDA_TRY(psam::launch(vox_quant_kernel, pb, tb, (size_t)0, stream, xyz, P, k21, st));
    PSAM_LAUNCH_CHECK();
    for (int step = 0; step < 5; ++step) {  // ceil(log2(22)) steps find L* in 0..21
        PSAM_CUDA_TRY(cudaMemsetAsync(table, 0xff, L.cap * 8, stream));
        PSAM_CUDA_TRY(psam::launch(vox_count_kernel, pb, tb, (size_t)0, stream, (const unsigned long long*)k21, P, table, mask, st));
        PSAM_LAUNCH_CHECK();
        PSAM_CUDA_TRY(psam::launch(vox_step_kernel, dim3(1), dim3(1), (size_t)0, stream, st, S));
        PSAM_LAUNCH_CHECK();
    }
    PSAM_CUDA_TRY(cudaMemsetAsync(table, 0xff, L.cap * 20, stream));  // table, rep_e and rep_i are contiguous
    PSAM_CUDA_TRY(psam::launch(vox_insert_kernel, pb, tb, (size_t)0, stream, (const unsigned long long*)k21, P, table, mask, pslot, rep_e, st));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(vox_rep_kernel, pb, tb, (size_t)0, stream, (const unsigned long long*)k21, P, (const unsigned*)pslot,
                               (const unsigned long long*)rep_e, rep_i, (const VoxState*)st));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(vox_list_kernel, dim3((unsigned)((L.cap + kThreads - 1) / kThreads)), tb, (size_t)0, stream,
                               (const unsigned long long*)table, L.cap, (const unsigned*)rep_i, seed, lh, li, st));
    PSAM_LAUNCH_CHECK();
    for (int pass = 0; pass < 8; ++pass) {
        PSAM_CUDA_TRY(psam::launch(vox_hist_kernel, pb, tb, (size_t)0, stream, (const unsigned long long*)lh, S, pass, hist, (const VoxState*)st));
        PSAM_LAUNCH_CHECK();
        PSAM_CUDA_TRY(psam::launch(vox_pick_kernel, dim3(1), dim3(1), (size_t)0, stream, S, pass, hist, st));
        PSAM_LAUNCH_CHECK();
    }
    PSAM_CUDA_TRY(psam::launch(vox_mark_kernel, pb, tb, (size_t)0, stream, (const unsigned long long*)lh, (const unsigned*)li, S, flag,
                               (const VoxState*)st, stats));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(vox_flag_scan_kernel, dim3(L.nb), dim3(kScan), (size_t)0, stream, (const unsigned char*)flag, P, bsum));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(nn_scan_sums_kernel, dim3(1), dim3(kScan), (size_t)0, stream, bsum, L.nb));
    PSAM_LAUNCH_CHECK();
    PSAM_CUDA_TRY(psam::launch(vox_compact_kernel, dim3(L.nb), dim3(kScan), (size_t)0, stream, (const unsigned char*)flag, P,
                               (const unsigned long long*)bsum, S, idx_out));
    PSAM_LAUNCH_CHECK();
    return PSAM_OK;
}
