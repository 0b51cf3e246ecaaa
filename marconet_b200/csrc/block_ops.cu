// Text blocks split into lines (DESIGN.md 7b, "Text blocks"): Otsu binarisation, a projection profile and line runs for every
// block of a call in four launches (histogram, threshold, profile, segmentation).  The threshold is OpenCV's fp64 loop with
// explicit-rounding intrinsics, so that nvcc cannot contract it into an FMA the host twin (oracle/blocks.py) does not have; the
// rest is integer arithmetic.  Skewed blocks (DESIGN.md 7b, "Skewed blocks") add an angle search and a rotated profile around
// the same kernels, in six launches.  Text pages (DESIGN.md 7b, "Text pages") reuse the histogram and threshold kernels and find
// blocks by a level-synchronous XY-cut over an ink bitmap.  Skewed pages (DESIGN.md 7b, "Skewed pages") run the same XY-cut on a
// bitmap of rotated-frame cells, and their blocks are windows of that frame.  Perspective pages (DESIGN.md 7b, "Perspective
// pages") find a photographed page's corners: the paper's largest 4-connected component, its hull and the largest quad on it.
// Curled blocks (DESIGN.md 7b, "Curled blocks") trace each line across column strips: per-strip profiles and runs, and a
// left-to-right link of the runs into lines, in seven launches.  Ruled pages (DESIGN.md 7b, "Ruled pages") find the ink runs of at
// least a rule length in rows and columns in three more launches, take them out of the page's bitmap and let them cut.  Figures
// (DESIGN.md 7b, "Figures") are the pass-1 leaves of at least a figure size, selected with the text size and painted out of the
// bitmap in one more launch before pass 2.  Mixed directions (DESIGN.md 7b, "Mixed directions") test each kept leaf's row and
// column bands for its own direction in one more launch after the leaves.  Reversed panels (DESIGN.md 7b, "Reversed panels")
// are the flat-filled pass-1 leaves of over half ink, tested and painted as paper-coloured ink inside a rule outline in two more
// launches before pass 2.
#include <climits>

#include "mn_common.cuh"

namespace {

constexpr int kTile = 32;             // tiles of kTile x kTile pixels, 256 threads: lane = column, warp w takes rows w + 8 j
constexpr int kTileThreads = 256;
constexpr int kSegThreads = 1024;

__device__ __forceinline__ int block_grey(const mn_text_block& b, int x, int y) {
    const uint8_t* p = b.img + (long long)(b.y0 + y) * b.pitch + (long long)(b.x0 + x) * 3;
    return ((int)p[0] + (int)p[1] + (int)p[2] + 1) / 3;
}

__device__ __forceinline__ bool tile_origin(const mn_text_block& b, int& tx, int& ty) {
    const int tiles_x = (b.w + kTile - 1) / kTile, tiles_y = (b.h + kTile - 1) / kTile;
    if ((long long)blockIdx.x >= (long long)tiles_x * tiles_y) return false;
    tx = (int)(blockIdx.x % tiles_x) * kTile;
    ty = (int)(blockIdx.x / tiles_x) * kTile;
    return true;
}

__global__ void __launch_bounds__(kTileThreads) block_hist_kernel(const mn_text_block* __restrict__ blocks) {
    mn_pdl_prologue();
    __shared__ int s_hist[256];
    const mn_text_block b = blocks[blockIdx.y];
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    const int x = tx + (threadIdx.x & 31);
    if (x < b.w) {
        for (int y = ty + (threadIdx.x >> 5); y < min(ty + kTile, b.h); y += 8) atomicAdd(&s_hist[block_grey(b, x, y)], 1);
    }
    __syncthreads();
    const int v = s_hist[threadIdx.x];
    if (v) atomicAdd(&b.hist[threadIdx.x], v);
}

// getThreshVal_Otsu_8u's loop, one thread per block.  A uniform crop keeps t = 0.
__global__ void block_threshold_kernel(const mn_text_block* __restrict__ blocks, int n) {
    mn_pdl_prologue();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const mn_text_block b = blocks[i];
    const int* h = b.hist;
    long long count = 0;                                // the pixels counted: w h, or a window's pixel set
    for (int k = 0; k < 256; ++k) count += h[k];
    const double scale = __ddiv_rn(1.0, (double)count);
    double mu = 0.0;
    for (int k = 0; k < 256; ++k) mu = __dadd_rn(mu, __dmul_rn((double)k, (double)h[k]));
    mu = __dmul_rn(mu, scale);
    const double eps = 1.1920928955078125e-07;    // FLT_EPSILON
    double mu1 = 0.0, q1 = 0.0, max_sigma = 0.0;
    int t = 0;
    for (int k = 0; k < (count ? 256 : 0); ++k) {
        const double p = __dmul_rn((double)h[k], scale);
        mu1 = __dmul_rn(mu1, q1);
        q1 = __dadd_rn(q1, p);
        const double q2 = __dsub_rn(1.0, q1);
        if (fmin(q1, q2) < eps || fmax(q1, q2) > 1.0 - eps) continue;
        mu1 = __ddiv_rn(__dadd_rn(mu1, __dmul_rn((double)k, p)), q1);
        const double mu2 = __ddiv_rn(__dsub_rn(mu, __dmul_rn(q1, mu1)), q2);
        const double d = __dsub_rn(mu1, mu2);
        const double sigma = __dmul_rn(__dmul_rn(__dmul_rn(q1, q2), d), d);
        if (sigma > max_sigma) {
            max_sigma = sigma;
            t = k;
        }
    }
    long long dark = 0;
    for (int k = 0; k <= t; ++k) dark += h[k];
    int ink = b.polarity;
    if (ink == MN_INK_AUTO) ink = 2 * dark <= count ? MN_INK_DARK : MN_INK_LIGHT;
    b.out->threshold = t;
    b.out->ink = ink;
}

// Per tile: the ink count, the least and the largest ink index along the line of each of its 32 lines (rows, or columns of a
// vertical block), gathered in shared memory and added into the block's profile with one atomic per line and quantity.
__global__ void __launch_bounds__(kTileThreads) block_profile_kernel(const mn_text_block* __restrict__ blocks) {
    mn_pdl_prologue();
    __shared__ int s_cnt[kTile], s_lo[kTile], s_hi[kTile];
    const mn_text_block b = blocks[blockIdx.y];
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    if (threadIdx.x < kTile) s_cnt[threadIdx.x] = s_lo[threadIdx.x] = s_hi[threadIdx.x] = 0;
    __syncthreads();
    const int t = b.out->threshold;
    const bool dark = b.out->ink == MN_INK_DARK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x = tx + lane, L = b.vertical ? b.w : b.h, M = b.vertical ? b.h : b.w;
    int cnt = 0, lo = 0, hi = 0;                       // lo = M - least index, hi = largest index + 1 (0: none)
    for (int j = 0; j < kTile / 8; ++j) {
        const int y = ty + warp + 8 * j;
        bool ink = false;
        if (x < b.w && y < b.h) {
            const int g = block_grey(b, x, y);
            ink = dark ? g <= t : g > t;
        }
        if (b.vertical) {                               // this lane's column: its own line
            if (ink) {
                ++cnt;
                lo = max(lo, M - y);
                hi = max(hi, y + 1);
            }
        } else {                                        // the warp's row: one line
            const int c = __reduce_add_sync(0xffffffffu, ink ? 1 : 0);
            const unsigned l = __reduce_max_sync(0xffffffffu, ink ? (unsigned)(M - x) : 0u);
            const unsigned h = __reduce_max_sync(0xffffffffu, ink ? (unsigned)(x + 1) : 0u);
            if (lane == 0) {
                s_cnt[warp + 8 * j] = c;
                s_lo[warp + 8 * j] = (int)l;
                s_hi[warp + 8 * j] = (int)h;
            }
        }
    }
    if (b.vertical && cnt) {
        atomicAdd(&s_cnt[lane], cnt);
        atomicMax(&s_lo[lane], lo);
        atomicMax(&s_hi[lane], hi);
    }
    __syncthreads();
    if (threadIdx.x < kTile && s_cnt[threadIdx.x]) {
        const int l = (b.vertical ? tx : ty) + threadIdx.x;
        atomicAdd(&b.prof[l], s_cnt[threadIdx.x]);
        atomicMax(&b.prof[L + l], s_lo[threadIdx.x]);
        atomicMax(&b.prof[2 * L + l], s_hi[threadIdx.x]);
    }
}

// Exclusive prefix sum of v over the CTA; *total receives the sum.  s holds 32 ints.
__device__ __forceinline__ int cta_scan(int v, int* s, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < n_warps ? s[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        s[lane] = w;
    }
    __syncthreads();
    const int pre = (warp ? s[warp - 1] : 0) + x - v;
    *total = s[n_warps - 1];
    __syncthreads();
    return pre;
}

// The lower median (element (n - 1) / 2 in sorted order) of b[j] - a[j], j < n, all in [1, L]: the least v with
// #{b[j] - a[j] <= v} > (n - 1) / 2, by bisection.
__device__ int cta_lower_median(const int* a, const int* b, int n, int L, int* s) {
    int lo = 1, hi = L;
    const int chunk = (n + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * chunk, j1 = min(n, j0 + chunk);
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        int c = 0, total;
        for (int j = j0; j < j1; ++j) c += b[j] - a[j] <= mid;
        cta_scan(c, s, &total);
        if (total > (n - 1) / 2) hi = mid; else lo = mid + 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kSegThreads) block_lines_kernel(const mn_text_block* __restrict__ blocks) {
    mn_pdl_prologue();
    __shared__ int s_scan[32];
    __shared__ int s_a[MN_BLOCK_MAX_LINES], s_b[MN_BLOCK_MAX_LINES];
    const mn_text_block b = blocks[blockIdx.x];
    const int L = b.vertical ? b.w : b.h, M = b.vertical ? b.h : b.w;
    const int* cnt = b.prof;
    const int m = b.min_ink > 0 ? b.min_ink : max(1, M / 128);
    const int half = (L + 2) / 2;                       // at most (L + 1) / 2 runs
    int* ra = b.scratch;                                // the runs [ra, rb), then the merged runs [ma, mb)
    int* rb = ra + half;
    int* ma = rb + half;
    int* mb = ma + half;
    int total;

    // 1. the runs of text lines: the k-th start and the k-th end pair up
    {
        const int chunk = (L + blockDim.x - 1) / blockDim.x, l0 = threadIdx.x * chunk, l1 = min(L, l0 + chunk);
        int c = 0;
        for (int l = l0; l < l1; ++l) {
            if (cnt[l] < m) continue;
            c += (l == 0 || cnt[l - 1] < m) ? 1 : 0;
            c += (l + 1 == L || cnt[l + 1] < m) ? 1 << 16 : 0;
        }
        int o = cta_scan(c, s_scan, &total);
        int os = o & 0xffff, oe = o >> 16;
        for (int l = l0; l < l1; ++l) {
            if (cnt[l] < m) continue;
            if (l == 0 || cnt[l - 1] < m) ra[os++] = l;
            if (l + 1 == L || cnt[l + 1] < m) rb[oe++] = l + 1;
        }
    }
    const int n = total & 0xffff;
    if (n == 0) {
        if (threadIdx.x == 0) b.out->n_lines = 0;
        return;
    }
    __syncthreads();

    // 2. merge across gaps <= G
    const int G = b.gap > 0 ? b.gap : max(1, cta_lower_median(ra, rb, n, L, s_scan) / 4);
    int nm;
    {
        const int chunk = (n + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * chunk, j1 = min(n, j0 + chunk);
        int c = 0;
        for (int j = j0; j < j1; ++j) c += j == 0 || ra[j] - rb[j - 1] > G;
        int g = cta_scan(c, s_scan, &nm) - 1;
        for (int j = j0; j < j1; ++j) {
            if (j == 0 || ra[j] - rb[j - 1] > G) ma[++g] = ra[j];
            if (j + 1 == n || ra[j + 1] - rb[j] > G) mb[g] = rb[j];
        }
    }
    __syncthreads();

    // 3. drop the short ones
    const int mh = b.min_height > 0 ? b.min_height : max(2, cta_lower_median(ma, mb, nm, L, s_scan) / 3);
    int nk;
    {
        const int chunk = (nm + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * chunk, j1 = min(nm, j0 + chunk);
        int c = 0;
        for (int j = j0; j < j1; ++j) c += mb[j] - ma[j] >= mh;
        int k = cta_scan(c, s_scan, &nk);
        if (nk > MN_BLOCK_MAX_LINES) {
            if (threadIdx.x == 0) b.out->n_lines = -nk;
            return;
        }
        for (int j = j0; j < j1; ++j) {
            if (mb[j] - ma[j] < mh) continue;
            s_a[k] = ma[j];
            s_b[k++] = mb[j];
        }
    }
    __syncthreads();

    // 4. one warp per line: pad, neighbours' midpoints, the ink's extent along the line over [a, b)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = warp; k < nk; k += blockDim.x >> 5) {
        const int a = s_a[k], e = s_b[k], p = (e - a + 3) / 4;
        const int l0 = max(a - p, k > 0 ? (s_b[k - 1] + a) / 2 : 0);
        const int l1 = min(e + p, k + 1 < nk ? (e + s_a[k + 1]) / 2 : L);
        int lo = 0, hi = 0;
        for (int l = a + lane; l < e; l += 32) {
            lo = max(lo, b.prof[L + l]);
            hi = max(hi, b.prof[2 * L + l]);
        }
        lo = (int)__reduce_max_sync(0xffffffffu, (unsigned)lo);
        hi = (int)__reduce_max_sync(0xffffffffu, (unsigned)hi);
        if (lane == 0) {
            const int c0 = max(0, M - lo - p), c1 = min(M, hi + p);
            int* r = b.out->rect[b.vertical ? nk - 1 - k : k];
            if (b.vertical) {
                r[0] = b.x0 + l0; r[1] = b.y0 + c0; r[2] = b.x0 + l1; r[3] = b.y0 + c1;
            } else {
                r[0] = b.x0 + c0; r[1] = b.y0 + l0; r[2] = b.x0 + c1; r[3] = b.y0 + l1;
            }
        }
    }
    if (threadIdx.x == 0) b.out->n_lines = nk;
}

// ---- Curled blocks (DESIGN.md 7b, "Curled blocks") ----
// Integer only, as the twin (oracle/curled_blocks.py).  A strip is at least 32 pixels wide (or the only one), so the 32 columns
// of a tile fall in at most two strips.
constexpr int kLinkThreads = 1024;
constexpr int kLinkActive = (MN_CURVE_MAX_GAP + 1) * MN_CURVE_RUN_CAP;   // lines whose last run lies in the last 3 strips
static_assert(kLinkActive + MN_CURVE_RUN_CAP <= kLinkThreads, "one link candidate per thread");

__device__ __forceinline__ int strip_of(int x, int w, int n_s) { return ((x + 1) * n_s - 1) / w; }   // largest j, x_j <= x

// Per tile and per row: the ink count, w - least ink column and largest ink column + 1 in each of the (at most) two strips the
// tile's columns fall in, gathered in shared memory and added with one atomic per non-zero entry.
__global__ void __launch_bounds__(kTileThreads) curve_profile_kernel(const mn_curve_block* __restrict__ curves) {
    mn_pdl_prologue();
    __shared__ int s_cnt[2][kTile], s_lo[2][kTile], s_hi[2][kTile];
    const mn_curve_block cb = curves[blockIdx.y];
    const mn_text_block& b = cb.b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const int t = b.out->threshold;
    const bool dark = b.out->ink == MN_INK_DARK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x = tx + lane, j0 = strip_of(tx, b.w, cb.n_strips);
    const int q = x < b.w ? strip_of(x, b.w, cb.n_strips) - j0 : 0;
    for (int r = 0; r < kTile / 8; ++r) {
        const int y = ty + warp + 8 * r;
        bool ink = false;
        if (x < b.w && y < b.h) {
            const int g = block_grey(b, x, y);
            ink = dark ? g <= t : g > t;
        }
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const bool in = ink && q == s;
            const int c = __reduce_add_sync(0xffffffffu, in ? 1 : 0);
            const unsigned l = __reduce_max_sync(0xffffffffu, in ? (unsigned)(b.w - x) : 0u);
            const unsigned h = __reduce_max_sync(0xffffffffu, in ? (unsigned)(x + 1) : 0u);
            if (lane == 0) {
                s_cnt[s][warp + 8 * r] = c;
                s_lo[s][warp + 8 * r] = (int)l;
                s_hi[s][warp + 8 * r] = (int)h;
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < 2 * kTile) {
        const int s = threadIdx.x / kTile, r = threadIdx.x % kTile;
        if (s_cnt[s][r]) {
            int* p = cb.sprof + (long long)3 * (j0 + s) * b.h + ty + r;
            atomicAdd(p, s_cnt[s][r]);
            atomicMax(p + b.h, s_lo[s][r]);
            atomicMax(p + 2 * b.h, s_hi[s][r]);
        }
    }
}

// Steps 1-3 of block_lines_kernel on the row profile of strip blockIdx.x of block blockIdx.y; the kept runs, unpadded, with
// their least and largest ink column.
__global__ void __launch_bounds__(kSegThreads) curve_runs_kernel(const mn_curve_block* __restrict__ curves) {
    mn_pdl_prologue();
    __shared__ int s_scan[32];
    __shared__ int s_a[MN_CURVE_RUN_CAP], s_b[MN_CURVE_RUN_CAP];
    const mn_curve_block cb = curves[blockIdx.y];
    const mn_text_block& b = cb.b;
    const int j = blockIdx.x;
    if (j >= cb.n_strips) return;
    const int L = b.h, M = (j + 1) * b.w / cb.n_strips - j * b.w / cb.n_strips;
    const int* cnt = cb.sprof + (long long)3 * j * L;
    const int m = b.min_ink > 0 ? b.min_ink : max(1, M / 128);
    const int half = (L + 2) / 2;
    int* ra = cb.sscratch + (long long)j * (2 * L + 4);
    int* rb = ra + half;
    int* ma = rb + half;
    int* mb = ma + half;
    int total;
    {
        const int chunk = (L + blockDim.x - 1) / blockDim.x, l0 = threadIdx.x * chunk, l1 = min(L, l0 + chunk);
        int c = 0;
        for (int l = l0; l < l1; ++l) {
            if (cnt[l] < m) continue;
            c += (l == 0 || cnt[l - 1] < m) ? 1 : 0;
            c += (l + 1 == L || cnt[l + 1] < m) ? 1 << 16 : 0;
        }
        int o = cta_scan(c, s_scan, &total);
        int os = o & 0xffff, oe = o >> 16;
        for (int l = l0; l < l1; ++l) {
            if (cnt[l] < m) continue;
            if (l == 0 || cnt[l - 1] < m) ra[os++] = l;
            if (l + 1 == L || cnt[l + 1] < m) rb[oe++] = l + 1;
        }
    }
    const int n = total & 0xffff;
    if (n == 0) {
        if (threadIdx.x == 0) cb.nruns[j] = 0;
        return;
    }
    __syncthreads();
    const int G = b.gap > 0 ? b.gap : max(1, cta_lower_median(ra, rb, n, L, s_scan) / 4);
    int nm;
    {
        const int chunk = (n + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * chunk, j1 = min(n, j0 + chunk);
        int c = 0;
        for (int k = j0; k < j1; ++k) c += k == 0 || ra[k] - rb[k - 1] > G;
        int g = cta_scan(c, s_scan, &nm) - 1;
        for (int k = j0; k < j1; ++k) {
            if (k == 0 || ra[k] - rb[k - 1] > G) ma[++g] = ra[k];
            if (k + 1 == n || ra[k + 1] - rb[k] > G) mb[g] = rb[k];
        }
    }
    __syncthreads();
    const int mh = b.min_height > 0 ? b.min_height : max(2, cta_lower_median(ma, mb, nm, L, s_scan) / 3);
    int nk;
    {
        const int chunk = (nm + blockDim.x - 1) / blockDim.x, j0 = threadIdx.x * chunk, j1 = min(nm, j0 + chunk);
        int c = 0;
        for (int k = j0; k < j1; ++k) c += mb[k] - ma[k] >= mh;
        int k = cta_scan(c, s_scan, &nk);
        if (nk > MN_CURVE_RUN_CAP) {
            if (threadIdx.x == 0) cb.nruns[j] = -nk;
            return;
        }
        for (int e = j0; e < j1; ++e) {
            if (mb[e] - ma[e] < mh) continue;
            s_a[k] = ma[e];
            s_b[k++] = mb[e];
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = warp; k < nk; k += blockDim.x >> 5) {
        int lo = 0, hi = 0;
        for (int l = s_a[k] + lane; l < s_b[k]; l += 32) {
            lo = max(lo, cnt[L + l]);
            hi = max(hi, cnt[2 * L + l]);
        }
        lo = (int)__reduce_max_sync(0xffffffffu, (unsigned)lo);
        hi = (int)__reduce_max_sync(0xffffffffu, (unsigned)hi);
        if (lane == 0) {
            int* r = cb.runs + ((long long)j * MN_CURVE_RUN_CAP + k) * 4;
            r[0] = s_a[k]; r[1] = s_b[k]; r[2] = b.w - lo; r[3] = hi - 1;
        }
    }
    if (threadIdx.x == 0) cb.nruns[j] = nk;
}

__device__ __forceinline__ int run_overlap(int a, int b, int a2, int b2) { return min(b, b2) - max(a, a2); }

// The link of one block: strip by strip, every run of the strip and every open line in parallel (one thread each), the new
// lines numbered in run order with a CTA scan; then the kept lines ranked, the median run height and the table.
__global__ void __launch_bounds__(kLinkThreads) curve_link_kernel(const mn_curve_block* __restrict__ curves) {
    mn_pdl_prologue();
    __shared__ int s_scan[32];
    __shared__ int s_act[kLinkActive];
    __shared__ int s_best[MN_CURVE_RUN_CAP];
    __shared__ int s_err;
    const mn_curve_block& cb = curves[blockIdx.x];      // read in place: a copy would not fit the 64 registers of 1024 threads
    const int n_s = cb.n_strips, cap = n_s * MN_CURVE_RUN_CAP, tid = threadIdx.x;
    int* hd = cb.cout->header;
    // per line: last strip, last run's a and b, runs, first run's a, its best run in the strip (then its rank, -1: dropped);
    // per (strip, run): its line.  One base pointer: seven would not fit the 64 registers of 1024 threads.
    int* lk = cb.link;
#define last_j(l) lk[(l)]
#define last_a(l) lk[cap + (l)]
#define last_b(l) lk[2 * cap + (l)]
#define count(l) lk[3 * cap + (l)]
#define first_a(l) lk[4 * cap + (l)]
#define rank(l) lk[5 * cap + (l)]
#define run_line(e) lk[6 * cap + (e)]
    if (tid == 0) {
        s_err = -1;
        for (int j = 0; j < n_s && s_err < 0; ++j) {
            if (cb.nruns[j] < 0) s_err = j;
        }
        if (s_err >= 0) {
            hd[0] = MN_CURVE_ERR_RUNS; hd[1] = 0; hd[2] = 0; hd[3] = s_err; hd[4] = -cb.nruns[s_err];
            hd[5] = hd[6] = hd[7] = 0;
        }
    }
    __syncthreads();
    if (s_err >= 0) return;
    int n_lines = 0, n_act = 0;
    for (int j = 0; j < n_s; ++j) {
        const int R = cb.nruns[j];
        const int* runs = cb.runs + (long long)j * MN_CURVE_RUN_CAP * 4;
        if (tid < R) {                                  // this run's line
            const int a = runs[4 * tid], e = runs[4 * tid + 1];
            int best = -1, bo = 0, ba = 0;
            for (int q = 0; q < n_act; ++q) {
                const int l = s_act[q], la = last_a(l), o = run_overlap(a, e, la, last_b(l));
                if (o > bo || (o == bo && o > 0 && (la < ba || (la == ba && l < best)))) {
                    best = l; bo = o; ba = la;
                }
            }
            s_best[tid] = best;
        }
        if (tid < n_act) {                              // this line's run
            const int l = s_act[tid], la = last_a(l), lb = last_b(l);
            int best = -1, bo = 0;
            for (int k = 0; k < R; ++k) {
                const int o = run_overlap(runs[4 * k], runs[4 * k + 1], la, lb);
                if (o > bo) { best = k; bo = o; }
            }
            rank(l) = best;
        }
        __syncthreads();
        const int l = tid < R ? s_best[tid] : -1;
        const bool cont = l >= 0 && rank(l) == tid;
        int fresh;
        const int id = n_lines + cta_scan(tid < R && !cont ? 1 : 0, s_scan, &fresh);
        if (tid < R) {
            const int a = runs[4 * tid], e = runs[4 * tid + 1], dst = cont ? l : id;
            last_j(dst) = j; last_a(dst) = a; last_b(dst) = e;
            count(dst) = cont ? count(dst) + 1 : 1;
            if (!cont) first_a(dst) = a;
            run_line(j * MN_CURVE_RUN_CAP + tid) = dst;
        }
        __syncthreads();
        // the lines open for strip j + 1: the open ones, then the new ones, whose last run lies at most MN_CURVE_MAX_GAP back
        const int cand = tid < n_act ? s_act[tid] : tid < n_act + fresh ? n_lines + tid - n_act : -1;
        const bool keep = cand >= 0 && last_j(cand) >= j - MN_CURVE_MAX_GAP;
        int n_next;
        const int o = cta_scan(keep ? 1 : 0, s_scan, &n_next);
        if (keep) s_act[o] = cand;
        n_lines += fresh;
        n_act = n_next;
        __syncthreads();
    }
    // drop the short lines, rank the rest by (first run's a, line)
    const int need = (n_s + 3) / 4;
    int kept = 0;
    for (int l = tid; l < n_lines; l += blockDim.x) {
        if (count(l) < need) {
            rank(l) = -1;
            continue;
        }
        ++kept;
        int r = 0;
        for (int m = 0; m < n_lines; ++m) {
            r += count(m) >= need && (first_a(m) < first_a(l) || (first_a(m) == first_a(l) && m < l));
        }
        rank(l) = r;
    }
    int n_kept;
    cta_scan(kept, s_scan, &n_kept);
    if (n_kept > MN_BLOCK_MAX_LINES) {
        if (tid == 0) {
            hd[0] = MN_CURVE_ERR_LINES; hd[1] = 0; hd[2] = 0; hd[3] = 0; hd[4] = n_kept;
            hd[5] = hd[6] = hd[7] = 0;
        }
        return;
    }
    // Hm: the lower median of the kept runs' heights, by bisection over [1, h]
    const int n_all = n_s * MN_CURVE_RUN_CAP;
    int n_runs = 0;
    for (int e = tid; e < n_all; e += blockDim.x) {
        const int j = e / MN_CURVE_RUN_CAP, k = e % MN_CURVE_RUN_CAP;
        n_runs += k < cb.nruns[j] && rank(run_line(e)) >= 0;
    }
    int total;
    cta_scan(n_runs, s_scan, &total);
    int lo = 1, hi = cb.b.h;
    while (total && lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        int c = 0, below;
        for (int e = tid; e < n_all; e += blockDim.x) {
            const int j = e / MN_CURVE_RUN_CAP, k = e % MN_CURVE_RUN_CAP;
            if (k < cb.nruns[j] && rank(run_line(e)) >= 0) c += cb.runs[4 * e + 1] - cb.runs[4 * e] <= mid;
        }
        cta_scan(c, s_scan, &below);
        if (below > (total - 1) / 2) hi = mid; else lo = mid + 1;
    }
    const int med = total ? lo : 0;
    for (int e = tid; e < n_kept * MN_CURVE_LINE_INTS; e += blockDim.x) {
        const int f = e % MN_CURVE_LINE_INTS;
        cb.cout->line[e / MN_CURVE_LINE_INTS][f] = f == 0 ? MN_CURVE_MAX_STRIPS : f == 3 ? 0x7fffffff : f >= 6 && f < 8 ? 0 :
                                                    f == 5 ? 0 : -1;
    }
    __syncthreads();
    for (int l = tid; l < n_lines; l += blockDim.x) {
        if (rank(l) >= 0) cb.cout->line[rank(l)][2] = count(l);
    }
    for (int e = tid; e < n_all; e += blockDim.x) {
        const int j = e / MN_CURVE_RUN_CAP, k = e % MN_CURVE_RUN_CAP;
        if (k >= cb.nruns[j] || rank(run_line(e)) < 0) continue;
        const int* r = cb.runs + 4 * e;
        int* row = cb.cout->line[rank(run_line(e))];
        row[8 + 2 * j] = r[0];
        row[9 + 2 * j] = r[1];
        atomicMin(&row[0], j);
        atomicMax(&row[1], j);
        atomicMin(&row[3], r[2]);
        atomicMax(&row[4], r[3]);
        if (2 * (r[1] - r[0]) <= 3 * med) atomicOr(&row[5], 1 << j);
    }
    if (tid == 0) {
        hd[0] = 0; hd[1] = n_kept; hd[2] = med; hd[3] = hd[4] = hd[5] = hd[6] = hd[7] = 0;
    }
#undef last_j
#undef last_a
#undef last_b
#undef count
#undef first_a
#undef rank
#undef run_line
}

// ---- Skewed blocks (DESIGN.md 7b, "Skewed blocks") ----
// Every frame quantity is fp64 with each operation rounded on its own, as in the twin (oracle/skewed_blocks.py).  A tile of
// 32 x 32 pixels spans at most floor(31 (|c| + |s|)) + 2 <= 45 bins at |angle| < 45 degrees; kBins leaves room, and a bin outside
// it (which the bound rules out) would go straight to the global profile.
constexpr int kBins = 64;
constexpr int kScoreThreads = 1024;

struct frame_t {
    double u_min, v_min;
    int L, M;
};

// Pixel centre x + 0.5 - n / 2 of index x on an axis of n pixels: exact in fp64.
__device__ __forceinline__ double centre(int x, int n) { return (double)(2 * x + 1 - n) * 0.5; }
__device__ __forceinline__ double frame_u(double X, double Y, double c, double s) {
    return __dsub_rn(__dmul_rn(X, c), __dmul_rn(Y, s));
}
__device__ __forceinline__ double frame_v(double X, double Y, double c, double s) {
    return __dadd_rn(__dmul_rn(X, s), __dmul_rn(Y, c));
}
__device__ __forceinline__ int frame_bin(double v, double v_min, int L) {
    return min(max((int)floor(__dsub_rn(v, v_min)), 0), L - 1);
}

// The crop's frame dimensions: wt x ht, transposed for a vertical block.
__device__ __forceinline__ void frame_dims(const mn_text_block& b, int& wt, int& ht) {
    wt = b.vertical ? b.h : b.w;
    ht = b.vertical ? b.w : b.h;
}

__device__ frame_t frame_of(int wt, int ht, double c, double s) {
    const double xs[2] = {centre(0, wt), centre(wt - 1, wt)}, ys[2] = {centre(0, ht), centre(ht - 1, ht)};
    double u_lo = 0, u_hi = 0, v_lo = 0, v_hi = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const double u = frame_u(xs[q & 1], ys[q >> 1], c, s), v = frame_v(xs[q & 1], ys[q >> 1], c, s);
        u_lo = q ? fmin(u_lo, u) : u;
        u_hi = q ? fmax(u_hi, u) : u;
        v_lo = q ? fmin(v_lo, v) : v;
        v_hi = q ? fmax(v_hi, v) : v;
    }
    frame_t f;
    f.u_min = u_lo;
    f.v_min = v_lo;
    f.L = (int)floor(__dsub_rn(v_hi, v_lo)) + 1;
    f.M = (int)floor(__dsub_rn(u_hi, u_lo)) + 1;
    return f;
}

// The tile's ink as 32 frame rows of bits: s_row[r] bit j = ink at frame pixel (fx0 + j, fy0 + r), where (fx0, fy0) is the
// tile's origin in the frame ((tx, ty), or (ty, tx) for a vertical block).  s_m: 32 words of scratch.  Ends with a barrier.
__device__ void tile_ink_rows(const mn_text_block& b, int tx, int ty, unsigned* s_m, unsigned* s_row) {
    const int t = b.out->threshold;
    const bool dark = b.out->ink == MN_INK_DARK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, x = tx + lane;
    for (int j = 0; j < kTile / 8; ++j) {
        const int y = ty + warp + 8 * j;
        bool ink = false;
        if (x < b.w && y < b.h) {
            const int g = block_grey(b, x, y);
            ink = dark ? g <= t : g > t;
        }
        const unsigned m = __ballot_sync(0xffffffffu, ink);
        if (lane == 0) (b.vertical ? s_m : s_row)[warp + 8 * j] = m;
    }
    if (b.vertical) {
        __syncthreads();
        if (warp == 0) {                                // transpose: frame row r is the tile's column r
            unsigned r = 0;
            for (int y = 0; y < kTile; ++y) r |= ((s_m[y] >> lane) & 1u) << y;
            s_row[lane] = r;
        }
    }
    __syncthreads();
}

// The least bin of a tile of frame pixels [fx0, fx0 + nx) x [fy0, fy0 + ny): v is monotone in X and in Y (each rounded operation
// is), so it is the least of the four corners' bins.
__device__ __forceinline__ int tile_bin0(int fx0, int fy0, int nx, int ny, int wt, int ht, double c, double s, double v_min, int L) {
    int k = L;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const double X = centre(fx0 + (q & 1) * (nx - 1), wt), Y = centre(fy0 + (q >> 1) * (ny - 1), ht);
        k = min(k, frame_bin(frame_v(X, Y, c, s), v_min, L));
    }
    return k;
}

// 3. Angle profiles: each warp takes angles warp, warp + 8, ...; lane r walks frame row r of the tile, counting runs of equal
// bins before adding them into the warp's shared bins, which then go to the angle's profile with one atomic per non-zero bin.
__global__ void __launch_bounds__(kTileThreads) skew_angle_profile_kernel(const mn_skew_block* __restrict__ blocks) {
    mn_pdl_prologue();
    __shared__ unsigned s_m[kTile], s_row[kTile];
    __shared__ int s_bins[kTileThreads / 32][kBins];
    const mn_skew_block& sb = blocks[blockIdx.y];
    const mn_text_block b = sb.b;
    const int n_ang = sb.n_ang, stride = sb.stride;
    if (n_ang < 2) return;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    tile_ink_rows(b, tx, ty, s_m, s_row);
    int wt, ht;
    frame_dims(b, wt, ht);
    const int fx0 = b.vertical ? ty : tx, fy0 = b.vertical ? tx : ty;
    const int nx = min(kTile, wt - fx0), ny = min(kTile, ht - fy0);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned row = lane < ny ? s_row[lane] : 0u;
    const double Y = centre(fy0 + lane, ht);
    int* bins = s_bins[warp];
    for (int a = warp; a < n_ang; a += kTileThreads / 32) {
        const double c = sb.table[2 * a], s = sb.table[2 * a + 1];
        const frame_t f = frame_of(wt, ht, c, s);
        const int k0 = tile_bin0(fx0, fy0, nx, ny, wt, ht, c, s, f.v_min, f.L);
        int* prof = sb.profiles + (long long)a * stride;
        bins[lane] = bins[lane + 32] = 0;
        __syncwarp();
        const double yc = __dmul_rn(Y, c);
        int cur = -1, cnt = 0;
        for (unsigned m = row; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const int k = frame_bin(__dadd_rn(__dmul_rn(centre(fx0 + j, wt), s), yc), f.v_min, f.L);
            if (k != cur) {
                if (cnt) {
                    if (cur - k0 >= 0 && cur - k0 < kBins) atomicAdd(&bins[cur - k0], cnt); else atomicAdd(&prof[cur], cnt);
                }
                cur = k;
                cnt = 0;
            }
            ++cnt;
        }
        if (cnt) {
            if (cur - k0 >= 0 && cur - k0 < kBins) atomicAdd(&bins[cur - k0], cnt); else atomicAdd(&prof[cur], cnt);
        }
        __syncwarp();
        for (int d = lane; d < kBins; d += 32) {
            if (bins[d]) atomicAdd(&prof[k0 + d], bins[d]);
        }
        __syncwarp();
    }
}

// Is (score sa, index a) ahead of (sb, b)?  The larger score; ties to the least |index - mid|, then the least index.
__device__ __forceinline__ bool ahead(long long sa, int a, long long sb, int b, int mid) {
    if (sa != sb) return sa > sb;
    const int da = abs(a - mid), db = abs(b - mid);
    return da != db ? da < db : a < b;
}

// 4. Scores and the chosen angle, one CTA per block: one warp per angle, then a CTA-wide argmax.  Writes the chosen frame into
// the skew record, and, for a frame that is not the crop's own (s != 0), the frame's record into blocks[] for the segmentation.
__global__ void __launch_bounds__(kScoreThreads) skew_score_kernel(mn_text_block* blocks, mn_skew_block* skew) {
    mn_pdl_prologue();
    __shared__ long long s_best[kScoreThreads / 32];
    __shared__ int s_arg[kScoreThreads / 32];
    mn_skew_block& sb = skew[blockIdx.x];
    const mn_text_block b = sb.b;
    const int n_ang = sb.n_ang, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, mid = (n_ang - 1) / 2;
    int wt, ht;
    frame_dims(b, wt, ht);
    int best = 0;
    if (n_ang > 1) {
        for (int a = warp; a < n_ang; a += kScoreThreads / 32) {
            const int L = frame_of(wt, ht, sb.table[2 * a], sb.table[2 * a + 1]).L;
            const int* r = sb.profiles + (long long)a * sb.stride;
            long long acc = 0;
            for (int k = lane; k + 1 < L; k += 32) {
                const long long d = (long long)r[k + 1] - r[k];
                acc += d * d;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) sb.scores[a] = acc;
        }
        __syncthreads();
        long long bs = -1;
        int ba = 0;
        for (int a = threadIdx.x; a < n_ang; a += kScoreThreads) {
            const long long v = sb.scores[a];
            if (bs < 0 || ahead(v, a, bs, ba, mid)) bs = v, ba = a;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const long long os = __shfl_xor_sync(0xffffffffu, bs, o);
            const int oa = __shfl_xor_sync(0xffffffffu, ba, o);
            if (os >= 0 && (bs < 0 || ahead(os, oa, bs, ba, mid))) bs = os, ba = oa;
        }
        if (lane == 0) s_best[warp] = bs, s_arg[warp] = ba;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < kScoreThreads / 32; ++w) {
                if (s_best[w] >= 0 && (bs < 0 || ahead(s_best[w], s_arg[w], bs, ba, mid))) bs = s_best[w], ba = s_arg[w];
            }
        }
        best = ba;
    }
    if (threadIdx.x != 0) return;
    const double c = sb.table[2 * best], s = sb.table[2 * best + 1];
    const frame_t f = frame_of(wt, ht, c, s);
    sb.chosen = best;
    sb.L = f.L;
    sb.M = f.M;
    sb.u_min = f.u_min;
    sb.v_min = f.v_min;
    sb.c = c;
    sb.s = s;
    if (s != 0.0) {                                     // the segmentation runs in the frame: its table holds frame indices
        mn_text_block g = b;
        g.x0 = g.y0 = 0;
        g.w = f.M;
        g.h = f.L;
        g.vertical = 0;
        blocks[blockIdx.x] = g;
    }
}

// 5. The chosen frame's profile over the tiles: per bin the ink count, M - the least j and the largest j + 1, gathered in
// shared memory and added into b.prof with one atomic per bin and quantity (mn_find_lines_u8's layout, L = the frame's).
__global__ void __launch_bounds__(kTileThreads) skew_profile_kernel(const mn_skew_block* __restrict__ blocks) {
    mn_pdl_prologue();
    __shared__ unsigned s_m[kTile], s_row[kTile];
    __shared__ int s_cnt[kBins], s_lo[kBins], s_hi[kBins];
    const mn_skew_block& sb = blocks[blockIdx.y];
    const mn_text_block b = sb.b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    if (threadIdx.x < kBins) s_cnt[threadIdx.x] = s_lo[threadIdx.x] = s_hi[threadIdx.x] = 0;
    tile_ink_rows(b, tx, ty, s_m, s_row);
    int wt, ht;
    frame_dims(b, wt, ht);
    const int fx0 = b.vertical ? ty : tx, fy0 = b.vertical ? tx : ty;
    const int nx = min(kTile, wt - fx0), ny = min(kTile, ht - fy0);
    const double c = sb.c, s = sb.s, u_min = sb.u_min, v_min = sb.v_min;
    const int L = sb.L, M = sb.M;
    const int k0 = tile_bin0(fx0, fy0, nx, ny, wt, ht, c, s, v_min, L);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double X = centre(fx0 + lane, wt);
    for (int r = warp; r < ny; r += kTileThreads / 32) {
        if (!((s_row[r] >> lane) & 1u)) continue;
        const double Y = centre(fy0 + r, ht);
        const int k = frame_bin(frame_v(X, Y, c, s), v_min, L);
        const int j = min(max((int)floor(__dsub_rn(frame_u(X, Y, c, s), u_min)), 0), M - 1);
        if (k - k0 >= 0 && k - k0 < kBins) {
            atomicAdd(&s_cnt[k - k0], 1);
            atomicMax(&s_lo[k - k0], M - j);
            atomicMax(&s_hi[k - k0], j + 1);
        } else {
            atomicAdd(&b.prof[k], 1);
            atomicMax(&b.prof[L + k], M - j);
            atomicMax(&b.prof[2 * L + k], j + 1);
        }
    }
    __syncthreads();
    if (threadIdx.x < kBins && s_cnt[threadIdx.x]) {
        const int k = k0 + threadIdx.x;
        atomicAdd(&b.prof[k], s_cnt[threadIdx.x]);
        atomicMax(&b.prof[L + k], s_lo[threadIdx.x]);
        atomicMax(&b.prof[2 * L + k], s_hi[threadIdx.x]);
    }
}

// ---- Text pages (DESIGN.md 7b, "Text pages") ----
// A recursive XY-cut run level by level over every page of a call: the ink is classified once into a bitmap, and each level
// runs an attempt on every open node (one CTA per node, grid-stride), a per-page scan of the child counts and an ordered emit.
// The twin is oracle/pages.py.
constexpr int kPageThreads = 256;
constexpr int kChunk = 4096;                           // profile values counted at a time
constexpr int kSpanWords = 1024;                       // one bit per index of a span of at most 32767
constexpr int kScanThreads = 1024;

struct page_smem {
    int cnt[kChunk];                                   // ink count, plus the U count << 16 on a ruled page
    unsigned nw[kSpanWords];                           // bit i: index lo + i of the node's span is not white
    unsigned ru[kSpanWords];                           // bit i: index lo + i is a rule index (ruled pages only)
    int scan[32];
    int first;
};

__device__ __forceinline__ unsigned word_mask(int wd, int a, int b) {
    const int lo = max(a - (wd << 5), 0), hi = min(b - (wd << 5), 32);
    if (hi <= lo) return 0u;
    return (hi == 32 ? ~0u : (1u << hi) - 1u) & (~0u << lo);
}

// 3. The ink bitmap, one ballot per row of a 32 x 32 tile; tile 0 also writes the root node.
__global__ void __launch_bounds__(kTileThreads) page_bits_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    mn_text_page& p = pages[blockIdx.y];
    const mn_text_block& b = p.b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const int t = b.out->threshold;
    const bool dark = b.out->ink == MN_INK_DARK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, x = tx + lane;
    for (int j = 0; j < kTile / 8; ++j) {
        const int y = ty + warp + 8 * j;
        bool ink = false;
        if (x < b.w && y < b.h) {
            const int g = block_grey(b, x, y);
            ink = dark ? g <= t : g > t;
        }
        const unsigned m = __ballot_sync(0xffffffffu, ink);
        if (lane == 0 && y < b.h) p.bits[(long long)y * p.wpitch + (tx >> 5)] = m;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        mn_page_node r;
        r.x0 = 0; r.y0 = 0; r.x1 = (int16_t)b.w; r.y1 = (int16_t)b.h;
        r.st = b.vertical ? 0 : MN_PAGE_ROWS;
        p.list[0][0] = r;
        p.n[0] = 1;
        p.src = 0;
        p.open = 1;
        p.gx = p.gy = 1;
    }
}

// Exclusive max-scan of v over the CTA (-1 before the first thread); *total receives the maximum.  s holds 32 ints.
__device__ int cta_max_scan(int v, int* s, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x = max(x, y);
    }
    const int before = __shfl_up_sync(0xffffffffu, x, 1);
    if (lane == 31) s[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < n_warps ? s[lane] : -1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w = max(w, y);
        }
        s[lane] = w;
    }
    __syncthreads();
    const int pre = max(warp ? s[warp - 1] : -1, lane ? before : -1);
    *total = s[n_warps - 1];
    __syncthreads();
    return pre;
}

// The node's non-white indices along its axis into s.nw: index l is white iff its ink count < max(1, extent / 128), extent the
// node's length on the other axis.  On a ruled page its rule indices (2 u >= extent, u the U count) go to s.ru and are white
// too; counts fit 16 bits (<= 32767), so u rides in the high half of s.cnt.  Ends with a barrier.
__device__ __forceinline__ void node_profile(const mn_text_page& p, const mn_page_node& nd, bool rows, page_smem& s) {
    const int lo = rows ? nd.y0 : nd.x0, L = (rows ? nd.y1 : nd.x1) - lo;
    const int ext = rows ? nd.x1 - nd.x0 : nd.y1 - nd.y0, m = max(1, ext / 128);
    const bool ruled = p.rbits != nullptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    __syncthreads();                                    // the previous node's readers of s are done
    for (int j = threadIdx.x; j < kSpanWords; j += blockDim.x) {
        s.nw[j] = 0u;
        if (ruled) s.ru[j] = 0u;
    }
    for (int c0 = 0; c0 < L; c0 += kChunk) {
        const int n = min(kChunk, L - c0);
        if (rows) {
            const int wx0 = nd.x0 >> 5, wx1 = (nd.x1 - 1) >> 5;
            for (int r = warp; r < n; r += n_warps) {
                const long long o = (long long)(lo + c0 + r) * p.wpitch;
                int c = 0;
                for (int wd = wx0 + lane; wd <= wx1; wd += 32) {
                    const unsigned mk = word_mask(wd, nd.x0, nd.x1);
                    c += __popc(p.bits[o + wd] & mk);
                    if (ruled) c += __popc(p.rbits[o + wd] & mk) << 16;
                }
                c = (int)__reduce_add_sync(0xffffffffu, (unsigned)c);
                if (lane == 0) s.cnt[r] = c;
            }
        } else {
            for (int i = threadIdx.x; i < n; i += blockDim.x) s.cnt[i] = 0;
            __syncthreads();
            const int a = lo + c0, e = a + n, w0 = a >> 5, nwords = ((e - 1) >> 5) - w0 + 1;
            const int total = nwords * (nd.y1 - nd.y0);
            for (int k = threadIdx.x; k < total; k += blockDim.x) {
                const int y = nd.y0 + k / nwords, wd = w0 + k % nwords;
                for (unsigned v = p.bits[(long long)y * p.wpitch + wd] & word_mask(wd, a, e); v; v &= v - 1u)
                    atomicAdd(&s.cnt[(wd << 5) + __ffs(v) - 1 - a], 1);
                if (ruled) {
                    for (unsigned v = p.rbits[(long long)y * p.wpitch + wd] & word_mask(wd, a, e); v; v &= v - 1u)
                        atomicAdd(&s.cnt[(wd << 5) + __ffs(v) - 1 - a], 1 << 16);
                }
            }
        }
        __syncthreads();
        for (int j = threadIdx.x; 32 * j < n; j += blockDim.x) {
            unsigned v = 0u, r = 0u;
            for (int t = 0; t < 32 && 32 * j + t < n; ++t) {
                const int c = s.cnt[32 * j + t];
                const bool rule = ruled && 2 * (c >> 16) >= ext;
                v |= (unsigned)(!rule && (c & 0xffff) >= m) << t;
                r |= (unsigned)rule << t;
            }
            s.nw[(c0 >> 5) + j] = v;
            if (ruled) s.ru[(c0 >> 5) + j] = r;
        }
        __syncthreads();
    }
}

// Child c's start a along the axis, the other axis' span [o0, o1) and its state; child_end writes its end.
__device__ __forceinline__ void child_start(mn_page_node* c, bool rows, int a, int o0, int o1, int st) {
    if (rows) {
        c->y0 = (int16_t)a; c->x0 = (int16_t)o0; c->x1 = (int16_t)o1;
    } else {
        c->x0 = (int16_t)a; c->y0 = (int16_t)o0; c->y1 = (int16_t)o1;
    }
    c->st = st;
}
__device__ __forceinline__ void child_end(mn_page_node* c, bool rows, int e) {
    if (rows) c->y1 = (int16_t)e; else c->x1 = (int16_t)e;
}

// The last rule index before index b of word j (32 j <= b < 32 j + 32), lr the last one before word j (-1: none).
__device__ __forceinline__ int rule_before(unsigned ru, int j, int b, int lr) {
    const unsigned below = ru & ((1u << (b & 31)) - 1u);
    return below ? 32 * j + 31 - __clz(below) : lr;
}

// One attempt on the open node nd (every thread of the CTA): returns its number of children (0: dropped) and, in *n_open, how
// many of them stay open.  With kEmit, writes them into dst[0 ..) in reading order.  A white run between the non-white
// indices prev and b cuts when it is at least g long or, on a ruled page, holds a rule index (the last one before b > prev).
template <bool kEmit>
__device__ __forceinline__ int page_attempt(const mn_text_page& p, const mn_page_node& nd, bool last_level, page_smem& s, mn_page_node* dst,
                            int* n_open) {
    const bool rows = nd.st & MN_PAGE_ROWS;
    const int lo = rows ? nd.y0 : nd.x0, g = rows ? p.gy : p.gx;
    const int o0 = rows ? nd.x0 : nd.y0, o1 = rows ? nd.x1 : nd.y1, failed = nd.st & MN_PAGE_FAILED;
    const bool ruled = p.rbits != nullptr;
    if (threadIdx.x == 0) s.first = 1 << 30;
    node_profile(p, nd, rows, s);
    constexpr int kPer = kSpanWords / kPageThreads;
    const int j0 = threadIdx.x * kPer;
    int my_first = 1 << 30, my_last = -1, my_rule = -1;
    for (int j = j0; j < j0 + kPer; ++j) {
        const unsigned v = s.nw[j];
        if (v) {
            my_first = min(my_first, 32 * j + __ffs(v) - 1);
            my_last = 32 * j + 31 - __clz(v);
        }
        if (ruled && s.ru[j]) my_rule = 32 * j + 31 - __clz(s.ru[j]);
    }
    if (my_last >= 0) atomicMin(&s.first, my_first);
    int last, any_rule;
    const int prev0 = cta_max_scan(my_last, s.scan, &last);
    const int rule0 = ruled ? cta_max_scan(my_rule, s.scan, &any_rule) : -1;
    *n_open = 0;
    if (last < 0) return 0;
    const int first = s.first;
    int c = 0, prev = prev0, lr = rule0;
    for (int j = j0; j < j0 + kPer; ++j) {
        const unsigned ru = ruled ? s.ru[j] : 0u;
        for (unsigned v = s.nw[j]; v; v &= v - 1u) {
            const int b = 32 * j + __ffs(v) - 1;
            c += prev >= 0 && (b - prev - 1 >= g || rule_before(ru, j, b, lr) > prev);
            prev = b;
        }
        if (ru) lr = 32 * j + 31 - __clz(ru);
    }
    int cuts;
    int k = cta_scan(c, s.scan, &cuts);
    if (cuts == 0) {                                    // the trimmed node tries the other axis, or is a leaf
        const bool leaf = failed || last_level;
        if (kEmit && threadIdx.x == 0) {
            child_start(dst, rows, lo + first, o0, o1, (rows ? 0 : MN_PAGE_ROWS) | MN_PAGE_FAILED | (leaf ? MN_PAGE_LEAF : 0));
            child_end(dst, rows, lo + last + 1);
        }
        *n_open = leaf ? 0 : 1;
        return 1;
    }
    if (kEmit) {
        const bool rev = !rows && p.b.vertical;          // columns of a vertical page read right to left
        const int st = (rows ? 0 : MN_PAGE_ROWS) | (last_level ? MN_PAGE_LEAF : 0);
        prev = prev0;
        lr = rule0;
        for (int j = j0; j < j0 + kPer; ++j) {
            const unsigned ru = ruled ? s.ru[j] : 0u;
            for (unsigned v = s.nw[j]; v; v &= v - 1u) {
                const int b = 32 * j + __ffs(v) - 1;
                if (prev >= 0 && (b - prev - 1 >= g || rule_before(ru, j, b, lr) > prev)) {
                    child_end(dst + (rev ? cuts - k : k), rows, lo + prev + 1);
                    child_start(dst + (rev ? cuts - k - 1 : k + 1), rows, lo + b, o0, o1, st);
                    ++k;
                }
                prev = b;
            }
            if (ru) lr = 32 * j + 31 - __clz(ru);
        }
        if (threadIdx.x == 0) {
            child_start(dst + (rev ? cuts : 0), rows, lo + first, o0, o1, st);
            child_end(dst + (rev ? 0 : cuts), rows, lo + last + 1);
        }
    }
    *n_open = last_level ? 0 : cuts + 1;
    return cuts + 1;
}

// 4. Per node of page blockIdx.y's current list (grid-stride over blockIdx.x): its number of children (a leaf is carried as itself) and of open ones.
__global__ void __launch_bounds__(kPageThreads) page_count_kernel(mn_text_page* pages, int level) {
    mn_pdl_prologue();
    __shared__ page_smem s;
    const mn_text_page& p = pages[blockIdx.y];
    if (p.open == 0) return;
    const mn_page_node* list = p.list[p.src];
    const int n = p.n[p.src];
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const mn_page_node nd = list[i];
        int nch = 1, nop = 0;
        if (!(nd.st & MN_PAGE_LEAF)) nch = page_attempt<false>(p, nd, level + 1 == MN_PAGE_LEVELS, s, nullptr, &nop);
        if (threadIdx.x == 0) {
            p.nch[i] = nch;
            p.nopen[i] = nop;
        }
    }
}

// 5. Per page: the children's offsets in reading order, the next list's count and the node limit; flips the page's list.
__global__ void __launch_bounds__(kScanThreads) page_scan_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ int s_scan[32];
    mn_text_page& p = pages[blockIdx.x];
    const int open = p.open, src = p.src, n = p.n[src];
    if (open == 0) {
        if (threadIdx.x == 0) p.active = 0;
        return;
    }
    const int chunk = (n + blockDim.x - 1) / blockDim.x, i0 = threadIdx.x * chunk, i1 = min(n, i0 + chunk);
    int c = 0, o = 0;
    for (int i = i0; i < i1; ++i) {
        c += p.nch[i];
        o += p.nopen[i];
    }
    int total, total_open;
    int pre = cta_scan(c, s_scan, &total);
    cta_scan(o, s_scan, &total_open);
    for (int i = i0; i < i1; ++i) {
        p.off[i] = pre;
        pre += p.nch[i];
    }
    if (threadIdx.x != 0) return;
    if (total > min(MN_PAGE_MAX_NODES, p.cap)) {
        p.res->error = MN_PAGE_ERR_NODES;
        p.open = p.active = 0;
        p.n[src] = 0;
        return;
    }
    p.n[1 - src] = total;
    p.src = 1 - src;
    p.open = total_open;
    p.active = 1;
}

// 6. The ordered emit: every node writes its children at its offset into the other list.
__global__ void __launch_bounds__(kPageThreads, 1) page_emit_kernel(mn_text_page* pages, int level) {
    mn_pdl_prologue();
    __shared__ page_smem s;
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.active) return;
    const mn_page_node* list = p.list[1 - p.src];
    mn_page_node* dst = p.list[p.src];
    const int n = p.n[1 - p.src];
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const mn_page_node nd = list[i];
        const int o = p.off[i];
        if (nd.st & MN_PAGE_LEAF) {
            if (threadIdx.x == 0) dst[o] = nd;
        } else if (p.nch[i] > 0) {
            int nop;
            page_attempt<true>(p, nd, level + 1 == MN_PAGE_LEVELS, s, dst + o, &nop);
        }
    }
}

// A page node read through L2: the panel test's last CTA reads nodes other CTAs have just marked.
__device__ __forceinline__ mn_page_node load_node(const mn_page_node* a) {
    const int* q = reinterpret_cast<const int*>(a);
    const int v0 = __ldcg(q), v1 = __ldcg(q + 1), v2 = __ldcg(q + 2);
    mn_page_node g;
    g.x0 = (int16_t)(v0 & 0xffff); g.y0 = (int16_t)(v0 >> 16); g.x1 = (int16_t)(v1 & 0xffff); g.y1 = (int16_t)(v1 >> 16);
    g.st = v2;
    return g;
}

// The pass-1 leaves list[0 .. n) for which keep(leaf) holds, by the CTA, in leaf order into table (st: the rows of the entries
// before it), unless they are more than max: returns their number, and their rows in *rows.  Ends with a barrier.
template <class Keep>
__device__ int page_table(const mn_page_node* list, int n, Keep keep, mn_page_node* table, int max, int* s_scan, int* rows) {
    const int chunk = (n + blockDim.x - 1) / blockDim.x, i0 = threadIdx.x * chunk, i1 = min(n, i0 + chunk);
    int c = 0, r = 0, total;
    for (int i = i0; i < i1; ++i) {
        const mn_page_node g = load_node(list + i);
        if (!keep(g)) continue;
        ++c;
        r += g.y1 - g.y0;
    }
    int k = cta_scan(c, s_scan, &total);
    r = cta_scan(r, s_scan, rows);                      // disjoint, sides >= 2: at most w h / 2 rows
    if (total <= max) {
        for (int i = i0; i < i1; ++i) {
            mn_page_node g = load_node(list + i);
            if (!keep(g)) continue;
            g.st = r;
            table[k++] = g;
            r += g.y1 - g.y0;
        }
    }
    __syncthreads();                                    // list is read before the root overwrites it
    return total;
}

// The figures of a figure page (DESIGN.md 7b, "Figures"), by the CTA: its pass-1 leaves that are not panels and whose shorter
// side is at least f, into p.figs (page_table), their rows into p.frows and f and their number into res; over
// MN_PAGE_MAX_FIGURES the page error.  Returns false on that error.  Ends with a barrier.
__device__ bool page_figures(mn_text_page& p, const mn_page_node* list, int n, int S, int* s_scan) {
    const int f = p.figure_size > 0 ? p.figure_size : 3 * S;
    auto figure = [f](const mn_page_node& g) {          // a panel is never a figure
        return !(g.st & MN_PAGE_PANEL) && min(g.x1 - g.x0, g.y1 - g.y0) >= f;
    };
    int rows;
    const int total = page_table(list, n, figure, p.figs, MN_PAGE_MAX_FIGURES, s_scan, &rows);
    if (threadIdx.x == 0) {
        p.res->figure_size = f;
        p.res->n_figures = total;
        if (total > MN_PAGE_MAX_FIGURES) p.res->error = MN_PAGE_ERR_FIGURES;
        else p.frows = rows;
    }
    return total <= MN_PAGE_MAX_FIGURES;
}

// The gaps of pass 2 for the text size S, and its root (thread 0).
__device__ void page_root(mn_text_page& p, int S) {
    const int wide = S, narrow = max(1, S / 2);
    p.src = 0;
    p.gx = p.gap_x > 0 ? p.gap_x : p.b.vertical ? narrow : wide;
    p.gy = p.gap_y > 0 ? p.gap_y : p.b.vertical ? wide : narrow;
    p.res->text_size = S;
    p.res->gap_x = p.gx;
    p.res->gap_y = p.gy;
    mn_page_node r;
    r.x0 = 0; r.y0 = 0; r.x1 = (int16_t)p.b.w; r.y1 = (int16_t)p.b.h;
    r.st = p.b.vertical ? 0 : MN_PAGE_ROWS;
    p.list[0][0] = r;
    p.n[0] = 1;
    p.open = 1;
}

// 7. Text size S: the lower median of max(h, w) over the leaves with max(h, w) >= 2, by bisection over counts; the gaps of
// pass 2 and its root.  A page without such a leaf has no blocks; a figure page's figures are selected first.  A panel page
// with such a leaf keeps its pass-1 leaves: S and p go to res, and the panel test selects its panels and figures and writes
// the root.
__global__ void __launch_bounds__(kScanThreads) page_size_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ int s_scan[32];
    mn_text_page& p = pages[blockIdx.x];
    if (p.res->error) return;
    const mn_page_node* list = p.list[p.src];
    const int n = p.n[p.src];
    const int chunk = (n + blockDim.x - 1) / blockDim.x, i0 = threadIdx.x * chunk, i1 = min(n, i0 + chunk);
    auto size = [&](int i) { return max(list[i].x1 - list[i].x0, list[i].y1 - list[i].y0); };
    int c = 0, n2;
    for (int i = i0; i < i1; ++i) c += size(i) >= 2;
    cta_scan(c, s_scan, &n2);
    int lo = 2, hi = 32767;
    while (n2 > 0 && lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        int k = 0, t;
        for (int i = i0; i < i1; ++i) {
            const int v = size(i);
            k += v >= 2 && v <= mid;
        }
        cta_scan(k, s_scan, &t);
        if (t > (n2 - 1) / 2) hi = mid; else lo = mid + 1;
    }
    if (n2 > 0 && p.pans) {
        if (threadIdx.x == 0) {
            p.res->text_size = lo;
            p.res->panel_size = p.panel_size > 0 ? p.panel_size : lo;
        }
        return;
    }
    const bool ok = n2 == 0 || !p.fbits || page_figures(p, list, n, lo, s_scan);
    if (threadIdx.x != 0) return;
    if (n2 == 0 || !ok) {
        p.src = 0;
        p.n[0] = 0;
        p.open = 0;
        return;
    }
    page_root(p, lo);
}

// The greatest (kMin: least) row (kRows) or column of the rectangle [xa, xb) x [ya, yb) of a ruled or figure page that holds a
// pixel of U or F, over the warp: -1 (kMin: 1 << 30) when there is none.
template <bool kRows, bool kMin>
__device__ int rule_edge(const mn_text_page& p, int xa, int ya, int xb, int yb) {
    const int w0 = xa >> 5, nwords = xb > xa ? ((xb - 1) >> 5) - w0 + 1 : 0;
    int best = kMin ? 1 << 30 : -1;
    for (int k = threadIdx.x & 31; k < nwords * max(0, yb - ya); k += 32) {
        const int y = ya + k / nwords, wd = w0 + k % nwords;
        const long long o = (long long)y * p.wpitch + wd;
        const unsigned m = ((p.rbits ? p.rbits[o] : 0u) | (p.fbits ? p.fbits[o] : 0u)) & word_mask(wd, xa, xb);
        if (!m) continue;
        const int v = kRows ? y : kMin ? 32 * wd + __ffs(m) - 1 : 32 * wd + 31 - __clz(m);
        best = kMin ? min(best, v) : max(best, v);
    }
    return kMin ? __reduce_min_sync(0xffffffffu, best) : __reduce_max_sync(0xffffffffu, best);
}

// 11. The leaves, one warp each: rejected when 2 ink > h w or min(h, w) < max(1, S / 3), else a block grown by q and clipped;
// on a ruled or figure page each side stops short of the nearest row (column) of its margin with U or F in the leaf's columns
// (rows).
__global__ void __launch_bounds__(kScanThreads) page_blocks_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ int s_blocks;
    mn_text_page& p = pages[blockIdx.x];
    mn_page_result* res = p.res;
    if (threadIdx.x == 0) {
        s_blocks = 0;
        res->threshold = p.b.out->threshold;
        res->ink = p.b.out->ink;
    }
    __syncthreads();
    if (res->error) return;
    const mn_page_node* list = p.list[p.src];
    const int n = p.n[p.src], S = res->text_size;
    const int q = (min(p.gx, p.gy) - 1) / 2, min_side = max(1, S / 3);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = warp; i < n; i += blockDim.x >> 5) {
        mn_page_node nd = list[i];
        const int wx0 = nd.x0 >> 5, wx1 = (nd.x1 - 1) >> 5, nwords = wx1 - wx0 + 1;
        long long ink = 0;
        for (int k = lane; k < nwords * (nd.y1 - nd.y0); k += 32) {
            const int y = nd.y0 + k / nwords, wd = wx0 + k % nwords;
            ink += __popc(p.bits[(long long)y * p.wpitch + wd] & word_mask(wd, nd.x0, nd.x1));
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) ink += __shfl_xor_sync(0xffffffffu, ink, o);
        const int h = nd.y1 - nd.y0, w = nd.x1 - nd.x0;
        const bool reject = 2 * ink > (long long)h * w || min(h, w) < min_side;
        int x0 = max(0, nd.x0 - q), y0 = max(0, nd.y0 - q), x1 = min(p.b.w, nd.x1 + q), y1 = min(p.b.h, nd.y1 + q);
        if (!reject && (p.rbits || p.fbits)) {
            const int top = rule_edge<true, false>(p, nd.x0, y0, nd.x1, nd.y0);
            const int bottom = rule_edge<true, true>(p, nd.x0, nd.y1, nd.x1, y1);
            const int left = rule_edge<false, false>(p, x0, nd.y0, nd.x0, nd.y1);
            const int right = rule_edge<false, true>(p, nd.x1, nd.y0, x1, nd.y1);
            y0 = top >= 0 ? top + 1 : y0;
            y1 = min(y1, bottom);
            x0 = left >= 0 ? left + 1 : x0;
            x1 = min(x1, right);
        }
        if (lane != 0) continue;
        if (reject) {
            nd.st |= MN_PAGE_REJECTED;
        } else {
            nd.x0 = (int16_t)x0; nd.y0 = (int16_t)y0; nd.x1 = (int16_t)x1; nd.y1 = (int16_t)y1;
            atomicAdd(&s_blocks, 1);
        }
        p.leaves[i] = nd;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        res->n_leaves = n;
        res->n_blocks = s_blocks;
        if (s_blocks > MN_PAGE_MAX_BLOCKS) res->error = MN_PAGE_ERR_BLOCKS;
    }
}

// ---- Ruled pages (DESIGN.md 7b, "Ruled pages") ----
// U, the ink pixels in a maximal row or column run of at least rule_length, for every ruled page of a call in three launches:
// the bitmap transposed into the scratch plane after rbits (w rows of ceil(h / 32) words, so that columns are rows), the long
// runs of every row of both planes, and the column runs transposed back, OR'd into rbits and cleared from bits.  A row of up to
// 1024 words is one warp's: per-iteration summaries of its zeros and two warp scans give each word the ink runs that continue
// past its ends, so the work is O(1) per word for any rule length.  Pages without rbits return at once.
constexpr int kRuleThreads = 256;

__device__ __forceinline__ uint32_t* rule_plane(const mn_text_page& p) { return p.rbits + (long long)p.b.h * p.wpitch; }

// A 32 x 32 bit transpose across the warp: lane r holds row r; returns column `lane` (bit r = row r's bit lane).
__device__ __forceinline__ unsigned warp_transpose(unsigned v) {
    unsigned out = 0u;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
        const unsigned t = __ballot_sync(0xffffffffu, (v >> c) & 1u);
        if ((threadIdx.x & 31) == c) out = t;
    }
    return out;
}

// Max of v over the lanes below this one (INT_MIN for lane 0), and min over the lanes above (INT_MAX for lane 31).
__device__ __forceinline__ int warp_max_below(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = max(v, y);
    }
    const int e = __shfl_up_sync(0xffffffffu, v, 1);
    return lane ? e : INT_MIN;
}
__device__ __forceinline__ int warp_min_above(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < 32) v = min(v, y);
    }
    const int e = __shfl_down_sync(0xffffffffu, v, 1);
    return lane < 31 ? e : INT_MAX;
}

// The bits of the word v in runs of ones at least l long, the run at bit 0 continuing `before` ones below the word and the run
// at bit 31 `after` ones above it.
__device__ __forceinline__ unsigned long_runs(unsigned v, int before, int after, int l) {
    unsigned out = 0u;
    while (v) {
        const int a = __ffs(v) - 1;
        const unsigned rest = ~(v >> a);                // zero only for a = 0 and v all ones
        const int len = rest ? __ffs(rest) - 1 : 32;
        const unsigned run = (len == 32 ? ~0u : (1u << len) - 1u) << a;
        if (len + (a == 0 ? before : 0) + (a + len == 32 ? after : 0) >= l) out |= run;
        v &= ~run;
    }
    return out;
}

// One line of n bits in words src[0 .. ceil(n / 32)) (bits past n zero; outside the line is paper) by the warp: dst[k] = the
// bits of src[k] in maximal runs of at least l ones.  dst may be src.
__device__ __forceinline__ void line_runs(const uint32_t* src, uint32_t* dst, int n, int l) {
    const int lane = threadIdx.x & 31, nwords = (n + 31) >> 5, nit = (nwords + 31) >> 5;
    int lz = -1, fz = INT_MAX;                          // lane `it`: the last and first zero of iteration it's 32 words
    for (int it = 0; it < nit; ++it) {
        const int k = 32 * it + lane;
        const unsigned z = ~(k < nwords ? src[k] : 0u);
        const int a = __reduce_max_sync(0xffffffffu, z ? 32 * k + 31 - __clz(z) : -1);
        const int b = __reduce_min_sync(0xffffffffu, z ? 32 * k + __ffs(z) - 1 : INT_MAX);
        if (lane == it) {
            lz = a;
            fz = b;
        }
    }
    const int lz_before = max(-1, warp_max_below(lz)), fz_after = min(32 * nwords, warp_min_above(fz));
    for (int it = 0; it < nit; ++it) {
        const int k = 32 * it + lane;
        const unsigned v = k < nwords ? src[k] : 0u, z = ~v;
        const int zb = max(__shfl_sync(0xffffffffu, lz_before, it), warp_max_below(z ? 32 * k + 31 - __clz(z) : -1));
        const int za = min(__shfl_sync(0xffffffffu, fz_after, it), warp_min_above(z ? 32 * k + __ffs(z) - 1 : INT_MAX));
        const unsigned m = long_runs(v, 32 * k - zb - 1, za - 32 * k - 32, l);
        if (k < nwords) dst[k] = m;
    }
}

// R1. The bitmap's 32 x 32 tiles transposed into the scratch plane, one warp per tile.
__global__ void __launch_bounds__(kRuleThreads) rule_transpose_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.rbits || !p.rule_length) return;
    const int w = p.b.w, h = p.b.h, nw = (w + 31) >> 5, th = (h + 31) >> 5, lane = threadIdx.x & 31;
    constexpr int kWarps = kRuleThreads / 32;
    uint32_t* tp = rule_plane(p);
    for (long long t = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5); t < (long long)nw * th; t += (long long)gridDim.x * kWarps) {
        const int ty = (int)(t % th), wd = (int)(t / th), y = 32 * ty + lane, x = 32 * wd + lane;
        const unsigned c = warp_transpose(y < h ? p.bits[(long long)y * p.wpitch + wd] : 0u);
        if (x < w) tp[(long long)x * th + ty] = c;
    }
}

// R2. The long runs of the h rows of bits into rbits, and of the w rows of the scratch plane in place, one warp per row.
__global__ void __launch_bounds__(kRuleThreads, 1) rule_runs_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.rbits || !p.rule_length) return;
    const int w = p.b.w, h = p.b.h, th = (h + 31) >> 5;
    constexpr int kWarps = kRuleThreads / 32;
    uint32_t* tp = rule_plane(p);
    for (int i = blockIdx.x * kWarps + (threadIdx.x >> 5); i < h + w; i += gridDim.x * kWarps) {
        if (i < h) line_runs(p.bits + (long long)i * p.wpitch, p.rbits + (long long)i * p.wpitch, w, p.rule_length);
        else line_runs(tp + (long long)(i - h) * th, tp + (long long)(i - h) * th, h, p.rule_length);
    }
}

// R3. The column runs transposed back and OR'd into rbits (U), U cleared from bits (I' = I and not U), |U| into res.
__global__ void __launch_bounds__(kRuleThreads) rule_merge_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ int s_count;
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.rbits || !p.rule_length) return;
    const int w = p.b.w, h = p.b.h, nw = (w + 31) >> 5, th = (h + 31) >> 5, lane = threadIdx.x & 31;
    constexpr int kWarps = kRuleThreads / 32;
    const uint32_t* tp = rule_plane(p);
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    int count = 0;
    for (long long t = (long long)blockIdx.x * kWarps + (threadIdx.x >> 5); t < (long long)nw * th; t += (long long)gridDim.x * kWarps) {
        const int ty = (int)(t % th), wd = (int)(t / th), y = 32 * ty + lane, x = 32 * wd + lane;
        const unsigned r = warp_transpose(x < w ? tp[(long long)x * th + ty] : 0u);
        if (y < h) {
            const long long o = (long long)y * p.wpitch + wd;
            const unsigned u = p.rbits[o] | r;
            p.rbits[o] = u;
            p.bits[o] &= ~u;
            count += __popc(u);
        }
    }
    count = (int)__reduce_add_sync(0xffffffffu, (unsigned)count);
    if (lane == 0 && count) atomicAdd(&s_count, count);
    __syncthreads();
    if (threadIdx.x == 0 && s_count) atomicAdd(&p.res->rule_pixels, s_count);
}

// ---- Figures (DESIGN.md 7b, "Figures") ----
// F1. Every row of every figure of a figure page (page_figures' table), one warp each: its words OR'd into fbits (F) and cleared
// from bits (I'' = I' and not F).  Figures may share a word at their ends, hence the atomics.  Pages without fbits, and pages
// with an error, return at once.
constexpr int kFigureThreads = 256;

__global__ void __launch_bounds__(kFigureThreads) figure_paint_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.fbits || p.res->error) return;
    const int nf = p.res->n_figures, lane = threadIdx.x & 31;
    constexpr int kWarps = kFigureThreads / 32;
    for (int t = blockIdx.x * kWarps + (threadIdx.x >> 5); t < p.frows; t += gridDim.x * kWarps) {
        int lo = 0, hi = nf - 1;                        // the last figure whose first row index is <= t
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (p.figs[mid].st <= t) lo = mid; else hi = mid - 1;
        }
        const mn_page_node g = p.figs[lo];
        const long long o = (long long)(g.y0 + t - g.st) * p.wpitch;
        for (int wd = (g.x0 >> 5) + lane; wd <= (g.x1 - 1) >> 5; wd += 32) {
            const unsigned m = word_mask(wd, g.x0, g.x1);
            atomicOr(p.fbits + o + wd, m);
            atomicAnd(p.bits + o + wd, ~m);
        }
    }
}

// ---- Reversed panels (DESIGN.md 7b, "Reversed panels") ----
// P1. The panel test of every pass-1 leaf of a panel page whose shorter side is at least p, one CTA per leaf (grid-stride over
// blockIdx.x): its ink count |I' & leaf| and, when that is over half the rectangle, the 256-bin histogram of its greys, the
// mode m (ties to the smaller grey) and the flat count of greys in [m - 8, m + 8]; a panel iff the flat count is over half, and
// its st gains MN_PAGE_PANEL.  The last CTA of each page then lists its panels (st: the rows of the panels before it), selects
// its figures among the other leaves and writes the root of pass 2.  Pages without pans, without a text size or with an error
// return at once.
constexpr int kPanelFlat = 8;
constexpr int kPanelThreads = 1024;                   // 32 warps: the pixel loads of one large leaf in flight
constexpr int kPanelWarps = kPanelThreads / 32;
constexpr int kPanelUnroll = 8;

__device__ __forceinline__ long long cta_sum64(long long v, long long* s) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s[warp] = v;
    __syncthreads();
    long long t = 0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += s[k];
    return t;
}

__global__ void __launch_bounds__(kPanelThreads) panel_test_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ int s_hist[kPanelWarps * 256];
    __shared__ long long s_sum[kPanelWarps];
    __shared__ unsigned long long s_best[8];
    __shared__ int s_scan[32];
    __shared__ bool s_last;
    mn_text_page& p = pages[blockIdx.y];
    if (!p.pans || p.res->error || p.res->panel_size == 0) return;
    mn_page_node* list = p.list[p.src];
    const mn_text_block b = p.b;                        // the crop record in registers for the pixel loop
    const int n = p.n[p.src], P = p.res->panel_size, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const mn_page_node nd = list[i];
        const int h = nd.y1 - nd.y0, w = nd.x1 - nd.x0;
        if (min(h, w) < P) continue;
        const int wx0 = nd.x0 >> 5, nwords = ((nd.x1 - 1) >> 5) - wx0 + 1;
        long long ink = 0;                              // one warp per row
        for (int y = nd.y0 + warp; y < nd.y1; y += kPanelWarps) {
            for (int wd = wx0 + lane; wd < wx0 + nwords; wd += 32)
                ink += __popc(p.bits[(long long)y * p.wpitch + wd] & word_mask(wd, nd.x0, nd.x1));
        }
        const long long area = (long long)h * w;
        if (2 * cta_sum64(ink, s_sum) <= area) continue;
        for (int k = threadIdx.x; k < kPanelWarps * 256; k += blockDim.x) s_hist[k] = 0;
        __syncthreads();
        int* hist = s_hist + 256 * warp;                // one histogram per warp; each thread counts runs of its greys
        int cur = -1, run = 0;
        for (int y = nd.y0 + warp; y < nd.y1; y += kPanelWarps) {
            for (int x0 = nd.x0 + lane; x0 < nd.x1; x0 += 32 * kPanelUnroll) {
                int g[kPanelUnroll];                    // the loads of kPanelUnroll pixels in flight together
#pragma unroll
                for (int u = 0; u < kPanelUnroll; ++u) g[u] = x0 + 32 * u < nd.x1 ? block_grey(b, x0 + 32 * u, y) : -1;
#pragma unroll
                for (int u = 0; u < kPanelUnroll; ++u) {
                    if (g[u] < 0 || g[u] == cur) {
                        run += g[u] >= 0;
                        continue;
                    }
                    if (run) atomicAdd(hist + cur, run);
                    cur = g[u];
                    run = 1;
                }
            }
        }
        if (run) atomicAdd(hist + cur, run);
        __syncthreads();
        const int t = threadIdx.x;                      // threads 0 .. 255: the bins
        int v = 0;
        for (int k = 0; k < kPanelWarps && t < 256; ++k) v += s_hist[256 * k + t];
        __syncthreads();
        if (t < 256) s_hist[t] = v;
        __syncthreads();
        unsigned long long key = t < 256 ? ((unsigned long long)v << 8) | (255u - t) : 0ull;
#pragma unroll
        for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
        if (lane == 0 && warp < 8) s_best[warp] = key;
        __syncthreads();
        unsigned long long best = 0;
        for (int k = 0; k < 8; ++k) best = max(best, s_best[k]);
        const int m = 255 - (int)(best & 255u);
        const long long flat = cta_sum64(t < 256 && abs(t - m) <= kPanelFlat ? v : 0, s_sum);
        if (threadIdx.x == 0 && 2 * flat > area) list[i].st = nd.st | MN_PAGE_PANEL;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();                                // this CTA's marks before its ticket
        s_last = atomicAdd(&p.pdone, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    int rows;
    auto panel = [](const mn_page_node& g) { return (g.st & MN_PAGE_PANEL) != 0; };
    const int total = page_table(list, n, panel, p.pans, MN_PAGE_MAX_PANELS, s_scan, &rows);
    const bool ok = total <= MN_PAGE_MAX_PANELS && (!p.fbits || page_figures(p, list, n, p.res->text_size, s_scan));
    if (threadIdx.x != 0) return;
    p.res->n_panels = total;
    if (total > MN_PAGE_MAX_PANELS) p.res->error = MN_PAGE_ERR_PANELS;
    if (!ok) {
        p.src = 0;
        p.n[0] = 0;
        p.open = 0;
        return;
    }
    p.prows = rows;
    page_root(p, p.res->text_size);
}

// P2. Every row of every panel of a panel page (panel_test_kernel's table), one warp each: its interior (the rectangle less its
// 1-pixel outline) inverted in bits, which holds I' = I and not U, to J = not I (its U pixels stay clear), and its outline
// cleared from bits and OR'd into rbits.  Panels may share a word at their ends, hence the atomics.  Pages without pans, and
// pages with an error, return at once.
__global__ void __launch_bounds__(kFigureThreads) panel_paint_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.pans || p.res->error) return;
    const int np = p.res->n_panels, lane = threadIdx.x & 31;
    constexpr int kWarps = kFigureThreads / 32;
    for (int t = blockIdx.x * kWarps + (threadIdx.x >> 5); t < p.prows; t += gridDim.x * kWarps) {
        int lo = 0, hi = np - 1;                        // the last panel whose first row index is <= t
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (p.pans[mid].st <= t) lo = mid; else hi = mid - 1;
        }
        const mn_page_node g = p.pans[lo];
        const int y = g.y0 + t - g.st;
        const bool edge_row = y == g.y0 || y == g.y1 - 1;
        const long long o = (long long)y * p.wpitch;
        for (int wd = (g.x0 >> 5) + lane; wd <= (g.x1 - 1) >> 5; wd += 32) {
            const unsigned all = word_mask(wd, g.x0, g.x1);
            const unsigned inner = edge_row ? 0u : word_mask(wd, g.x0 + 1, g.x1 - 1), edge = all & ~inner;
            if (inner) atomicXor(p.bits + o + wd, inner & ~p.rbits[o + wd]);
            if (edge) {
                atomicOr(p.rbits + o + wd, edge);
                atomicAnd(p.bits + o + wd, ~edge);
            }
        }
    }
}

// ---- Mixed directions (DESIGN.md 7b, "Mixed directions") ----
// The bands of a leaf along rows (or columns), by the CTA from node_profile's non-white bits: *n the number of maximal runs
// of non-white indices, *b the longest and *g the white indices between the first and the last non-white one.  A run's
// length at each of its indices is its distance to the last white index before it, carried across threads by a max-scan.
__device__ void leaf_bands(const mn_text_page& p, const mn_page_node& nd, bool rows, page_smem& s, int* n, int* b, int* g) {
    node_profile(p, nd, rows, s);
    constexpr int kPer = kSpanWords / kPageThreads;
    const int j0 = threadIdx.x * kPer;
    int my_n = 0, my_set = 0, my_first = -1, my_last = -1, my_white = -1, t;
    for (int j = j0; j < j0 + kPer; ++j) {
        const unsigned v = s.nw[j], carry = j ? s.nw[j - 1] >> 31 : 0u;
        my_n += __popc(v & ~((v << 1) | carry));         // the indices that start a band
        my_set += __popc(v);
        if (v && my_first < 0) my_first = 32 * j + __ffs(v) - 1;
        if (v) my_last = 32 * j + 31 - __clz(v);
        if (~v) my_white = 32 * j + 31 - __clz(~v);
    }
    int white = cta_max_scan(my_white, s.scan, &t), best = 0;
    for (int j = j0; j < j0 + kPer; ++j) {
        for (unsigned v = s.nw[j]; v; v &= v - 1u) {
            const int i = 32 * j + __ffs(v) - 1;
            if (i == 0 || !((s.nw[(i - 1) >> 5] >> ((i - 1) & 31)) & 1u)) white = i - 1;
            best = max(best, i - white);
        }
    }
    int set, first, last;
    cta_scan(my_n, s.scan, n);
    cta_scan(my_set, s.scan, &set);
    cta_max_scan(my_first < 0 ? -1 : kSpanWords * 32 - my_first, s.scan, &first);
    cta_max_scan(my_last, s.scan, &last);
    cta_max_scan(best, s.scan, b);
    *g = last < 0 ? 0 : last - (kSpanWords * 32 - first) + 1 - set;
}

// D1. The direction of every kept leaf of a direction page, one CTA per leaf (grid-stride over blockIdx.x): with its row bands
// (n_r, b_r, G_y) and column bands (n_c, b_c, G_x) on its ungrown h x w rectangle, horizontal iff A > B and vertical iff
// A < B for (A, B) = (w, h) when n_r = n_c = 1, (2 b_c, h) when n_r = 1 < n_c, (w, 2 b_r) when n_c = 1 < n_r and
// (G_y (n_c - 1), G_x (n_r - 1)) when both exceed 1 (the mean gaps between row bands and between column bands); otherwise
// (A = B, or no band) undecided, and the page's direction.  Pages without dirs, and pages with an error, return at once.
__global__ void __launch_bounds__(kPageThreads) page_direction_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ page_smem s;
    const mn_text_page& p = pages[blockIdx.y];
    if (!p.dirs || p.res->error) return;
    const mn_page_node* list = p.list[p.src];
    const int n = p.res->n_leaves;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int st = p.leaves[i].st;
        if (st & MN_PAGE_REJECTED) continue;
        const mn_page_node nd = list[i];
        int nr, br, gy, nc, bc, gx;
        leaf_bands(p, nd, true, s, &nr, &br, &gy);
        leaf_bands(p, nd, false, s, &nc, &bc, &gx);
        const long long h = nd.y1 - nd.y0, w = nd.x1 - nd.x0;
        long long a = 0, b = 0;
        if (nr == 1 && nc == 1) { a = w; b = h; }
        else if (nr == 1 && nc > 1) { a = 2ll * bc; b = h; }
        else if (nc == 1 && nr > 1) { a = w; b = 2ll * br; }
        else if (nr > 1 && nc > 1) { a = (long long)gy * (nc - 1); b = (long long)gx * (nr - 1); }
        if (threadIdx.x != 0) continue;
        const bool vertical = a == b ? p.b.vertical != 0 : a < b;
        p.leaves[i].st = st | (vertical ? MN_PAGE_VERTICAL : 0) | (a == b ? MN_PAGE_UNDECIDED : 0);
    }
}

// ---- Page turns (DESIGN.md 7b, "Page turns") ----
// A turn page's vote table: cap mn_page_turn entries at the first 16-byte boundary after its leaf table.
__device__ __forceinline__ mn_page_turn* turn_table(const mn_text_page& p) {
    return reinterpret_cast<mn_page_turn*>((reinterpret_cast<uintptr_t>(p.leaves + p.cap) + 15) & ~(uintptr_t)15);
}

// Exclusive max-scan of v over the CTA (0 before the first thread); *total receives the maximum.  s holds 32 values.
__device__ unsigned long long cta_max_scan64(unsigned long long v, unsigned long long* s, unsigned long long* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x = max(x, y);
    }
    const unsigned long long before = __shfl_up_sync(0xffffffffu, x, 1);
    if (lane == 31) s[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = lane < n_warps ? s[lane] : 0ull;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w = max(w, y);
        }
        s[lane] = w;
    }
    __syncthreads();
    const unsigned long long pre = max(warp ? s[warp - 1] : 0ull, lane ? before : 0ull);
    *total = s[n_warps - 1];
    __syncthreads();
    return pre;
}

// T1. The vote statistics of every kept leaf of a turn page, one CTA per leaf (grid-stride over blockIdx.x), after the
// direction launch: along the leaf's direction (rows when horizontal, columns when vertical) its bands are node_profile's
// maximal runs of non-white indices, and band k spans [lo_k, hi_k] across, the least and largest index of an ink bit of its
// rows (columns) inside the leaf.  Its table entry is (n, E_lo, E_hi): n bands, E_lo = sum (lo_k - min lo) and
// E_hi = sum (max hi - hi_k), all 0 without a band.  4096 indices at a time: each index's extent into shared memory (rows by a
// warp's ffs / clz over its words, columns by per-bit atomicMin / atomicMax), then each band's by a max-scan of the keys
// (w + 1) << 32 | value, w the last white index before it, which is constant along a band and grows from band to band.
// Pages without a vote table, and pages with an error, return at once.
__global__ void __launch_bounds__(kPageThreads) page_turn_kernel(mn_text_page* pages) {
    mn_pdl_prologue();
    __shared__ page_smem s;
    __shared__ int s_hi[kChunk];
    __shared__ unsigned long long s_key[32];
    __shared__ long long s_sum[32];
    const mn_text_page& p = pages[blockIdx.y];
    if (!(p.dirs & MN_PAGE_DIRS_TURN) || p.res->error) return;
    mn_page_turn* votes = turn_table(p);
    const mn_page_node* list = p.list[p.src];
    const int n = p.res->n_leaves;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    constexpr int kPer = kChunk / kPageThreads;
    constexpr int kFar = 32767;                         // lo is keyed as kFar - lo, so that the max-scan takes the least
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int st = p.leaves[i].st;
        if (st & MN_PAGE_REJECTED) continue;
        const mn_page_node nd = list[i];
        const bool rows = !(st & MN_PAGE_VERTICAL);
        node_profile(p, nd, rows, s);
        const int lo = rows ? nd.y0 : nd.x0, L = (rows ? nd.y1 : nd.x1) - lo;
        unsigned long long kl = 0, kh = 0;             // the keys carried from the chunks before
        int white = -1, nb = 0, min_lo = kFar, max_hi = -1;
        long long sum_lo = 0, sum_hi = 0;
        for (int c0 = 0; c0 < L; c0 += kChunk) {
            const int m = min(kChunk, L - c0);
            __syncthreads();                            // the previous chunk's readers of s.cnt and s_hi are done
            if (rows) {
                const int wx0 = nd.x0 >> 5, wx1 = (nd.x1 - 1) >> 5;
                for (int r = warp; r < m; r += n_warps) {
                    const long long o = (long long)(lo + c0 + r) * p.wpitch;
                    int f = 1 << 30, l = -1;
                    for (int wd = wx0 + lane; wd <= wx1; wd += 32) {
                        const unsigned v = p.bits[o + wd] & word_mask(wd, nd.x0, nd.x1);
                        if (v) {
                            f = min(f, 32 * wd + __ffs(v) - 1);
                            l = max(l, 32 * wd + 31 - __clz(v));
                        }
                    }
                    f = __reduce_min_sync(0xffffffffu, f);
                    l = __reduce_max_sync(0xffffffffu, l);
                    if (lane == 0) {
                        s.cnt[r] = f - nd.x0;
                        s_hi[r] = l - nd.x0;
                    }
                }
            } else {
                for (int j = threadIdx.x; j < m; j += blockDim.x) {
                    s.cnt[j] = kFar;
                    s_hi[j] = -1;
                }
                __syncthreads();
                const int a = lo + c0, e = a + m, w0 = a >> 5, nwords = ((e - 1) >> 5) - w0 + 1;
                const int total = nwords * (nd.y1 - nd.y0);
                for (int k = threadIdx.x; k < total; k += blockDim.x) {
                    const int y = nd.y0 + k / nwords, wd = w0 + k % nwords;
                    for (unsigned v = p.bits[(long long)y * p.wpitch + wd] & word_mask(wd, a, e); v; v &= v - 1u) {
                        const int c = (wd << 5) + __ffs(v) - 1 - a;
                        atomicMin(&s.cnt[c], y - nd.y0);
                        atomicMax(&s_hi[c], y - nd.y0);
                    }
                }
            }
            __syncthreads();
            const int j0 = threadIdx.x * kPer, j1 = min(j0 + kPer, m);
            auto inked = [&](int x) { return (s.nw[x >> 5] >> (x & 31)) & 1u; };
            int my_white = -1;
            unsigned long long my_kl = 0, my_kh = 0;
            for (int j = j0; j < j1; ++j)
                if (!inked(c0 + j)) my_white = c0 + j;
            int w_total;
            int w = max(white, cta_max_scan(my_white, s.scan, &w_total));
            const int w_in = w;
            for (int j = j0; j < j1; ++j) {
                if (!inked(c0 + j)) {
                    w = c0 + j;
                    continue;
                }
                const unsigned long long key = (unsigned long long)(w + 1) << 32;
                my_kl = max(my_kl, key | (unsigned)(kFar - s.cnt[j]));
                my_kh = max(my_kh, key | (unsigned)s_hi[j]);
            }
            unsigned long long tl, th;
            unsigned long long pl = max(kl, cta_max_scan64(my_kl, s_key, &tl));
            unsigned long long ph = max(kh, cta_max_scan64(my_kh, s_key, &th));
            w = w_in;
            for (int j = j0; j < j1; ++j) {
                const int x = c0 + j;
                if (!inked(x)) {
                    w = x;
                    continue;
                }
                const unsigned long long key = (unsigned long long)(w + 1) << 32;
                pl = max(pl, key | (unsigned)(kFar - s.cnt[j]));
                ph = max(ph, key | (unsigned)s_hi[j]);
                if (x + 1 == L || !inked(x + 1)) {      // the band ends here: its extent is complete
                    const int blo = kFar - (int)(pl & 0xffffffffull), bhi = (int)(ph & 0xffffffffull);
                    ++nb;
                    sum_lo += blo;
                    sum_hi += bhi;
                    min_lo = min(min_lo, blo);
                    max_hi = max(max_hi, bhi);
                }
            }
            kl = max(kl, tl);
            kh = max(kh, th);
            white = max(white, w_total);
        }
        int n_bands, far_lo, top_hi;
        cta_scan(nb, s.scan, &n_bands);
        cta_max_scan(kFar - min_lo, s.scan, &far_lo);
        cta_max_scan(max_hi, s.scan, &top_hi);
        const long long s_lo = cta_sum64(sum_lo, s_sum), s_hi_sum = cta_sum64(sum_hi, s_sum);
        if (threadIdx.x == 0) {
            mn_page_turn r;
            r.n_bands = n_bands;
            r.pad = 0;
            r.e_lo = n_bands ? s_lo - (long long)n_bands * (kFar - far_lo) : 0;
            r.e_hi = n_bands ? (long long)n_bands * top_hi - s_hi_sum : 0;
            votes[i] = r;
        }
    }
}

// ---- Skewed pages (DESIGN.md 7b, "Skewed pages") ----
// The page's angle is searched by the skewed-block kernels on its mn_skew_block record; the XY-cut then runs unchanged on a
// bitmap of frame cells, whose sides the page record takes.  A vertical page's bitmap is of the untransposed frame at the
// reported angle: with the rounded operations u(X, Y, c, -s) = v(Y, X, c, s) and v(X, Y, c, -s) = u(Y, X, c, s), so negating s
// on the untransposed crop swaps the axes of the transposed search frame exactly.

// 3'. The frame bitmap: every ink pixel sets its cell's bit (bit j & 31 of bits[k wpitch + j / 32]); tile 0 writes the root
// node and the frame's sides (M x L) into the page record.  At s = 0 the cell of (x, y) is (x, y): page_bits_kernel's words.
__global__ void __launch_bounds__(kTileThreads) page_frame_bits_kernel(mn_text_page* pages, const mn_skew_block* __restrict__ skew) {
    mn_pdl_prologue();
    mn_text_page& p = pages[blockIdx.y];
    const mn_skew_block& sb = skew[blockIdx.y];
    const mn_text_block b = sb.b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const double c = sb.c, s = b.vertical ? -sb.s : sb.s;
    const frame_t f = frame_of(b.w, b.h, c, s);
    const int t = b.out->threshold;
    const bool dark = b.out->ink == MN_INK_DARK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, x = tx + lane;
    const double X = centre(x, b.w);
    for (int j = 0; j < kTile / 8; ++j) {
        const int y = ty + warp + 8 * j;
        if (x >= b.w || y >= b.h) continue;
        const int g = block_grey(b, x, y);
        if (!(dark ? g <= t : g > t)) continue;
        const double Y = centre(y, b.h);
        const int k = frame_bin(frame_v(X, Y, c, s), f.v_min, f.L);
        const int i = min(max((int)floor(__dsub_rn(frame_u(X, Y, c, s), f.u_min)), 0), f.M - 1);
        atomicOr(&p.bits[(long long)k * p.wpitch + (i >> 5)], 1u << (i & 31));
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        mn_page_node r;
        r.x0 = 0; r.y0 = 0; r.x1 = (int16_t)f.M; r.y1 = (int16_t)f.L;
        r.st = b.vertical ? 0 : MN_PAGE_ROWS;
        p.b.w = f.M;
        p.b.h = f.L;
        p.list[0][0] = r;
        p.n[0] = 1;
        p.src = 0;
        p.open = 1;
        p.gx = p.gy = 1;
    }
}

// ---- Windowed blocks (DESIGN.md 7b, "Skewed pages") ----
// A block that is the pixels of its crop whose frame cell at a given angle lies in a window.  Its histogram and profile cover
// the tiles of the window's footprint and test every pixel's cell; the threshold and segmentation kernels run on the window's
// own frame record.

__device__ __forceinline__ bool window_tile(const mn_window_block& wb, int& tx, int& ty) {
    const int tiles_x = (wb.pw + kTile - 1) / kTile, tiles_y = (wb.ph + kTile - 1) / kTile;
    if ((long long)blockIdx.x >= (long long)tiles_x * tiles_y) return false;
    tx = wb.px0 + (int)(blockIdx.x % tiles_x) * kTile;
    ty = wb.py0 + (int)(blockIdx.x / tiles_x) * kTile;
    return true;
}

// The cell (k, j) of frame pixel (fx, fy); true when it lies in the window.
__device__ __forceinline__ bool window_cell(const mn_window_block& wb, const frame_t& f, int wt, int ht, int fx, int fy, int& k,
                                            int& j) {
    const double X = centre(fx, wt), Y = centre(fy, ht);
    k = frame_bin(frame_v(X, Y, wb.c, wb.s), f.v_min, f.L);
    j = min(max((int)floor(__dsub_rn(frame_u(X, Y, wb.c, wb.s), f.u_min)), 0), f.M - 1);
    return k >= wb.l0 && k < wb.l1 && j >= wb.c0 && j < wb.c1;
}

__global__ void __launch_bounds__(kTileThreads) window_hist_kernel(const mn_window_block* __restrict__ wins) {
    mn_pdl_prologue();
    __shared__ int s_hist[256];
    const mn_window_block& wb = wins[blockIdx.y];
    const mn_text_block b = wb.b;
    int tx, ty;
    if (!window_tile(wb, tx, ty)) return;
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    int wt, ht;
    frame_dims(b, wt, ht);
    const frame_t f = frame_of(wt, ht, wb.c, wb.s);
    const int x = tx + (threadIdx.x & 31);
    if (x < b.w) {
        for (int y = ty + (threadIdx.x >> 5); y < min(ty + kTile, b.h); y += 8) {
            int k, j;
            if (window_cell(wb, f, wt, ht, b.vertical ? y : x, b.vertical ? x : y, k, j)) atomicAdd(&s_hist[block_grey(b, x, y)], 1);
        }
    }
    __syncthreads();
    const int v = s_hist[threadIdx.x];
    if (v) atomicAdd(&b.hist[threadIdx.x], v);
}

// The window's profile in its own frame: bin k - l0, index j - c0, laid out as mn_find_lines_u8's (L = l1 - l0, M = c1 - c0).
__global__ void __launch_bounds__(kTileThreads) window_profile_kernel(const mn_window_block* __restrict__ wins) {
    mn_pdl_prologue();
    __shared__ unsigned s_m[kTile], s_row[kTile];
    __shared__ int s_cnt[kBins], s_lo[kBins], s_hi[kBins];
    const mn_window_block& wb = wins[blockIdx.y];
    const mn_text_block b = wb.b;
    int tx, ty;
    if (!window_tile(wb, tx, ty)) return;
    if (threadIdx.x < kBins) s_cnt[threadIdx.x] = s_lo[threadIdx.x] = s_hi[threadIdx.x] = 0;
    tile_ink_rows(b, tx, ty, s_m, s_row);
    int wt, ht;
    frame_dims(b, wt, ht);
    const int fx0 = b.vertical ? ty : tx, fy0 = b.vertical ? tx : ty;
    const int nx = min(kTile, wt - fx0), ny = min(kTile, ht - fy0);
    const frame_t f = frame_of(wt, ht, wb.c, wb.s);
    const int L = wb.l1 - wb.l0, M = wb.c1 - wb.c0;
    const int k0 = tile_bin0(fx0, fy0, nx, ny, wt, ht, wb.c, wb.s, f.v_min, f.L) - wb.l0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = warp; r < ny; r += kTileThreads / 32) {
        int k, j;
        if (!((s_row[r] >> lane) & 1u) || !window_cell(wb, f, wt, ht, fx0 + lane, fy0 + r, k, j)) continue;
        k -= wb.l0;
        j -= wb.c0;
        if (k - k0 >= 0 && k - k0 < kBins) {
            atomicAdd(&s_cnt[k - k0], 1);
            atomicMax(&s_lo[k - k0], M - j);
            atomicMax(&s_hi[k - k0], j + 1);
        } else {
            atomicAdd(&b.prof[k], 1);
            atomicMax(&b.prof[L + k], M - j);
            atomicMax(&b.prof[2 * L + k], j + 1);
        }
    }
    __syncthreads();
    if (threadIdx.x < kBins && s_cnt[threadIdx.x]) {
        const int k = k0 + threadIdx.x;
        atomicAdd(&b.prof[k], s_cnt[threadIdx.x]);
        atomicMax(&b.prof[L + k], s_lo[threadIdx.x]);
        atomicMax(&b.prof[2 * L + k], s_hi[threadIdx.x]);
    }
}

// Page corners (DESIGN.md 7b, "Perspective pages"): the paper's 4-connected components by label-equivalence union-find, whose
// roots are always the smallest index of their set (a union links the larger root under the smaller one), so the labels do
// not depend on scheduling; then the largest component's hull and its largest inscribed quad, exact in integers.
constexpr int kHullThreads = 1024;

__device__ __forceinline__ bool paper_at(const mn_text_block& b, int t, int x, int y) {
    const int g = block_grey(b, x, y);
    return b.polarity == MN_INK_LIGHT ? g <= t : g > t;
}

__device__ __forceinline__ int uf_find(const int* L, int x) {
    const volatile int* v = L;                          // other threads link and compress while this one walks
    for (int p = v[x]; p != x; p = v[x]) x = p;
    return x;
}

__device__ void uf_union(int* L, int a, int b) {
    for (;;) {
        a = uf_find(L, a);
        b = uf_find(L, b);
        if (a == b) return;
        if (a > b) {
            const int t = a;
            a = b;
            b = t;
        }
        const int old = atomicMin(&L[b], a);
        if (old == b) return;
        b = old;                                        // b was linked meanwhile: join its new root too
    }
}

__global__ void __launch_bounds__(kTileThreads) quad_label_local_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    __shared__ int s_l[kTile * kTile];
    const mn_text_block b = pages[blockIdx.y].b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const int t = b.out->threshold, lx = threadIdx.x & 31;
    for (int r = threadIdx.x >> 5; r < kTile; r += 8) {
        const int x = tx + lx, y = ty + r;
        s_l[r * kTile + lx] = x < b.w && y < b.h && paper_at(b, t, x, y) ? r * kTile + lx : -1;
    }
    __syncthreads();
    for (int r = threadIdx.x >> 5; r < kTile; r += 8) {
        const int k = r * kTile + lx;
        if (s_l[k] < 0) continue;
        if (lx > 0 && s_l[k - 1] >= 0) uf_union(s_l, k - 1, k);
        if (r > 0 && s_l[k - kTile] >= 0) uf_union(s_l, k - kTile, k);
    }
    __syncthreads();
    int* label = pages[blockIdx.y].label;
    for (int r = threadIdx.x >> 5; r < kTile; r += 8) {
        const int x = tx + lx, y = ty + r;
        if (x >= b.w || y >= b.h) continue;
        int v = -1;
        if (s_l[r * kTile + lx] >= 0) {
            const int root = uf_find(s_l, r * kTile + lx);
            v = (ty + root / kTile) * b.w + tx + root % kTile;
        }
        label[(long long)y * b.w + x] = v;
    }
}

// Thread k < 32 joins row k of the tile's left column to its left neighbour, thread 32 + k column k of its top row to the
// pixel above.
__global__ void __launch_bounds__(64) quad_label_border_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_text_block b = pages[blockIdx.y].b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const bool left = threadIdx.x < 32;
    const int k = threadIdx.x & 31, x = left ? tx : tx + k, y = left ? ty + k : ty;
    if ((left ? tx : ty) == 0 || x >= b.w || y >= b.h) return;
    int* label = pages[blockIdx.y].label;
    const int p = y * b.w + x, q = left ? p - 1 : p - b.w;
    if (label[p] >= 0 && label[q] >= 0) uf_union(label, q, p);
}

// Path compression, and each component's pixels counted at its root with one atomic per label and warp row.
__global__ void __launch_bounds__(kTileThreads) quad_label_count_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_text_block b = pages[blockIdx.y].b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    int* label = pages[blockIdx.y].label;
    int* count = pages[blockIdx.y].count;
    const int x = tx + (threadIdx.x & 31);
    for (int y = ty + (threadIdx.x >> 5); y < ty + kTile; y += 8) {
        int r = -1;
        if (x < b.w && y < b.h) {
            const int p = y * b.w + x;
            if (label[p] >= 0) {
                r = uf_find(label, p);
                label[p] = r;
            }
        }
        const unsigned same = __match_any_sync(0xffffffffu, r);
        if (r >= 0 && (int)(threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&count[r], __popc(same));
    }
}

__global__ void __launch_bounds__(kTileThreads) quad_pick_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_text_block b = pages[blockIdx.y].b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const int* label = pages[blockIdx.y].label;
    const int* count = pages[blockIdx.y].count;
    const int x = tx + (threadIdx.x & 31);
    unsigned long long key = 0;
    for (int y = ty + (threadIdx.x >> 5); y < min(ty + kTile, b.h) && x < b.w; y += 8) {
        const int p = y * b.w + x;
        if (label[p] == p) key = max(key, (unsigned long long)count[p] << 32 | (unsigned)~p);
    }
    for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    if ((threadIdx.x & 31) == 0 && key) atomicMax(pages[blockIdx.y].best, key);
}

__global__ void __launch_bounds__(kTileThreads) quad_rows_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_text_block b = pages[blockIdx.y].b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const unsigned long long best = *pages[blockIdx.y].best;
    if (!best) return;
    const int page = (int)~(unsigned)best;
    const int* label = pages[blockIdx.y].label;
    int* ext = pages[blockIdx.y].ext;
    const int x = tx + (threadIdx.x & 31);
    for (int y = ty + (threadIdx.x >> 5); y < min(ty + kTile, b.h); y += 8) {
        const bool in = x < b.w && label[y * b.w + x] == page;
        const unsigned lo = __reduce_max_sync(0xffffffffu, in ? (unsigned)(b.w - x) : 0u);
        const unsigned hi = __reduce_max_sync(0xffffffffu, in ? (unsigned)(x + 1) : 0u);
        if ((threadIdx.x & 31) == 0 && hi) {
            atomicMax(&ext[2 * y], (int)lo);
            atomicMax(&ext[2 * y + 1], (int)hi);
        }
    }
}

__device__ __forceinline__ long long cross3(int2 o, int2 a, int2 c) {
    return (long long)(a.x - o.x) * (c.y - o.y) - (long long)(a.y - o.y) * (c.x - o.x);
}

__device__ __forceinline__ long long tri2(const int2* v, int i, int m, int j) {
    const long long c = cross3(v[i], v[m], v[j]);
    return c < 0 ? -c : c;
}

// Point i of the rows' pixel-square corners, sorted by (y, x): y = y0 + i / 2, the left end (even i) or the right end (odd i)
// of rows y - 1 and y.
__device__ __forceinline__ int2 row_point(const int* ext, int w, int y0, int y1, int i) {
    const int y = y0 + (i >> 1);
    int v = 0;
    for (int r = max(y - 1, y0); r <= min(y, y1); ++r) v = max(v, ext[2 * r + (i & 1)]);
    return make_int2((i & 1) ? v : w - v, y);
}

__device__ __forceinline__ bool quad_before(long long a, int4 ia, long long b, int4 ib) {
    if (a != b) return a > b;
    if (ia.x != ib.x) return ia.x < ib.x;
    if (ia.y != ib.y) return ia.y < ib.y;
    if (ia.z != ib.z) return ia.z < ib.z;
    return ia.w < ib.w;
}

// One CTA per page: the monotone chain on one thread, then the O(k^2) quad search over the first index, each thread with two
// rotating apex pointers (on a strictly convex polygon the smallest apex of the largest triangle over a diagonal i-j moves
// forward with j), and a tree reduction.
__global__ void __launch_bounds__(kHullThreads) quad_hull_kernel(const mn_quad_page* __restrict__ pages) {
    mn_pdl_prologue();
    __shared__ long long s_area[kHullThreads];
    __shared__ int4 s_idx[kHullThreads];
    __shared__ int s_y0, s_y1, s_k;
    const mn_quad_page& pg = pages[blockIdx.x];
    const mn_text_block b = pg.b;
    mn_page_quad* res = pg.res;
    const unsigned long long best = *pg.best;
    const int* ext = pg.ext;
    int2* hull = reinterpret_cast<int2*>(pg.hull);
    if (threadIdx.x == 0) {
        s_y0 = b.h;
        s_y1 = -1;
        res->threshold = b.out->threshold;
        res->label = best ? (int)~(unsigned)best : -1;
        res->size = (int)(best >> 32);
    }
    __syncthreads();
    if (!best) return;
    for (int y = threadIdx.x; y < b.h; y += blockDim.x) {
        if (ext[2 * y + 1]) {
            atomicMin(&s_y0, y);
            atomicMax(&s_y1, y);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int y0 = s_y0, y1 = s_y1, n = 2 * (y1 - y0 + 2);
        int k = 0;
        for (int i = 0; i < n; ++i) {
            const int2 p = row_point(ext, b.w, y0, y1, i);
            while (k >= 2 && cross3(hull[k - 2], hull[k - 1], p) <= 0) --k;
            hull[k++] = p;
        }
        for (int i = n - 2, lo = k + 1; i >= 0; --i) {
            const int2 p = row_point(ext, b.w, y0, y1, i);
            while (k >= lo && cross3(hull[k - 2], hull[k - 1], p) <= 0) --k;
            hull[k++] = p;
        }
        s_k = k - 1;
        res->n_hull = k - 1;
    }
    __syncthreads();
    const int k = s_k;
    long long area = -1;
    int4 id = make_int4(0, 0, 0, 0);
    for (int i = threadIdx.x; i + 3 < k; i += blockDim.x) {
        int a = i + 1, c = i + 3;
        for (int j = i + 2; j + 1 < k; ++j) {
            while (a + 1 < j && tri2(hull, i, a + 1, j) > tri2(hull, i, a, j)) ++a;
            c = max(c, j + 1);
            while (c + 1 < k && tri2(hull, j, c + 1, i) > tri2(hull, j, c, i)) ++c;
            const long long s = tri2(hull, i, a, j) + tri2(hull, j, c, i);
            if (s > area) {
                area = s;
                id = make_int4(i, a, j, c);
            }
        }
    }
    s_area[threadIdx.x] = area;
    s_idx[threadIdx.x] = id;
    __syncthreads();
    for (int h = blockDim.x / 2; h; h >>= 1) {
        if (threadIdx.x < h && quad_before(s_area[threadIdx.x + h], s_idx[threadIdx.x + h], s_area[threadIdx.x], s_idx[threadIdx.x])) {
            s_area[threadIdx.x] = s_area[threadIdx.x + h];
            s_idx[threadIdx.x] = s_idx[threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int4 q = s_idx[0];
        const bool cw = cross3(hull[q.x], hull[q.y], hull[q.z]) > 0;   // clockwise on screen (y down)
        int2 c[4] = {hull[q.x], hull[cw ? q.y : q.w], hull[q.z], hull[cw ? q.w : q.y]};
        int s = 0, sx = c[0].x, sy = c[0].y;
#pragma unroll
        for (int m = 1; m < 4; ++m) {
            const int d = (c[m].x + c[m].y) - (sx + sy);
            if (d < 0 || (d == 0 && c[m].y < sy)) {
                s = m;
                sx = c[m].x;
                sy = c[m].y;
            }
        }
        res->area2 = s_area[0];
        res->idx[0] = q.x;
        res->idx[1] = q.y;
        res->idx[2] = q.z;
        res->idx[3] = q.w;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const int2 p = s == 0 ? c[m] : s == 1 ? c[(m + 1) & 3] : s == 2 ? c[(m + 2) & 3] : c[(m + 3) & 3];
            res->quad[2 * m] = p.x;
            res->quad[2 * m + 1] = p.y;
        }
    }
}

// Book spreads (DESIGN.md 7b, "Book spreads"): each column's first row t(x) and last row + 1 b(x) of the page component, as
// h - t(x) and b(x) by atomicMax into zeroed memory (0: the column holds none of it); each warp takes rows w + 8 j of the
// tile, and warp 0 folds the eight and issues one pair of atomics per column.
__global__ void __launch_bounds__(kTileThreads) spine_cols_kernel(const mn_spine_page* __restrict__ spines) {
    mn_pdl_prologue();
    __shared__ int s_top[kTileThreads / 32][kTile], s_bot[kTileThreads / 32][kTile];
    const mn_spine_page sp = spines[blockIdx.y];
    const mn_quad_page* pg = sp.page;
    const mn_text_block b = pg->b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    const unsigned long long best = *pg->best;
    if (!best) return;
    const int page = (int)~(unsigned)best, lx = threadIdx.x & 31, wp = threadIdx.x >> 5, x = tx + lx;
    const int* label = pg->label;
    int top = 0, bot = 0;
    for (int y = ty + wp; x < b.w && y < min(ty + kTile, b.h); y += kTileThreads / 32) {
        if (label[(long long)y * b.w + x] == page) {
            top = max(top, b.h - y);
            bot = y + 1;
        }
    }
    s_top[wp][lx] = top;
    s_bot[wp][lx] = bot;
    __syncthreads();
    if (wp == 0) {
#pragma unroll
        for (int k = 1; k < kTileThreads / 32; ++k) {
            top = max(top, s_top[k][lx]);
            bot = max(bot, s_bot[k][lx]);
        }
        if (bot) {
            atomicMax(&sp.cols[x], top);
            atomicMax(&sp.cols[b.w + x], bot);
        }
    }
}

// (depth, x) as one int64 that orders by depth, then by the smaller x: |depth| < 2^31 (sides up to 32767), so it cannot wrap.
__device__ __forceinline__ long long spine_key(long long d, int x) {
    return d * 4294967296ll + (long long)(0xffffffffu - (unsigned)x);
}

__device__ __forceinline__ bool spine_deep(long long d, int2 a, int2 c) {
    const long long l2 = (long long)(c.x - a.x) * (c.x - a.x) + (long long)(c.y - a.y) * (c.y - a.y);
    return d > 0 && d * d >= 4 * l2 && 100 * d >= l2;
}

// One CTA per spread: the keyed max of D over the top edge's middle half and of E over the bottom edge's, then the test.
__global__ void __launch_bounds__(kHullThreads) spine_kernel(const mn_spine_page* __restrict__ spines) {
    mn_pdl_prologue();
    __shared__ long long s_key[2][kHullThreads / 32];
    const mn_spine_page sp = spines[blockIdx.x];
    const mn_quad_page* pg = sp.page;
    const int w = pg->b.w, h = pg->b.h;
    const int* q = pg->res->quad;
    const int2 tl = make_int2(q[0], q[1]), tr = make_int2(q[2], q[3]), br = make_int2(q[4], q[5]), bl = make_int2(q[6], q[7]);
    long long kt = LLONG_MIN, kb = LLONG_MIN;
    for (int x = threadIdx.x; x < w; x += blockDim.x) {
        const int top = sp.cols[x];
        if (!top) continue;
        if (4ll * (x - tl.x) >= tr.x - tl.x && 4ll * (tr.x - x) >= tr.x - tl.x)
            kt = max(kt, spine_key(cross3(tl, tr, make_int2(x, h - top)), x));
        if (4ll * (x - bl.x) >= br.x - bl.x && 4ll * (br.x - x) >= br.x - bl.x)
            kb = max(kb, spine_key(-cross3(bl, br, make_int2(x, sp.cols[w + x])), x));
    }
    for (int o = 16; o; o >>= 1) {
        kt = max(kt, (long long)__shfl_xor_sync(0xffffffffu, kt, o));
        kb = max(kb, (long long)__shfl_xor_sync(0xffffffffu, kb, o));
    }
    if ((threadIdx.x & 31) == 0) {
        s_key[0][threadIdx.x >> 5] = kt;
        s_key[1][threadIdx.x >> 5] = kb;
    }
    __syncthreads();
    if (threadIdx.x >= 32) return;
    kt = threadIdx.x < blockDim.x / 32 ? s_key[0][threadIdx.x] : LLONG_MIN;
    kb = threadIdx.x < blockDim.x / 32 ? s_key[1][threadIdx.x] : LLONG_MIN;
    for (int o = 16; o; o >>= 1) {
        kt = max(kt, (long long)__shfl_xor_sync(0xffffffffu, kt, o));
        kb = max(kb, (long long)__shfl_xor_sync(0xffffffffu, kb, o));
    }
    if (threadIdx.x) return;
    mn_page_spine* res = sp.res;
    const int xt = kt == LLONG_MIN ? -1 : (int)(0xffffffffu - (unsigned)(kt & 0xffffffffll));
    const int xb = kb == LLONG_MIN ? -1 : (int)(0xffffffffu - (unsigned)(kb & 0xffffffffll));
    const long long D = kt == LLONG_MIN ? LLONG_MIN : kt >> 32, E = kb == LLONG_MIN ? LLONG_MIN : kb >> 32;
    res->st[0] = xt;
    res->st[1] = xt < 0 ? -1 : h - sp.cols[xt];
    res->sb[0] = xb;
    res->sb[1] = xb < 0 ? -1 : sp.cols[w + xb];
    res->pad = 0;
    res->D = D;
    res->E = E;
    res->found = xt >= 0 && xb >= 0 && spine_deep(D, tl, tr) && spine_deep(E, bl, br);
}

// Seals (DESIGN.md 7b, "Seals"): cells of seal-coloured pixels, their 8-connected components by union-find on the cell grid,
// the components' boxes, then one CTA per candidate with its radial x sector histogram in shared memory, all in integers.
constexpr int kSealCellsX = 32, kSealCellsY = 8;      // a cell tile: one thread per cell, a warp per cell row
constexpr int kSealThreads = 512;
__constant__ int2 c_seal_dirs[MN_SEAL_SECTORS / 2] = MN_SEAL_DIRS;

__device__ __forceinline__ bool seal_coloured(const uint8_t* p) {
    const int a = p[0], b = p[1], c = p[2];
    return max(a, max(b, c)) - min(a, min(b, c)) >= MN_SEAL_CHROMA;
}

__device__ __forceinline__ const uint8_t* crop_px(const mn_text_block& b, int x, int y) {
    return b.img + (long long)(b.y0 + y) * b.pitch + (long long)(b.x0 + x) * 3;
}

__device__ __forceinline__ bool cell_origin(const mn_text_block& b, int& cx, int& cy, int& cw, int& ch) {
    cw = (b.w + MN_SEAL_CELL - 1) / MN_SEAL_CELL;
    ch = (b.h + MN_SEAL_CELL - 1) / MN_SEAL_CELL;
    const int tiles_x = (cw + kSealCellsX - 1) / kSealCellsX, tiles_y = (ch + kSealCellsY - 1) / kSealCellsY;
    if ((long long)blockIdx.x >= (long long)tiles_x * tiles_y) return false;
    cx = (int)(blockIdx.x % tiles_x) * kSealCellsX + (threadIdx.x & 31);
    cy = (int)(blockIdx.x / tiles_x) * kSealCellsY + (threadIdx.x >> 5);
    return cx < cw && cy < ch;
}

// 1: each cell's count of seal-coloured pixels and their box.
__global__ void __launch_bounds__(kTileThreads) seal_cells_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_seal_page sp = pages[blockIdx.y];
    const mn_text_block b = sp.b;
    int cx, cy, cw, ch;
    if (!cell_origin(b, cx, cy, cw, ch)) return;
    int n = 0, x0 = INT_MAX, y0 = INT_MAX, x1 = 0, y1 = 0;
    for (int y = cy * MN_SEAL_CELL; y < min(cy * MN_SEAL_CELL + MN_SEAL_CELL, b.h); ++y) {
        for (int x = cx * MN_SEAL_CELL; x < min(cx * MN_SEAL_CELL + MN_SEAL_CELL, b.w); ++x) {
            if (!seal_coloured(crop_px(b, x, y))) continue;
            ++n;
            x0 = min(x0, x);
            y0 = min(y0, y);
            x1 = max(x1, x + 1);
            y1 = y + 1;
        }
    }
    const int c = cy * cw + cx;
    const bool on = n >= MN_SEAL_CELL_MIN;
    sp.label[c] = on ? c : -1;
    if (on) reinterpret_cast<int4*>(sp.box)[c] = make_int4(x0, y0, x1, y1);
}

// 2: each on cell joined to its on neighbours W, NW, N and NE.
__global__ void __launch_bounds__(kTileThreads) seal_union_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_seal_page sp = pages[blockIdx.y];
    int cx, cy, cw, ch;
    if (!cell_origin(sp.b, cx, cy, cw, ch)) return;
    int* label = sp.label;
    const int c = cy * cw + cx;
    if (label[c] < 0) return;
    if (cx > 0 && label[c - 1] >= 0) uf_union(label, c - 1, c);
    if (cy > 0) {
        for (int d = -1; d <= 1; ++d) {
            if (cx + d >= 0 && cx + d < cw && label[c - cw + d] >= 0) uf_union(label, c - cw + d, c);
        }
    }
}

// 3: path compression and each on cell's box folded into its root's.
__global__ void __launch_bounds__(kTileThreads) seal_box_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_seal_page sp = pages[blockIdx.y];
    int cx, cy, cw, ch;
    if (!cell_origin(sp.b, cx, cy, cw, ch)) return;
    const int c = cy * cw + cx;
    if (sp.label[c] < 0) return;
    const int r = uf_find(sp.label, c);
    sp.label[c] = r;
    if (r == c) return;
    const int4 bx = reinterpret_cast<const int4*>(sp.box)[c];
    atomicMin(&sp.box[4 * r], bx.x);
    atomicMin(&sp.box[4 * r + 1], bx.y);
    atomicMax(&sp.box[4 * r + 2], bx.z);
    atomicMax(&sp.box[4 * r + 3], bx.w);
}

// 4: each root whose box passes the size test appended as a candidate.
__global__ void __launch_bounds__(kTileThreads) seal_cand_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    const mn_seal_page sp = pages[blockIdx.y];
    int cx, cy, cw, ch;
    if (!cell_origin(sp.b, cx, cy, cw, ch)) return;
    const int c = cy * cw + cx;
    if (sp.label[c] != c) return;
    const int4 bx = reinterpret_cast<const int4*>(sp.box)[c];
    const int A = bx.z - bx.x, B = bx.w - bx.y, lo = min(A, B), hi = max(A, B);
    if (lo < sp.seal_size || hi > MN_SEAL_MAX_SIDE || 2 * hi > 3 * lo) return;
    const int slot = atomicAdd(&sp.out->n_cand, 1);
    if (slot >= MN_PAGE_MAX_SEALS) return;
    int* e = sp.cand + 8 * slot;
    e[0] = bx.x;
    e[1] = bx.y;
    e[2] = bx.z;
    e[3] = bx.w;
    e[4] = c;
}

// The radial bin k = floor(32 rho) of (X, Y) in an A x B box, exact: q = floor(1024 (X^2 B^2 + Y^2 A^2) / (A^2 B^2)) <= 2048,
// and floor(sqrt(q)) = floor(32 rho).
__device__ __forceinline__ int seal_bin(long long X, long long Y, long long A, long long B) {
    const long long q = 1024 * (X * X * B * B + Y * Y * A * A) / (A * A * B * B);
    int k = (int)sqrtf((float)q);
    while ((long long)k * k > q) --k;
    while ((long long)(k + 1) * (k + 1) <= q) ++k;
    return k;
}

__device__ __forceinline__ int seal_half_sector(long long px, long long py) {
    int lo = 0, hi = MN_SEAL_SECTORS / 2 - 1;                   // the largest s < 36 with cross(d_s, p) >= 0; s = 0 holds
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        const int2 d = c_seal_dirs[mid];
        if ((long long)d.x * py - (long long)d.y * px >= 0) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ int seal_sector(long long px, long long py) {
    if (px == 0 && py == 0) return 0;
    if (py > 0 || (py == 0 && px > 0)) return seal_half_sector(px, py);
    return MN_SEAL_SECTORS / 2 + seal_half_sector(-px, -py);
}

// The band walk's first bin inside the ring's edge: from k = 32 inward past the ring's outer bins, the ring run and its edge.
__device__ __forceinline__ int seal_gap_top(const int* ink, const int* area) {
    int k = MN_SEAL_BINS - 1;
    while (k >= 0 && MN_SEAL_RING_DENSITY * ink[k] < area[k]) --k;                         // the ring's outer bin
    while (k >= 0 && MN_SEAL_RING_DENSITY * ink[k] >= area[k]) --k;                        // the ring run
    while (k >= 0 && MN_SEAL_BAND_DENSITY * ink[k] >= area[k]) --k;                        // its edge
    return k;
}

// The gap (g0, n) of per-sector ink sec, band its sum: the longest circular run of empty sectors; returns the arc's why.
__device__ __forceinline__ int seal_arc_gap(const int* sec, int band, int& g0, int& n) {
    const int lim = max(MN_SEAL_EMPTY_DIV, band);
    int all = 1;
    g0 = 0, n = 0;
    for (int s = 0; s < MN_SEAL_SECTORS; ++s) all &= MN_SEAL_EMPTY_DIV * sec[s] < lim;
    if (all) {
        n = MN_SEAL_SECTORS;
    } else {
        for (int s = 0; s < MN_SEAL_SECTORS; ++s) {           // runs start at an empty sector after a non-empty one
            const int prev = (s + MN_SEAL_SECTORS - 1) % MN_SEAL_SECTORS;
            if (!(MN_SEAL_EMPTY_DIV * sec[s] < lim) || MN_SEAL_EMPTY_DIV * sec[prev] < lim) continue;
            int m = 0;
            while (MN_SEAL_EMPTY_DIV * sec[(s + m) % MN_SEAL_SECTORS] < lim) ++m;
            if (m > n) g0 = s, n = m;
        }
    }
    return n < MN_SEAL_MIN_GAP ? MN_SEAL_NO_GAP : MN_SEAL_SECTORS - n < MN_SEAL_MIN_TEXT ? MN_SEAL_SHORT : 0;
}

// 5: one CTA per candidate slot: the histograms, then thread 0 reads the ring, band and arc off them.
__global__ void __launch_bounds__(kSealThreads) seal_test_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    __shared__ int s_ink[MN_SEAL_BINS][MN_SEAL_SECTORS];
    __shared__ int s_area[MN_SEAL_BINS];
    __shared__ int s_sum[MN_SEAL_BINS + MN_SEAL_SECTORS];     // ink_k, then the ring's sectors hit
    __shared__ int s_sec[MN_SEAL_SECTORS];
    __shared__ int s_rank;
    const mn_seal_page sp = pages[blockIdx.y];
    mn_seal_table* out = sp.out;
    const int n_cand = out->n_cand, slot = blockIdx.x;
    if (n_cand > MN_PAGE_MAX_SEALS) {
        if (slot == 0 && threadIdx.x == 0) out->error = MN_SEAL_ERR_SEALS;
        return;
    }
    if (slot >= n_cand) return;
    const int* e = sp.cand + 8 * slot;
    const int x0 = e[0], y0 = e[1], x1 = e[2], y1 = e[3], root = e[4];
    for (int i = threadIdx.x; i < MN_SEAL_BINS * MN_SEAL_SECTORS; i += blockDim.x) (&s_ink[0][0])[i] = 0;
    if (threadIdx.x < MN_SEAL_BINS) s_area[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_rank = 0;
    __syncthreads();
    const mn_text_block b = sp.b;
    const long long A = x1 - x0, B = y1 - y0;
    const long long n_px = A * B;
    for (long long i = threadIdx.x; i < n_px; i += blockDim.x) {
        const int x = x0 + (int)(i % A), y = y0 + (int)(i / A);
        const long long X = 2 * x + 1 - (x0 + x1), Y = 2 * y + 1 - (y0 + y1);
        const int k = seal_bin(X, Y, A, B);
        if (k >= MN_SEAL_BINS) continue;
        atomicAdd(&s_area[k], 1);
        if (seal_coloured(crop_px(b, x, y))) atomicAdd(&s_ink[k][seal_sector(X * B, -Y * A)], 1);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < MN_SEAL_BINS + MN_SEAL_SECTORS; j += blockDim.x) {
        int t = 0;
        if (j < MN_SEAL_BINS) {                                  // ink_k
            for (int s = 0; s < MN_SEAL_SECTORS; ++s) t += s_ink[j][s];
        } else {                                                 // a sector hit by the ring
            for (int k = MN_SEAL_RING_K; k < MN_SEAL_BINS; ++k) t |= s_ink[k][j - MN_SEAL_BINS];
            t = t != 0;
        }
        s_sum[j] = t;
    }
    int rank = 0;                                                // by (y0, x0, root) among the page's candidates
    for (int j = threadIdx.x; j < n_cand; j += blockDim.x) {
        const int* f = sp.cand + 8 * j;
        rank += f[1] < y0 || (f[1] == y0 && (f[0] < x0 || (f[0] == x0 && f[4] < root)));
    }
    if (rank) atomicAdd(&s_rank, rank);
    __syncthreads();
    if (threadIdx.x) return;
    const int* ink = s_sum;
    int ring = 0;
    for (int s = 0; s < MN_SEAL_SECTORS; ++s) ring += s_sum[MN_SEAL_BINS + s];
    mn_seal r;
    r.x0 = x0, r.y0 = y0, r.x1 = x1, r.y1 = y1, r.root = root, r.ring = ring;
    r.found = ring >= MN_SEAL_RING_SECTORS;
    r.k_bottom = r.k_top = r.g0 = r.n_gap = -1;
    r.why = 0, r.band_ink = 0, r.pad[0] = r.pad[1] = r.pad[2] = 0;
    if (r.found) {
        const int gap_top = seal_gap_top(ink, s_area);
        int k = gap_top;
        while (k >= MN_SEAL_BAND_MIN_K && MN_SEAL_BAND_DENSITY * ink[k] < s_area[k]) --k;      // the gap
        if (gap_top >= MN_SEAL_BAND_MIN_K && k < gap_top && k >= MN_SEAL_BAND_MIN_K) {
            r.k_top = k;
            while (k >= MN_SEAL_BAND_MIN_K && MN_SEAL_BAND_DENSITY * ink[k] >= s_area[k]) --k;
            r.k_bottom = k + 1;
        }
        if (r.k_top < 0) {
            r.why = MN_SEAL_NO_BAND;
        } else {
            int* sec = s_sec;
            int band = 0;
            for (int s = 0; s < MN_SEAL_SECTORS; ++s) {
                int t = 0;
                for (int kk = r.k_bottom; kk <= r.k_top; ++kk) t += s_ink[kk][s];
                sec[s] = t;
                band += t;
            }
            r.band_ink = band;
            r.why = seal_arc_gap(sec, band, r.g0, r.n_gap);
        }
    }
    out->seal[s_rank] = r;
    if (r.found) atomicAdd(&out->n_seals, 1);
}

// 6: the layout copy, the seals' own ink set to paper.
__global__ void __launch_bounds__(kTileThreads) seal_copy_kernel(const mn_seal_page* __restrict__ pages) {
    mn_pdl_prologue();
    __shared__ int4 s_box[MN_PAGE_MAX_SEALS];
    __shared__ int s_n;
    const mn_seal_page sp = pages[blockIdx.y];
    const mn_text_block b = sp.b;
    int tx, ty;
    if (!tile_origin(b, tx, ty)) return;
    if (threadIdx.x == 0) {
        const mn_seal_table* t = sp.out;
        int n = 0;
        if (!t->error) {
            for (int j = 0; j < min(t->n_cand, MN_PAGE_MAX_SEALS); ++j) {
                const mn_seal& s = t->seal[j];
                if (s.found && s.x0 < tx + kTile && tx < s.x1 && s.y0 < ty + kTile && ty < s.y1)
                    s_box[n++] = make_int4(s.x0, s.y0, s.x1, s.y1);
            }
        }
        s_n = n;
    }
    __syncthreads();
    const int x = tx + (threadIdx.x & 31), n = s_n;
    if (x >= b.w) return;
    for (int y = ty + (threadIdx.x >> 5); y < min(ty + kTile, b.h); y += 8) {
        const uint8_t* p = crop_px(b, x, y);
        uint8_t v0 = p[0], v1 = p[1], v2 = p[2];
        if (n && seal_coloured(p)) {
            for (int j = 0; j < n; ++j) {
                const int4 s = s_box[j];
                if (x < s.x || x >= s.z || y < s.y || y >= s.w) continue;
                const long long A = s.z - s.x, B = s.w - s.y, X = 2 * x + 1 - (s.x + s.z), Y = 2 * y + 1 - (s.y + s.w);
                if (1024 * (X * X * B * B + Y * Y * A * A) < (long long)MN_SEAL_BINS * MN_SEAL_BINS * A * A * B * B) {
                    v0 = v1 = v2 = 255;
                    break;
                }
            }
        }
        uint8_t* q = sp.copy + (long long)y * 3 * b.w + (long long)x * 3;
        q[0] = v0;
        q[1] = v1;
        q[2] = v2;
    }
}

// Seal centre lines (DESIGN.md 7b, "Seal centre lines"): one CTA per seal slot rebuilds the seal's histograms, reads its head
// gap, turn and arc band off them (thread 0), then the min and max u of each interior row in the stamp frame.
constexpr int kCentreRows = MN_SEAL_MAX_SIDE + 4;     // v in [-M / 2 - 1, M / 2] for M = max(A, B): row v at v + M / 2 + 2
__constant__ int2 c_seal_turns[MN_SEAL_TURN_STEPS / 4] = MN_SEAL_TURNS;

__global__ void __launch_bounds__(kSealThreads) centre_lines_kernel(const mn_centre_page* __restrict__ pages) {
    mn_pdl_prologue();
    __shared__ int s_ink[MN_SEAL_BINS][MN_SEAL_SECTORS];
    __shared__ int s_area[MN_SEAL_BINS];
    __shared__ int s_sum[MN_SEAL_BINS];
    __shared__ int s_sec[MN_SEAL_SECTORS];
    __shared__ int s_lo[kCentreRows], s_hi[kCentreRows];
    __shared__ int s_k_in, s_k_gap, s_g0, s_n, s_c, s_s, s_vlo, s_vhi;
    __shared__ mn_seal_lines s_rec;
    const mn_centre_page cp = pages[blockIdx.y];
    const mn_seal_table* t = cp.seals;
    const int slot = blockIdx.x;
    if (t->error || slot >= min(t->n_cand, MN_PAGE_MAX_SEALS) || !t->seal[slot].found) {     // a zero record
        int* z = reinterpret_cast<int*>(&cp.lines->seal[slot]);
        for (int i = threadIdx.x; i < (int)(sizeof(mn_seal_lines) / 4); i += blockDim.x) z[i] = 0;
        return;
    }
    const mn_seal sl = t->seal[slot];
    const int x0 = sl.x0, y0 = sl.y0, x1 = sl.x1, y1 = sl.y1;
    const long long A = x1 - x0, B = y1 - y0, n_px = A * B;
    const int off = (int)(max(A, B) / 2) + 2;
    for (int i = threadIdx.x; i < MN_SEAL_BINS * MN_SEAL_SECTORS; i += blockDim.x) (&s_ink[0][0])[i] = 0;
    for (int i = threadIdx.x; i < kCentreRows; i += blockDim.x) s_lo[i] = INT_MAX, s_hi[i] = INT_MIN;
    if (threadIdx.x < MN_SEAL_BINS) s_area[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_vlo = INT_MAX, s_vhi = INT_MIN;
    __syncthreads();
    const mn_text_block b = cp.b;
    for (long long i = threadIdx.x; i < n_px; i += blockDim.x) {
        const int x = x0 + (int)(i % A), y = y0 + (int)(i / A);
        const long long X = 2 * x + 1 - (x0 + x1), Y = 2 * y + 1 - (y0 + y1);
        const int k = seal_bin(X, Y, A, B);
        if (k >= MN_SEAL_BINS) continue;
        atomicAdd(&s_area[k], 1);
        if (seal_coloured(crop_px(b, x, y))) atomicAdd(&s_ink[k][seal_sector(X * B, -Y * A)], 1);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < MN_SEAL_BINS; k += blockDim.x) {
        int v = 0;
        for (int s = 0; s < MN_SEAL_SECTORS; ++s) v += s_ink[k][s];
        s_sum[k] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        mn_seal_lines& r = s_rec;
        r.turn = 0, r.g0 = r.n_gap = r.k_bottom = r.k_top = -1, r.why = MN_SEAL_NO_BAND;
        r.k_in = r.k_gap = max(seal_gap_top(s_sum, s_area), 0);
        r.n_found = r.n_lines = 0, r.pad[0] = r.pad[1] = 0;
        for (int j = 0; j < MN_SEAL_MAX_LINES; ++j) r.box[j][0] = r.box[j][1] = r.box[j][2] = r.box[j][3] = 0;
        if (sl.k_top >= MN_SEAL_HEAD_MIN_K) {
            const int kt = sl.k_top;
            int head = 0;
            for (int s = 0; s < MN_SEAL_SECTORS; ++s) {
                int v = 0;
                for (int k = kt - MN_SEAL_HEAD_BINS + 1; k <= kt; ++k) v += s_ink[k][s];
                s_sec[s] = v;
                head += v;
            }
            int g0, n;
            r.why = seal_arc_gap(s_sec, head, g0, n);
            int turn = (2 * g0 + n - 108 + MN_SEAL_TURN_STEPS) % MN_SEAL_TURN_STEPS;
            if (turn > MN_SEAL_TURN_STEPS / 2) turn -= MN_SEAL_TURN_STEPS;
            int k = kt;                                          // the walk over the arc sectors [g0 + n, g0 + 72)
            for (; k - 1 >= MN_SEAL_BAND_MIN_K; --k) {
                long long arc = 0;
                for (int m = n; m < MN_SEAL_SECTORS; ++m) arc += s_ink[k - 1][(g0 + m) % MN_SEAL_SECTORS];
                if ((long long)MN_SEAL_BAND_DENSITY * MN_SEAL_SECTORS * arc < (long long)s_area[k - 1] * (MN_SEAL_SECTORS - n)) break;
            }
            r.turn = r.why ? 0 : turn, r.g0 = g0, r.n_gap = n, r.k_bottom = k, r.k_top = kt, r.k_in = k;
            r.k_gap = max(k, kt - MN_SEAL_HEAD_BINS + 1);
        }
        const int j = (r.turn % MN_SEAL_TURN_STEPS + MN_SEAL_TURN_STEPS) % MN_SEAL_TURN_STEPS;
        int c = c_seal_turns[j % (MN_SEAL_TURN_STEPS / 4)].x, s = c_seal_turns[j % (MN_SEAL_TURN_STEPS / 4)].y;
        for (int q = 0; q < j / (MN_SEAL_TURN_STEPS / 4); ++q) {
            const int c0 = c;
            c = -s, s = c0;
        }
        s_k_in = r.k_in, s_k_gap = r.k_gap, s_g0 = r.g0, s_n = r.n_gap, s_c = c, s_s = s;
    }
    __syncthreads();
    const int k_in = s_k_in, k_gap = s_k_gap, g0 = s_g0 + MN_SEAL_GAP_MARGIN, n_in = s_n - 2 * MN_SEAL_GAP_MARGIN;
    const long long c = s_c, s = s_s;
    for (long long i = threadIdx.x; i < n_px; i += blockDim.x) {
        const int x = x0 + (int)(i % A), y = y0 + (int)(i / A);
        const long long X = 2 * x + 1 - (x0 + x1), Y = 2 * y + 1 - (y0 + y1);
        const int k = seal_bin(X, Y, A, B);                     // the interior: k < k_in, or k < k_gap inside the head gap
        if (k >= k_gap || !seal_coloured(crop_px(b, x, y))) continue;
        if (k >= k_in && (seal_sector(X * B, -Y * A) - g0 + 2 * MN_SEAL_SECTORS) % MN_SEAL_SECTORS >= n_in) continue;
        const int u = (int)((X * c - Y * s) >> 21), v = (int)((X * s + Y * c) >> 21);
        atomicMin(&s_lo[v + off], u);
        atomicMax(&s_hi[v + off], u);
        atomicMin(&s_vlo, v);
        atomicMax(&s_vhi, v);
    }
    __syncthreads();
    if (threadIdx.x) return;
    mn_seal_lines& r = s_rec;
    const int min_h = max(MN_SEAL_LINE_MIN_H, (int)((A + B) / MN_SEAL_LINE_H_DIV)), R = (int)(k_gap * max(A, B) / 64);
    int u0 = 0, u1 = 0, v0 = 0, last = INT_MIN / 2;
    auto close = [&]() {                                         // the run [v0, last] ends
        const int h = last - v0 + 1;
        if (h < min_h || u1 - u0 + 1 < MN_SEAL_LINE_RATIO * h) return;
        if (r.n_found < MN_SEAL_MAX_LINES) {
            const int p = max(MN_SEAL_LINE_PAD, h / MN_SEAL_LINE_PAD_DIV);
            int* o = r.box[r.n_found];
            o[0] = max(u0 - p, -R - 1), o[1] = max(v0 - p, -R - 1), o[2] = min(u1 + 1 + p, R + 1), o[3] = min(last + 1 + p, R + 1);
        }
        ++r.n_found;
    };
    for (int v = s_vlo; v <= s_vhi; ++v) {
        const int lo = s_lo[v + off], hi = s_hi[v + off];
        if (lo > hi) continue;
        if (v > s_vlo && v - last - 1 < MN_SEAL_LINE_GAP) {
            u0 = min(u0, lo), u1 = max(u1, hi), last = v;
            continue;
        }
        if (v > s_vlo) close();
        u0 = lo, u1 = hi, v0 = last = v;
    }
    if (s_vlo <= s_vhi) close();
    r.n_lines = min(r.n_found, MN_SEAL_MAX_LINES);
    cp.lines->seal[slot] = r;
}

// 4-11 of the XY-cut: both passes of levels, the text size between them and the leaves, on pages whose bitmap and root are
// written; under MN_PAGE_RULES, the three rule launches first, under MN_PAGE_PANELS the panel test and paint after the text
// size, under MN_PAGE_FIGURES the figure launch after those, and under MN_PAGE_DIRECTIONS the direction launch after the leaves.
int page_levels(mn_text_page* pages, int n, long long max_tiles, int flags, cudaStream_t st) {
    const dim3 rgrid((unsigned)mn_cdiv64(max_tiles, kRuleThreads / 32), (unsigned)n);
    if (flags & MN_PAGE_RULES) {
        MN_CUDA_CHECK((mn_launch(rule_transpose_kernel, rgrid, dim3(kRuleThreads), 0, st, pages)));
        MN_LAUNCH_CHECK();
        MN_CUDA_CHECK((mn_launch(rule_runs_kernel, rgrid, dim3(kRuleThreads), 0, st, pages)));
        MN_LAUNCH_CHECK();
        MN_CUDA_CHECK((mn_launch(rule_merge_kernel, rgrid, dim3(kRuleThreads), 0, st, pages)));
        MN_LAUNCH_CHECK();
    }
    const dim3 grid((unsigned)max(1, 4 * mn_num_sms() / n), (unsigned)n);   // about four CTAs per SM over all pages
    for (int pass = 0; pass < 2; ++pass) {
        for (int level = 0; level < MN_PAGE_LEVELS; ++level) {
            MN_CUDA_CHECK((mn_launch(page_count_kernel, grid, dim3(kPageThreads), 0, st, pages, level)));
            MN_LAUNCH_CHECK();
            MN_CUDA_CHECK((mn_launch(page_scan_kernel, dim3(n), dim3(kScanThreads), 0, st, pages)));
            MN_LAUNCH_CHECK();
            MN_CUDA_CHECK((mn_launch(page_emit_kernel, grid, dim3(kPageThreads), 0, st, pages, level)));
            MN_LAUNCH_CHECK();
        }
        if (pass == 0) {
            MN_CUDA_CHECK((mn_launch(page_size_kernel, dim3(n), dim3(kScanThreads), 0, st, pages)));
            MN_LAUNCH_CHECK();
            if (flags & MN_PAGE_PANELS) {
                MN_CUDA_CHECK((mn_launch(panel_test_kernel, grid, dim3(kPanelThreads), 0, st, pages)));
                MN_LAUNCH_CHECK();
                MN_CUDA_CHECK((mn_launch(panel_paint_kernel, rgrid, dim3(kFigureThreads), 0, st, pages)));
                MN_LAUNCH_CHECK();
            }
            if (flags & MN_PAGE_FIGURES) {
                MN_CUDA_CHECK((mn_launch(figure_paint_kernel, rgrid, dim3(kFigureThreads), 0, st, pages)));
                MN_LAUNCH_CHECK();
            }
        }
    }
    MN_CUDA_CHECK((mn_launch(page_blocks_kernel, dim3(n), dim3(kScanThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    if (flags & MN_PAGE_DIRECTIONS) {
        MN_CUDA_CHECK((mn_launch(page_direction_kernel, grid, dim3(kPageThreads), 0, st, pages)));
        MN_LAUNCH_CHECK();
    }
    if (flags & MN_PAGE_TURNS) {
        MN_CUDA_CHECK((mn_launch(page_turn_kernel, grid, dim3(kPageThreads), 0, st, pages)));
        MN_LAUNCH_CHECK();
    }
    return MN_OK;
}

// 1-2 of every text-block entry: the zeroed work, then each crop's histogram and Otsu threshold.
int block_threshold(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes, cudaStream_t st) {
    MN_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)work_bytes, st));
    MN_CUDA_CHECK((mn_launch(block_hist_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_threshold_kernel, dim3(mn_cdiv(n, 128)), dim3(128), 0, st, blocks, n)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

}  // namespace

// The histogram and threshold launches for the other files of the library (light_ops.cu).
int mn_block_threshold(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes, cudaStream_t st) {
    return block_threshold(blocks, n, max_tiles, work, work_bytes, st);
}

extern "C" int mn_find_lines_u8(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes,
                                void* stream) {
    MN_REQUIRE(blocks && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_lines_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    MN_CUDA_CHECK((mn_launch(block_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_lines_skewed_u8(mn_text_block* blocks, mn_skew_block* skew, int n, long long max_tiles, void* work,
                                       long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && skew && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_lines_skewed_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    MN_CUDA_CHECK((mn_launch(skew_angle_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_score_kernel, dim3(n), dim3(kScoreThreads), 0, st, blocks, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_blocks_u8(const mn_text_block* blocks, mn_text_page* pages, int n, long long max_tiles, int flags, void* work,
                                 long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && pages && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_blocks_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    MN_CUDA_CHECK((mn_launch(page_bits_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    return page_levels(pages, n, max_tiles, flags, st);
}

extern "C" int mn_find_blocks_skewed_u8(mn_text_block* blocks, mn_skew_block* skew, mn_text_page* pages, int n, long long max_tiles,
                                        int flags, void* work, long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && skew && pages && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_blocks_skewed_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    MN_CUDA_CHECK((mn_launch(skew_angle_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_score_kernel, dim3(n), dim3(kScoreThreads), 0, st, blocks, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(page_frame_bits_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, pages, skew)));
    MN_LAUNCH_CHECK();
    return page_levels(pages, n, max_tiles, flags, st);
}

extern "C" int mn_find_lines_window_u8(const mn_text_block* blocks, const mn_window_block* wins, int n, long long max_tiles,
                                       void* work, long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && wins && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_lines_window_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    MN_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)work_bytes, st));
    MN_CUDA_CHECK((mn_launch(window_hist_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, wins)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_threshold_kernel, dim3(mn_cdiv(n, 128)), dim3(128), 0, st, blocks, n)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(window_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, wins)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_page_quads_u8(const mn_text_block* blocks, const mn_quad_page* pages, int n, long long max_tiles, void* work,
                                     long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && pages && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_page_quads_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    const dim3 grid((unsigned)max_tiles, n);
    MN_CUDA_CHECK((mn_launch(quad_label_local_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(quad_label_border_kernel, grid, dim3(64), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(quad_label_count_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(quad_pick_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(quad_rows_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(quad_hull_kernel, dim3(n), dim3(kHullThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_page_spines_u8(const mn_spine_page* spines, int n, long long max_tiles, void* stream) {
    MN_REQUIRE(spines && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31), "mn_find_page_spines_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    MN_CUDA_CHECK((mn_launch(spine_cols_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, spines)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(spine_kernel, dim3(n), dim3(kHullThreads), 0, st, spines)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_seal_layout_u8(const mn_seal_page* pages, int n, long long max_tiles, void* stream) {
    MN_REQUIRE(pages && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31), "mn_seal_layout_u8: bad args");
    MN_CUDA_CHECK((mn_launch(seal_copy_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, (cudaStream_t)stream, pages)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_seal_lines_u8(const mn_centre_page* pages, int n, void* stream) {
    MN_REQUIRE(pages && n > 0 && n <= 65535, "mn_find_seal_lines_u8: bad args");
    MN_CUDA_CHECK((mn_launch(centre_lines_kernel, dim3(MN_PAGE_MAX_SEALS, n), dim3(kSealThreads), 0, (cudaStream_t)stream, pages)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_find_seals_u8(const mn_seal_page* pages, int n, long long max_tiles, long long max_cell_tiles, void* work,
                                long long work_bytes, void* stream) {
    MN_REQUIRE(pages && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && max_cell_tiles > 0 &&
               max_cell_tiles < (1ll << 31) && work && work_bytes > 0, "mn_find_seals_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    MN_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)work_bytes, st));
    const dim3 grid((unsigned)max_cell_tiles, n);
    MN_CUDA_CHECK((mn_launch(seal_cells_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(seal_union_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(seal_box_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(seal_cand_kernel, grid, dim3(kTileThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(seal_test_kernel, dim3(MN_PAGE_MAX_SEALS, n), dim3(kSealThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    return mn_seal_layout_u8(pages, n, max_tiles, stream);
}

extern "C" int mn_find_lines_curved_u8(const mn_text_block* blocks, const mn_curve_block* curves, int n, long long max_tiles,
                                       int max_strips, void* work, long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && curves && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && max_strips >= 1 &&
               max_strips <= MN_CURVE_MAX_STRIPS && work && work_bytes > 0, "mn_find_lines_curved_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = block_threshold(blocks, n, max_tiles, work, work_bytes, st);
    if (rc != MN_OK) return rc;
    MN_CUDA_CHECK((mn_launch(block_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(curve_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, curves)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(curve_runs_kernel, dim3((unsigned)max_strips, n), dim3(kSegThreads), 0, st, curves)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(curve_link_kernel, dim3(n), dim3(kLinkThreads), 0, st, curves)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
