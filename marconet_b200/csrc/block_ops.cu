// Text blocks split into lines (DESIGN.md 7b, "Text blocks"): Otsu binarisation, a projection profile and line runs for every
// block of a call in four launches (histogram, threshold, profile, segmentation).  The threshold is OpenCV's fp64 loop with
// explicit-rounding intrinsics, so that nvcc cannot contract it into an FMA the host twin (oracle/blocks.py) does not have; the
// rest is integer arithmetic.
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
    const double scale = __ddiv_rn(1.0, (double)(b.w * b.h));
    double mu = 0.0;
    for (int k = 0; k < 256; ++k) mu = __dadd_rn(mu, __dmul_rn((double)k, (double)h[k]));
    mu = __dmul_rn(mu, scale);
    const double eps = 1.1920928955078125e-07;    // FLT_EPSILON
    double mu1 = 0.0, q1 = 0.0, max_sigma = 0.0;
    int t = 0;
    for (int k = 0; k < 256; ++k) {
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
    if (ink == MN_INK_AUTO) ink = 2 * dark <= (long long)b.w * b.h ? MN_INK_DARK : MN_INK_LIGHT;
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
__device__ int cta_scan(int v, int* s, int* total) {
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

}  // namespace

extern "C" int mn_find_lines_u8(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes,
                                void* stream) {
    MN_REQUIRE(blocks && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_lines_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    MN_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)work_bytes, st));
    MN_CUDA_CHECK((mn_launch(block_hist_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_threshold_kernel, dim3(mn_cdiv(n, 128)), dim3(128), 0, st, blocks, n)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, blocks)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
