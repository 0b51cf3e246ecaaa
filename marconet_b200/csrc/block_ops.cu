// Text blocks split into lines (DESIGN.md 7b, "Text blocks"): Otsu binarisation, a projection profile and line runs for every
// block of a call in four launches (histogram, threshold, profile, segmentation).  The threshold is OpenCV's fp64 loop with
// explicit-rounding intrinsics, so that nvcc cannot contract it into an FMA the host twin (oracle/blocks.py) does not have; the
// rest is integer arithmetic.  Skewed blocks (DESIGN.md 7b, "Skewed blocks") add an angle search and a rotated profile around
// the same kernels, in six launches.
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

extern "C" int mn_find_lines_skewed_u8(mn_text_block* blocks, mn_skew_block* skew, int n, long long max_tiles, void* work,
                                       long long work_bytes, void* stream) {
    MN_REQUIRE(blocks && skew && n > 0 && n <= 65535 && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0,
               "mn_find_lines_skewed_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    const mn_text_block* cblocks = blocks;
    const mn_skew_block* cskew = skew;
    MN_CUDA_CHECK(cudaMemsetAsync(work, 0, (size_t)work_bytes, st));
    MN_CUDA_CHECK((mn_launch(block_hist_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, cblocks)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_threshold_kernel, dim3(mn_cdiv(n, 128)), dim3(128), 0, st, cblocks, n)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_angle_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, cskew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_score_kernel, dim3(n), dim3(kScoreThreads), 0, st, blocks, skew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(skew_profile_kernel, dim3((unsigned)max_tiles, n), dim3(kTileThreads), 0, st, cskew)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(block_lines_kernel, dim3(n), dim3(kSegThreads), 0, st, cblocks)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
