// Even lighting (DESIGN.md 7b, "Even lighting"): a page divided by its paper, the grey closing of the page with a k x k window,
// every page of a call in six launches (the histogram and threshold of block_ops.cu, then four separable 1-D passes).  Each pass
// runs the van Herk / Gil-Werman scheme: the window [i - k / 2, i + k / 2] of output i is, on the line padded by k / 2
// identities at each end, the padded positions [i, i + k - 1], which span the suffix of one segment of k positions and the
// prefix of the next.  One thread per (line, segment) walks its segment's suffix backwards and the next one's prefix forwards,
// so a pass costs O(1) comparisons per pixel whatever k, and the padding is the running value's start, never read.  The three
// channels travel packed in one 32-bit word (__vmaxu4 / __vminu4); the divide is IEEE fp32, exact against OpenCV's fp64.
#include "mn_common.cuh"

int mn_block_threshold(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes, cudaStream_t st);

namespace {

constexpr int kLightThreads = 256;

__device__ __forceinline__ uint32_t load3(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
}

__device__ __forceinline__ void store3(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)v;
    p[1] = (uint8_t)(v >> 8);
    p[2] = (uint8_t)(v >> 16);
}

// cv2.divide(f, b, scale=255) for one channel: rint(255 f / b), half to even, 0 where b = 0, saturated.
__device__ __forceinline__ uint32_t light_div(uint32_t f, uint32_t b) {
    if (b == 0) return 0;
    return (uint32_t)fminf(rintf(__fdiv_rn(255.f * (float)f, (float)b)), 255.f);
}

// Stage 0: row max, src -> s1; 1: column max, s1 -> s2; 2: row min, s2 -> s1; 3: column min of s1 with the divide, -> dst.
// The suffix extrema go to `tmp` (the output plane, or s2 in stage 3 so that dst may be src), read back by the same thread.
template <int kStage>
__global__ void __launch_bounds__(kLightThreads) light_pass_kernel(const mn_light_page* __restrict__ pages) {
    mn_pdl_prologue();
    constexpr bool kMin = kStage >= 2, kCols = (kStage & 1) != 0;
    const mn_light_page& pg = pages[blockIdx.y];
    const int h = pg.h, w = pg.w, k = pg.k, r = k >> 1;
    const int n = kCols ? h : w, lines = kCols ? w : h;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)lines * ((n + k - 1) / k)) return;
    const int line = (int)(t % lines), lo = (int)(t / lines) * k;
    const uint32_t mask = pg.b.out->ink == MN_INK_LIGHT ? 0xFFFFFFu : 0u;
    const uint32_t ident = kMin ? 0xFFFFFFu : 0u;
    const int64_t plane = 3ll * w;
    const uint8_t* in = kStage == 0 ? pg.src : kStage == 2 ? pg.s2 : pg.s1;
    const int64_t in_pitch = kStage == 0 ? pg.src_pitch : plane;
    uint8_t* out = kStage == 1 ? pg.s2 : kStage == 3 ? pg.dst : pg.s1;
    const int64_t out_pitch = kStage == 3 ? pg.dst_pitch : plane;
    uint8_t* tmp = kStage == 0 || kStage == 2 ? pg.s1 : pg.s2;
    const uint32_t in_mask = kStage == 0 ? mask : 0u;
    // byte offset of index j along the line in a plane of the given pitch
    auto at = [&](int64_t pitch, int j) -> int64_t {
        return kCols ? (int64_t)j * pitch + 3ll * line : (int64_t)line * pitch + 3ll * j;
    };
    auto op = [](uint32_t a, uint32_t b) { return kMin ? __vminu4(a, b) : __vmaxu4(a, b); };
    // Suffix extrema of segment [lo, lo + k) in padded positions p (pixel p - r), kept for the outputs p < n.  Positions with
    // nothing to read (p - r < 0) and nothing to keep (p >= n) are skipped in one step.
    uint32_t m = ident;
    for (int p = min(lo + k - 1, n - 1 + r); p >= lo; --p) {
        if (p >= n && p < r) p = n - 1;
        if (p >= r) m = op(m, load3(in + at(in_pitch, p - r)) ^ in_mask);
        if (p < n) store3(tmp + at(plane, p), m);
    }
    // Prefix extrema of the next segment: output i (lo < i) takes pixels up to i + r; output lo is the whole segment lo.
    uint32_t g = ident;
    const int end = min(lo + k, n);
    for (int i = lo; i < end; ++i) {
        if (i > lo && i + r < n) g = op(g, load3(in + at(in_pitch, i + r)) ^ in_mask);
        const uint32_t v = op(load3(tmp + at(plane, i)), g);
        if (kStage < 3) {
            store3(out + at(out_pitch, i), v);
        } else {
            const uint32_t f = load3(pg.src + at(pg.src_pitch, i)) ^ mask;
            const uint32_t e = light_div(f & 0xFF, v & 0xFF) | (light_div((f >> 8) & 0xFF, (v >> 8) & 0xFF) << 8) |
                               (light_div(f >> 16, v >> 16) << 16);
            store3(out + at(out_pitch, i), e ^ mask);
        }
    }
}

}  // namespace

extern "C" int mn_even_light_u8(const mn_text_block* blocks, const mn_light_page* pages, int n, int threshold, long long max_tiles,
                                long long max_lines, void* work, long long work_bytes, void* stream) {
    MN_REQUIRE(pages && n > 0 && n <= 65535 && max_lines > 0 && max_lines < (1ll << 40) &&
               (!threshold || (blocks && max_tiles > 0 && max_tiles < (1ll << 31) && work && work_bytes > 0)),
               "mn_even_light_u8: bad args");
    cudaStream_t st = (cudaStream_t)stream;
    if (threshold) {
        const int rc = mn_block_threshold(blocks, n, max_tiles, work, work_bytes, st);
        if (rc != MN_OK) return rc;
    }
    const dim3 grid((unsigned)mn_cdiv64(max_lines, kLightThreads), n);
    MN_CUDA_CHECK((mn_launch(light_pass_kernel<0>, grid, dim3(kLightThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(light_pass_kernel<1>, grid, dim3(kLightThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(light_pass_kernel<2>, grid, dim3(kLightThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    MN_CUDA_CHECK((mn_launch(light_pass_kernel<3>, grid, dim3(kLightThreads), 0, st, pages)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
