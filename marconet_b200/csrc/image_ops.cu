// Host pre/post-processing of the reference scripts moved onto the device (SURVEY 8f n2, row a18):
//   test_sr.py:98-111   cv2.resize(img, (0,0), fx=32/h, fy=32/h, INTER_CUBIC) -> zero-pad to 32x512 -> ToTensor -> Normalize(.5,.5)
//   test_sr.py:198-201  sr*0.5+0.5 -> HWC -> channel flip -> clip(.,0,1)*255 -> (cv2.imwrite :231) round to uint8
// Byte/integer work: results are bit-identical to OpenCV's own 8-bit cubic resize (imgproc/src/resize.cpp: fp32
// interpolateCubic with A=-0.75, taps rounded to 11-bit fixed point, integer horizontal pass with replicated borders, vertical
// pass in fp32 -- separate multiply and add, rows 3..0, round-half-even -- for the first floor(W*cn/8)*8 elements of a row (the
// baseline-SSE vector body) and in fixed point for the tail) and to torchvision's ToTensor/Normalize arithmetic.
// HBM-bound and tiny (one 32x512 line); every float operation uses an explicit-rounding intrinsic so that nvcc cannot contract
// a multiply-add into an FMA the CPU code does not have.
#include "mn_common.cuh"

namespace {

struct CubicTaps { int ofs; int t[4]; };

// OpenCV's interpolateCubic (A = -0.75) at fraction f, every fp32 operation rounded on its own.
__device__ __forceinline__ void cubic_coeffs(float f, float c[4]) {
    const float A = -0.75f;
    const float xp1 = __fadd_rn(f, 1.f), omx = __fsub_rn(1.f, f);
    c[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, xp1), 5.f * A), xp1), 8.f * A), xp1), 4.f * A);
    c[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, f), A + 3.f), f), f), 1.f);
    c[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, omx), A + 3.f), omx), omx), 1.f);
    c[3] = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c[0]), c[1]), c[2]);
}

__device__ __forceinline__ CubicTaps cubic_taps(int d, double scale) {
    // fx = (float)((dx+0.5)*scale_x - 0.5); sx = cvFloor(fx); fx -= sx;  ialpha = saturate_cast<short>(coeff * 2048)
    float f = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
    const int s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    float c[4];
    cubic_coeffs(f, c);
    CubicTaps r;
    r.ofs = s;
#pragma unroll
    for (int k = 0; k < 4; ++k) r.t[k] = __float2int_rn(__fmul_rn(c[k], 2048.f));
    return r;
}

// OpenCV's 8-bit INTER_CUBIC value of one destination element: source channel sc at the destination pixel whose taps are
// (tx, ty), for an h x w image whose rows start `row_pitch` bytes apart.  The taps replicate the border of [0, h) x [0, w): a crop
// passed as (pointer to its first pixel, the source image's pitch, its own size) is resized as an isolated image.  `vec`: the
// element lies in the vector body of VResizeCubicVec_32s8u (the first floor(dw*cn/8)*8 elements of a destination row, dw*cn
// counted in the destination's channel order), else in the fixed-point tail.  Byte offsets are 64-bit.
__device__ __forceinline__ int cubic_u8(const uint8_t* __restrict__ img, long long row_pitch, int h, int w, int cn, int sc,
                                        const CubicTaps& tx, const CubicTaps& ty, bool vec) {
    int S[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int yy = min(max(ty.ofs - 1 + r, 0), h - 1);
        int acc = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int xx = min(max(tx.ofs - 1 + j, 0), w - 1);
            acc += (int)img[(long long)yy * row_pitch + (long long)xx * cn + sc] * tx.t[j];
        }
        S[r] = acc;
    }
    int v;
    if (vec) {                                            // vector body of VResizeCubicVec_32s8u: fp32, mul then add, rows 3..0
        const float f = 1.f / (2048.f * 2048.f);
        float acc = __fmul_rn((float)S[3], __fmul_rn((float)ty.t[3], f));
        acc = __fadd_rn(__fmul_rn((float)S[2], __fmul_rn((float)ty.t[2], f)), acc);
        acc = __fadd_rn(__fmul_rn((float)S[1], __fmul_rn((float)ty.t[1], f)), acc);
        acc = __fadd_rn(__fmul_rn((float)S[0], __fmul_rn((float)ty.t[0], f)), acc);
        v = __float2int_rn(acc);
    } else {                                              // scalar tail: FixedPtCast<int, uchar, 22>
        v = (S[0] * ty.t[0] + S[1] * ty.t[1] + S[2] * ty.t[2] + S[3] * ty.t[3] + (1 << 21)) >> 22;
    }
    return min(max(v, 0), 255);
}

// One canvas element (idx over [out_h][out_w][cn]) of test_sr.py:98-111 for an 8-bit image whose rows start `row_pitch` bytes
// apart (cubic_u8: a crop is resized as an isolated image, exactly what cv2.resize(img[:, a:b], ...) computes).
// Returns the resized byte (0 outside the dh x dw image); lq (fp32 canvas) and lq_u8 (resized bytes) are optional outputs.
__device__ __forceinline__ int preprocess_lq_element(const uint8_t* __restrict__ img, long long row_pitch, int h, int w, int cn,
                                                     double scale_x, double scale_y, int dh, int dw, int idx,
                                                     float* __restrict__ lq, uint8_t* __restrict__ lq_u8, int out_h, int out_w) {
    const int c = idx % cn;
    const int dx = (idx / cn) % out_w;
    const int dy = idx / (cn * out_w);
    int v = 0;                                            // the canvas is zero outside the resized image (test_sr.py:104-106)
    if (dx < dw && dy < dh) {
        v = cubic_u8(img, row_pitch, h, w, cn, c, cubic_taps(dx, scale_x), cubic_taps(dy, scale_y), dx * cn + c < (dw * cn / 8) * 8);
        if (lq_u8) lq_u8[((size_t)dy * dw + dx) * cn + c] = (uint8_t)v;
    }
    if (lq) {
        // ToTensor: float(u8) / 255 ; Normalize: (x - 0.5) / 0.5
        const float t = __fdiv_rn(__fsub_rn(__fdiv_rn((float)v, 255.f), 0.5f), 0.5f);
        lq[((size_t)c * out_h + dy) * out_w + dx] = t;
    }
    return v;
}

__global__ void preprocess_lq_kernel(const uint8_t* __restrict__ img, int h, int w, int cn, double scale_x, double scale_y,
                                     int dh, int dw, float* __restrict__ lq, uint8_t* __restrict__ lq_u8, int out_h, int out_w) {
    mn_pdl_prologue();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= out_h * out_w * cn) return;
    preprocess_lq_element(img, (long long)w * cn, h, w, cn, scale_x, scale_y, dh, dw, idx, lq, lq_u8, out_h, out_w);
}

// blockIdx.y = crop; every crop fills its own [cn][out_h][out_w] canvas of lq.
__global__ void preprocess_lq_crops_kernel(const mn_lq_crop* __restrict__ crops, int cn, float* __restrict__ lq, int out_h, int out_w) {
    mn_pdl_prologue();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= out_h * out_w * cn) return;
    const mn_lq_crop k = crops[blockIdx.y];
    preprocess_lq_element(k.img, k.row_pitch, k.h, k.w, cn, __ddiv_rn(1.0, k.fx), __ddiv_rn(1.0, k.fy), k.dh, k.dw, idx,
                          lq + (size_t)blockIdx.y * cn * out_h * out_w, nullptr, out_h, out_w);
}

// test_sr.py:198-201 + cv2.imwrite's rounding for one value
__device__ __forceinline__ uint8_t sr_to_u8(float x) {
    float v = __fadd_rn(__fmul_rn(x, 0.5f), 0.5f);
    v = fminf(fmaxf(v, 0.f), 1.f);
    const int q = __float2int_rn(__fmul_rn(v, 255.f));
    return (uint8_t)min(max(q, 0), 255);
}

__global__ void postprocess_sr_kernel(const float* __restrict__ sr, long long sn, long long sc, long long sh, long long sw,
                                      uint8_t* __restrict__ out, int B, int C, int H, int W) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)B * H * W) return;
    const int x = (int)(idx % W), y = (int)((idx / W) % H), b = (int)(idx / ((long long)W * H));
    const float* p = sr + b * sn + y * sh + x * sw;
    uint8_t* o = out + idx * C;
    for (int c = 0; c < C; ++c) o[C - 1 - c] = sr_to_u8(p[c * sc]);          // .flip(2): channel c lands in byte C-1-c
}

// blockIdx.y = piece; threads cover [H][max_width] pixels, those at x >= the piece's width exit.
__global__ void postprocess_sr_pieces_kernel(const float* __restrict__ sr, long long sn, long long sc, long long sh, long long sw,
                                             int C, int H, const mn_sr_piece* __restrict__ pieces, int max_width) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)H * max_width) return;
    const mn_sr_piece pc = pieces[blockIdx.y];
    const int x = (int)(idx % max_width), y = (int)(idx / max_width);
    if (x >= pc.width) return;
    const float* p = sr + pc.line * sn + y * sh + (long long)(pc.src_x0 + x) * sw;
    uint8_t* o = pc.dst + y * pc.dst_pitch + (long long)x * C;
    for (int c = 0; c < C; ++c) o[C - 1 - c] = sr_to_u8(p[c * sc]);
}

// test_sr.py:206-211 for one value of the prior strip hstack(prior*0.5+0.5): character k, channel c, row y, column x.
__device__ __forceinline__ float prior_value(const mn_figure_prior* __restrict__ pr, int k, int c, int y, int x) {
    const mn_figure_prior p = pr[k];
    return __fadd_rn(__fmul_rn(p.img[c * p.stride_c + y * p.stride_h + x * p.stride_w], 0.5f), 0.5f);
}

// *255, cvRound and saturation: how cv2.imwrite stores a float prior value (test_sr.py:210-231, test_w.py:114).
__device__ __forceinline__ uint8_t prior_u8(float v) {
    const int q = __float2int_rn(__fmul_rn(v, 255.f));
    return (uint8_t)min(max(q, 0), 255);
}

// blockIdx.y = image; one thread per pixel (y, x) of the 128 x max_width panel rows, those at x >= the image's W exit.
// Panels 1-2 (ShowLQ, ShowLocs; test_sr.py:98,214-231) share one cubic resize (preprocess_lq_element at fx = fy = 128/h, the
// vector / tail split taken at width S); panel 4 is OpenCV's float INTER_LINEAR of the prior strip to width S (test_sr.py:210),
// *255 and cvRound with saturation (cv2.imwrite).  Panel 3 (ShowSR) is written by postprocess_sr_pieces_kernel.
__global__ void figure_kernel(const mn_figure_image* __restrict__ images, int max_width) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 128ll * max_width) return;
    const mn_figure_image im = images[blockIdx.y];
    const int x = (int)(idx % max_width), y = (int)(idx / max_width);
    if (x >= im.W) return;
    uint8_t* row = im.fig + (long long)y * im.fig_pitch + (long long)x * 3;

    const double fx = __ddiv_rn(128.0, (double)im.h), scale = __ddiv_rn(1.0, fx);       // the script's fx=128/h
    const int* marks = im.marks + (y < 64 ? 0 : 2 * im.n_top);
    const int n_marks = y < 64 ? im.n_top : im.n_bot;
    bool marked = false;
    for (int m = 0; m < n_marks; ++m) marked |= (x >= marks[2 * m]) & (x < marks[2 * m + 1]);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int v = preprocess_lq_element(im.img, im.row_pitch, im.h, im.w, 3, scale, scale, 128, im.S, (y * im.S + x) * 3 + c,
                                            nullptr, nullptr, 128, im.S);
        // ShowLocs: (255, 0, 0) at the x markers of rows 0-63, (0, 0, 255) at the y markers of rows 64-127; both panels flipped
        const int mark = c == (y < 64 ? 0 : 2) ? 255 : 0;
        row[2 - c] = (uint8_t)v;
        row[128 * im.fig_pitch + 2 - c] = (uint8_t)(marked ? mark : v);
    }

    const int sw = 128 * im.n_chars;
    float a1 = 0.f;
    int sx = x;
    if (im.S != sw) {                                    // cv2.resize copies when the size is unchanged
        const double sc = __ddiv_rn(1.0, __ddiv_rn((double)im.S, (double)sw));
        float f = __double2float_rn(__dsub_rn(__dmul_rn((double)x + 0.5, sc), 0.5));
        sx = (int)floorf(f);
        a1 = __fsub_rn(f, (float)sx);
        if (sx < 0) sx = 0, a1 = 0.f;
        if (sx >= sw - 1) sx = sw - 1, a1 = 0.f;
    }
    const float a0 = __fsub_rn(1.f, a1);
    const int s1 = min(sx + 1, sw - 1);
    uint8_t* prow = row + 384 * im.fig_pitch;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v0 = prior_value(im.priors, sx >> 7, c, y, sx & 127);
        float v = v0;
        if (im.S != sw) v = __fadd_rn(__fmul_rn(v0, a0), __fmul_rn(prior_value(im.priors, s1 >> 7, c, y, s1 & 127), a1));
        prow[c] = prior_u8(v);                           // not channel-flipped: the script writes the prior panel as RGB
    }
}

// blockIdx.y = generator image n; one thread per pixel of its 128 x 128 tile: the figure's prior panel at its identity width.
__global__ void prior_tiles_kernel(const float* __restrict__ priors, long long sn, long long sc, long long sh, long long sw,
                                   const mn_prior_tile* __restrict__ tiles) {
    mn_pdl_prologue();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 128 * 128) return;
    const int x = idx & 127, y = idx >> 7;
    const mn_figure_prior p{priors + blockIdx.y * sn, sc, sh, sw};
    const mn_prior_tile t = tiles[blockIdx.y];
    uint8_t* o = t.dst + (long long)y * t.dst_pitch + (long long)x * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = prior_u8(prior_value(&p, 0, c, y, x));
}

// blockIdx.y = image; one thread per destination pixel (row y, column x) of the [dh][dw][cn] resized image, those past its
// dh*dw pixels exit.  cv2.resize(src, (dw, dh), interpolation=INTER_CUBIC), the split at the destination's width.
__global__ void resize_cubic_batched_kernel(const mn_resize_image* __restrict__ images, int cn) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const mn_resize_image im = images[blockIdx.y];
    if (idx >= (long long)im.dh * im.dw) return;
    const int x = (int)(idx % im.dw), y = (int)(idx / im.dw);
    const CubicTaps tx = cubic_taps(x, im.scale_x), ty = cubic_taps(y, im.scale_y);
    const long long nvec = ((long long)im.dw * cn / 8) * 8;
    uint8_t* o = im.dst + (long long)y * im.dst_pitch + (long long)x * cn;
    for (int c = 0; c < cn; ++c) o[c] = (uint8_t)cubic_u8(im.src, im.src_pitch, im.h, im.w, cn, c, tx, ty, (long long)x * cn + c < nvec);
}

__device__ __forceinline__ bool region_holds(const mn_region& r, int X, int Y) {
    return X >= r.x0 && X < r.x1 && Y >= r.y0 && Y < r.y1;
}

// alpha of output pixel (X, Y) inside region r: the distance d to the nearest side not on the page border,
// min(1, fl((float)d + 0.5) / F); 1 when F = 0 or every side lies on the border.
__device__ __forceinline__ float region_alpha(const mn_region& r, int X, int Y) {
    int d = INT_MAX;
    if (r.x0 > 0) d = min(d, X - r.x0);
    if (r.x1 < r.page_w) d = min(d, r.x1 - 1 - X);
    if (r.y0 > 0) d = min(d, Y - r.y0);
    if (r.y1 < r.page_h) d = min(d, r.y1 - 1 - Y);
    if (r.feather == 0 || d == INT_MAX) return 1.f;
    return fminf(1.f, __fdiv_rn(__fadd_rn((float)d, 0.5f), (float)r.feather));
}

// P of rectangle q at output pixel (X, Y) blended over v: the cubic resize of the region's restored bytes (read through their
// pitch, channels flipped back) onto its rectangle, at OpenCV's dsize scale 1/((double)dw/sw) per axis, the vector / tail split
// taken at the rectangle's width;  v = sat_u8(rint(fl(fl(a*P) + fl(fl(1 - a)*v)))).
__device__ __forceinline__ void region_blend(const mn_region& q, int X, int Y, int v[3]) {
    const int dw = q.x1 - q.x0, dh = q.y1 - q.y0, dx = X - q.x0, dy = Y - q.y0;
    const CubicTaps tx = cubic_taps(dx, __ddiv_rn(1.0, __ddiv_rn((double)dw, (double)q.sr_w)));
    const CubicTaps ty = cubic_taps(dy, __ddiv_rn(1.0, __ddiv_rn((double)dh, (double)q.sr_h)));
    const float a = region_alpha(q, X, Y), b = __fsub_rn(1.f, a);
    const int nvec = (dw * 3 / 8) * 8;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int p = cubic_u8(q.sr, q.sr_pitch, q.sr_h, q.sr_w, 3, 2 - c, tx, ty, dx * 3 + c < nvec);
        const int t = __float2int_rn(__fadd_rn(__fmul_rn(a, (float)p), __fmul_rn(b, (float)v[c])));
        v[c] = min(max(t, 0), 255);
    }
}

// cv2.warpAffine's fixed-point source coordinates of destination pixel (x, y) under m (WARP_INVERSE_MAP), in 1/32 pixel:
// X0 = cvRound(fl(fl(m1 y) + m2) * 1024) + 16 (the row's start, round_delta = 1024/32/2), adelta = cvRound(fl(m0 x) * 1024),
// Xq = (X0 + adelta) >> 5; the source pixel is Xq >> 5 and the fraction Xq & 31.  Callers keep |fixed-point values| < 2^30.
struct WarpCoord { int xq, yq; };
__device__ __forceinline__ WarpCoord warp_coord(const double* m, int x, int y) {
    const double xd = (double)x, yd = (double)y;
    const int x0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], yd), m[2]), 1024.0)) + 16;
    const int y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], yd), m[5]), 1024.0)) + 16;
    const int ad = __double2int_rn(__dmul_rn(__dmul_rn(m[0], xd), 1024.0));
    const int bd = __double2int_rn(__dmul_rn(__dmul_rn(m[3], xd), 1024.0));
    return {(x0 + ad) >> 5, (y0 + bd) >> 5};
}

// remap's 8-bit INTER_CUBIC value at fixed-point source coordinates c with BORDER_REPLICATE: source channel sc of the h x w
// image whose rows start row_pitch bytes apart.  The 2-D taps are initInterTab2D's: w = saturate_cast<short>(fl(vy vx) * 32768)
// of the fp32 interpolateCubic weights at (Yq & 31)/32 and (Xq & 31)/32; a sum other than 32768 is corrected on the smallest
// (too large) or largest (too small) tap among rows and columns 2..3, the first found in row-major order (OpenCV searches from
// ksize/2).  Then (sum + 2^14) >> 15 saturated.  Integer sums, so the tap order is free.
__device__ __forceinline__ void warp_taps(const WarpCoord& c, int w[16]) {
    float cy[4], cx[4];
    cubic_coeffs(__fmul_rn((float)(c.yq & 31), 1.f / 32.f), cy);
    cubic_coeffs(__fmul_rn((float)(c.xq & 31), 1.f / 32.f), cx);
    int isum = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        w[k] = min(max(__float2int_rn(__fmul_rn(__fmul_rn(cy[k >> 2], cx[k & 3]), 32768.f)), -32768), 32767);
        isum += w[k];
    }
    const int diff = isum - 32768;
    int mk = 10, Mk = 10, mv = w[10], Mv = w[10];         // from tap (2, 2) over (2, 3), (3, 2), (3, 3)
#pragma unroll
    for (int k = 11; k < 16; k += (k == 11) ? 3 : 1) {
        if (w[k] < mv) mv = w[k], mk = k;
        else if (w[k] > Mv) Mv = w[k], Mk = k;
    }
    const int fix = diff < 0 ? Mk : mk;
#pragma unroll
    for (int k = 10; k < 16; ++k) w[k] -= (diff != 0 && k == fix) ? diff : 0;
}

__device__ __forceinline__ int warp_cubic_u8(const uint8_t* __restrict__ img, long long row_pitch, int h, int w, int cn, int sc,
                                             const WarpCoord& c, const int wt[16]) {
    const int ix = c.xq >> 5, iy = c.yq >> 5;
    int acc = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const uint8_t* row = img + (long long)min(max(iy - 1 + r, 0), h - 1) * row_pitch + sc;
#pragma unroll
        for (int j = 0; j < 4; ++j) acc += (int)row[(long long)min(max(ix - 1 + j, 0), w - 1) * cn] * wt[4 * r + j];
    }
    return min(max((acc + (1 << 14)) >> 15, 0), 255);
}

// cv2.warpPerspective's fixed-point source coordinates of pixel (x, y) of a dw x dh destination under the 3 x 3 m
// (WARP_INVERSE_MAP), in 1/32 pixel.  OpenCV walks the destination in column blocks of bw = min(1024 / min(16, dh), dw) and at
// each block's first column xb forms X0 = fl(fl(fl(m0 xb) + fl(m1 y)) + m2) (Y0, W0 likewise); then with x1 = x - xb,
// W = fl(W0 + fl(m6 x1)), W = W ? fl(32 / W) : 0, Xq = cvRound(clamp(fl(fl(X0 + fl(m0 x1)) W), INT_MIN, INT_MAX)).  The block
// origin changes the rounding, so it is part of the result.
__device__ __forceinline__ WarpCoord warp_coord_perspective(const double* m, int x, int y, int dw, int dh) {
    const int bw = min(1024 / min(16, dh), dw);
    const double xb = (double)(x - x % bw), x1 = (double)(x % bw), yd = (double)y;
    const double x0 = __dadd_rn(__dadd_rn(__dmul_rn(m[0], xb), __dmul_rn(m[1], yd)), m[2]);
    const double y0 = __dadd_rn(__dadd_rn(__dmul_rn(m[3], xb), __dmul_rn(m[4], yd)), m[5]);
    const double w0 = __dadd_rn(__dadd_rn(__dmul_rn(m[6], xb), __dmul_rn(m[7], yd)), m[8]);
    double w = __dadd_rn(w0, __dmul_rn(m[6], x1));
    w = w != 0.0 ? __ddiv_rn(32.0, w) : 0.0;
    const double fx = fmin(fmax(__dmul_rn(__dadd_rn(x0, __dmul_rn(m[0], x1)), w), (double)INT_MIN), (double)INT_MAX);
    const double fy = fmin(fmax(__dmul_rn(__dadd_rn(y0, __dmul_rn(m[3], x1)), w), (double)INT_MIN), (double)INT_MAX);
    return {__double2int_rn(fx), __double2int_rn(fy)};
}

__device__ __forceinline__ bool footprint_holds(const mn_region& r, const WarpCoord& c) {
    return c.xq >= -16 && c.xq < 32 * r.sr_w - 16 && c.yq >= -16 && c.yq < 32 * r.sr_h - 16;
}

__device__ __forceinline__ bool region_holds(const mn_region_affine& q, int X, int Y) {
    if (!region_holds(q.r, X, Y)) return false;
    return q.kind == MN_REGION_RECT || footprint_holds(q.r, warp_coord(q.n, X, Y));
}

// P of a warped region r (T = r.sr) at fixed-point T coordinates wc, feathered with slopes kx, ky on all four sides, blended over v.
__device__ __forceinline__ void footprint_blend(const mn_region& r, float kx, float ky, const WarpCoord& wc, int v[3]) {
    float a = 1.f;
    if (r.feather != 0) {
        const float u = __fmul_rn((float)(wc.xq + 16), 1.f / 32.f), t = __fmul_rn((float)(wc.yq + 16), 1.f / 32.f);
        const float du = __fmul_rn(kx, fminf(u, __fsub_rn((float)r.sr_w, u)));
        const float dv = __fmul_rn(ky, fminf(t, __fsub_rn((float)r.sr_h, t)));
        a = fminf(1.f, __fdiv_rn(fminf(du, dv), (float)r.feather));
    }
    const float b = __fsub_rn(1.f, a);
    int wt[16];
    warp_taps(wc, wt);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int p = warp_cubic_u8(r.sr, r.sr_pitch, r.sr_h, r.sr_w, 3, 2 - c, wc, wt);
        const int t = __float2int_rn(__fadd_rn(__fmul_rn(a, (float)p), __fmul_rn(b, (float)v[c])));
        v[c] = min(max(t, 0), 255);
    }
}

__device__ __forceinline__ void region_blend(const mn_region_affine& q, int X, int Y, int v[3]) {
    if (q.kind == MN_REGION_RECT) {
        region_blend(q.r, X, Y, v);
        return;
    }
    footprint_blend(q.r, q.kx, q.ky, warp_coord(q.n, X, Y), v);
}

// The T coordinates of page pixel (X, Y) under an affine or perspective region's n (the whole page is the destination).
__device__ __forceinline__ WarpCoord quad_coord(const mn_region_quad& q, int X, int Y) {
    return q.kind == MN_REGION_PERSPECTIVE ? warp_coord_perspective(q.n, X, Y, q.r.page_w, q.r.page_h) : warp_coord(q.n, X, Y);
}

__device__ __forceinline__ bool region_holds(const mn_region_quad& q, int X, int Y) {
    if (!region_holds(q.r, X, Y)) return false;
    return q.kind == MN_REGION_RECT || footprint_holds(q.r, quad_coord(q, X, Y));
}

__device__ __forceinline__ void region_blend(const mn_region_quad& q, int X, int Y, int v[3]) {
    if (q.kind == MN_REGION_RECT) {
        region_blend(q.r, X, Y, v);
        return;
    }
    footprint_blend(q.r, q.kx, q.ky, quad_coord(q, X, Y), v);
}

__device__ __forceinline__ const mn_region& rect_of(const mn_region& r) { return r; }
__device__ __forceinline__ const mn_region& rect_of(const mn_region_affine& r) { return r.r; }
__device__ __forceinline__ const mn_region& rect_of(const mn_region_quad& r) { return r.r; }

// Curved text regions (DESIGN.md 7b, "Curved text regions").  One lerp of de Casteljau's: fl(fl(s a) + fl(t b)), s = 1 - t.
__device__ __forceinline__ double bez_lerp(double a, double b, double s, double t) {
    return __dadd_rn(__dmul_rn(s, a), __dmul_rn(t, b));
}

// The cubic Bezier of the 4 (x, y) points at p (x, y interleaved) at t, three levels of lerps per coordinate.
struct Pt { double x, y; };
__device__ __forceinline__ Pt bezier(const double* __restrict__ p, double t) {
    const double s = __dsub_rn(1.0, t);
    double c[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const double a0 = bez_lerp(p[k], p[2 + k], s, t), a1 = bez_lerp(p[2 + k], p[4 + k], s, t);
        const double a2 = bez_lerp(p[4 + k], p[6 + k], s, t);
        c[k] = bez_lerp(bez_lerp(a0, a1, s, t), bez_lerp(a1, a2, s, t), s, t);
    }
    return {c[0], c[1]};
}

// The top and bottom control points of segment m of a curve table with k segments (layout: mn_remap_curved_image).
__device__ __forceinline__ const double* curve_top(const double* curve, int k, int m) { return curve + k + 2 + 6 * m; }
__device__ __forceinline__ const double* curve_bottom(const double* curve, int k, int m) { return curve + 7 * k + 4 + 6 * m; }

// The crop map of crop pixel (x, y) of a dw x dh rectified crop, as fixed-point remap coordinates rint(fl32(map) 32).
__device__ __forceinline__ WarpCoord curved_crop_coord(const double* __restrict__ curve, int k, int x, int y, int dw, int dh) {
    const double a = __ddiv_rn(__dadd_rn((double)x, 0.5), (double)dw), b = __ddiv_rn(__dadd_rn((double)y, 0.5), (double)dh);
    const double* c = curve + 1;
    int m = 0;
    for (int j = 1; j < k; ++j) m = c[j] <= a ? j : m;
    const double t = __ddiv_rn(__dsub_rn(a, c[m]), __dsub_rn(c[m + 1], c[m]));
    const Pt T = bezier(curve_top(curve, k, m), t), B = bezier(curve_bottom(curve, k, m), t);
    const double omb = __dsub_rn(1.0, b);
    const double mx = __dsub_rn(__dadd_rn(__dmul_rn(omb, T.x), __dmul_rn(b, B.x)), 0.5);
    const double my = __dsub_rn(__dadd_rn(__dmul_rn(omb, T.y), __dmul_rn(b, B.y)), 0.5);
    return {__float2int_rn(__fmul_rn(__double2float_rn(mx), 32.f)), __float2int_rn(__fmul_rn(__double2float_rn(my), 32.f))};
}

// g(t) = cross(d, p - T) of segment (top, bot) at t, d = B - T: the side of the ruling at t on which p lies.
__device__ __forceinline__ double ruling_side(const double* __restrict__ top, const double* __restrict__ bot, double px, double py,
                                              double t) {
    const Pt T = bezier(top, t), B = bezier(bot, t);
    const double dx = __dsub_rn(B.x, T.x), dy = __dsub_rn(B.y, T.y);
    return __dsub_rn(__dmul_rn(dx, __dsub_rn(py, T.y)), __dmul_rn(dy, __dsub_rn(px, T.x)));
}

// The T coordinates of page pixel (X, Y) under a curved region: false where no segment accepts the pixel.
__device__ __forceinline__ bool curved_coord(const mn_region_curved& q, int X, int Y, WarpCoord& wc) {
    const double* curve = q.curve;
    const int k = q.n_seg;
    const double s = curve[0];
    const double px = __ddiv_rn(__dadd_rn((double)X, 0.5), s), py = __ddiv_rn(__dadd_rn((double)Y, 0.5), s);
    for (int m = 0; m < k; ++m) {
        const double* top = curve_top(curve, k, m);
        const double* bot = curve_bottom(curve, k, m);
        double x0 = top[0], x1 = top[0], y0 = top[1], y1 = top[1];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            x0 = fmin(x0, fmin(top[2 * j], bot[2 * j])), x1 = fmax(x1, fmax(top[2 * j], bot[2 * j]));
            y0 = fmin(y0, fmin(top[2 * j + 1], bot[2 * j + 1])), y1 = fmax(y1, fmax(top[2 * j + 1], bot[2 * j + 1]));
        }
        if (!(px >= x0 && px <= x1 && py >= y0 && py <= y1)) continue;
        const bool neg = ruling_side(top, bot, px, py, 0.0) < 0.0;
        if (neg == (ruling_side(top, bot, px, py, 1.0) < 0.0)) continue;
        double lo = 0.0, hi = 1.0;
        for (int it = 0; it < 48; ++it) {
            const double mid = __dmul_rn(0.5, __dadd_rn(lo, hi));
            if ((ruling_side(top, bot, px, py, mid) < 0.0) == neg) lo = mid; else hi = mid;
        }
        const double t = __dmul_rn(0.5, __dadd_rn(lo, hi));
        const Pt T = bezier(top, t), B = bezier(bot, t);
        const double dx = __dsub_rn(B.x, T.x), dy = __dsub_rn(B.y, T.y), rx = __dsub_rn(px, T.x), ry = __dsub_rn(py, T.y);
        const double b = __ddiv_rn(__dadd_rn(__dmul_rn(rx, dx), __dmul_rn(ry, dy)), __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
        if (!(b >= 0.0 && b <= 1.0)) continue;
        const double* c = curve + 1;
        const double a = __dadd_rn(c[m], __dmul_rn(t, __dsub_rn(c[m + 1], c[m])));
        const double u = __dsub_rn(__dmul_rn(a, (double)q.q.r.sr_w), 0.5), v = __dsub_rn(__dmul_rn(b, (double)q.q.r.sr_h), 0.5);
        wc = {__float2int_rn(__fmul_rn(__double2float_rn(u), 32.f)), __float2int_rn(__fmul_rn(__double2float_rn(v), 32.f))};
        return true;
    }
    return false;
}

__device__ __forceinline__ bool region_holds(const mn_region_curved& q, int X, int Y) {
    if (q.q.kind != MN_REGION_CURVED) return region_holds(q.q, X, Y);
    if (!region_holds(q.q.r, X, Y)) return false;
    WarpCoord wc;
    return curved_coord(q, X, Y, wc) && footprint_holds(q.q.r, wc);
}

__device__ __forceinline__ void region_blend(const mn_region_curved& q, int X, int Y, int v[3]) {
    if (q.q.kind != MN_REGION_CURVED) {
        region_blend(q.q, X, Y, v);
        return;
    }
    WarpCoord wc;
    curved_coord(q, X, Y, wc);                             // region_holds accepted the pixel
    footprint_blend(q.q.r, q.q.kx, q.q.ky, wc, v);
}

__device__ __forceinline__ const mn_region& rect_of(const mn_region_curved& r) { return r.q.r; }

// blockIdx.y = region; one thread per output pixel of its rectangle, those past its pixels (or outside its footprint) exit.  The
// pixel belongs to the last region of its chain (every region of the page whose rectangle meets this one, in page order) that
// holds it; only that region's thread writes it, composing the page's background through every region of the chain that holds
// it, in order (region_blend).
template <class Region>
__device__ __forceinline__ void composite_pixel(const Region* __restrict__ regions) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int me = blockIdx.y;
    const Region r = regions[me];
    const mn_region& rr = rect_of(r);
    const int rw = rr.x1 - rr.x0;
    if (idx >= (long long)rw * (rr.y1 - rr.y0)) return;
    const int X = rr.x0 + (int)(idx % rw), Y = rr.y0 + (int)(idx / rw);
    if (!region_holds(r, X, Y)) return;
    for (int k = rr.n_chain - 1; k >= 0; --k) {
        const int j = rr.chain[k];
        if (j == me) break;
        if (region_holds(regions[j], X, Y)) return;                     // a later region owns the pixel
    }
    uint8_t* o = rr.page + (long long)Y * rr.page_pitch + (long long)X * 3;
    int v[3] = {o[0], o[1], o[2]};
    for (int k = 0; k < rr.n_chain; ++k) {
        const int j = rr.chain[k];
        const Region q = regions[j];
        if (region_holds(q, X, Y)) region_blend(q, X, Y, v);
        if (j == me) break;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (uint8_t)v[c];
}

__global__ void composite_regions_kernel(const mn_region* __restrict__ regions) {
    mn_pdl_prologue();
    composite_pixel(regions);
}

__global__ void composite_regions_affine_kernel(const mn_region_affine* __restrict__ regions) {
    mn_pdl_prologue();
    composite_pixel(regions);
}

// blockIdx.y = image; one thread per destination pixel of its [dh][dw][cn] image, those past its dh*dw pixels exit.
__global__ void warp_affine_batched_kernel(const mn_warp_image* __restrict__ images, int cn) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const mn_warp_image im = images[blockIdx.y];
    if (idx >= (long long)im.dh * im.dw) return;
    const int x = (int)(idx % im.dw), y = (int)(idx / im.dw);
    const WarpCoord wc = warp_coord(im.m, x, y);
    int wt[16];
    warp_taps(wc, wt);
    uint8_t* o = im.dst + (long long)y * im.dst_pitch + (long long)x * cn;
    for (int c = 0; c < cn; ++c) o[c] = (uint8_t)warp_cubic_u8(im.src, im.src_pitch, im.h, im.w, cn, c, wc, wt);
}

__global__ void composite_regions_quad_kernel(const mn_region_quad* __restrict__ regions) {
    mn_pdl_prologue();
    composite_pixel(regions);
}

// blockIdx.y = image; one thread per destination pixel of its [dh][dw][cn] image, those past its dh*dw pixels exit.
__global__ void warp_perspective_batched_kernel(const mn_warp_perspective_image* __restrict__ images, int cn) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const mn_warp_perspective_image im = images[blockIdx.y];
    if (idx >= (long long)im.dh * im.dw) return;
    const int x = (int)(idx % im.dw), y = (int)(idx / im.dw);
    const WarpCoord wc = warp_coord_perspective(im.m, x, y, im.dw, im.dh);
    int wt[16];
    warp_taps(wc, wt);
    uint8_t* o = im.dst + (long long)y * im.dst_pitch + (long long)x * cn;
    for (int c = 0; c < cn; ++c) o[c] = (uint8_t)warp_cubic_u8(im.src, im.src_pitch, im.h, im.w, cn, c, wc, wt);
}

__global__ void composite_regions_curved_kernel(const mn_region_curved* __restrict__ regions) {
    mn_pdl_prologue();
    composite_pixel(regions);
}

// blockIdx.y = image; one thread per destination pixel of its [dh][dw][cn] crop, those past its dh*dw pixels exit.
__global__ void remap_curved_batched_kernel(const mn_remap_curved_image* __restrict__ images, int cn) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const mn_remap_curved_image im = images[blockIdx.y];
    if (idx >= (long long)im.dh * im.dw) return;
    const int x = (int)(idx % im.dw), y = (int)(idx / im.dw);
    const WarpCoord wc = curved_crop_coord(im.curve, im.n_seg, x, y, im.dw, im.dh);
    int wt[16];
    warp_taps(wc, wt);
    uint8_t* o = im.dst + (long long)y * im.dst_pitch + (long long)x * cn;
    for (int c = 0; c < cn; ++c) o[c] = (uint8_t)warp_cubic_u8(im.src, im.src_pitch, im.h, im.w, cn, c, wc, wt);
}

// blockIdx.y = column; one thread per destination pixel of its [dh][dw][3] destination, those past its dh*dw pixels exit.
// kUnlayout false: the layout of C into the line L, the cell picked by the destination column; true: the inverse layout of T
// into T_col, the cell picked by the destination row (the last k with R(c_k) <= y, a binary search over the table).
template <bool kUnlayout>
__global__ void vertical_gather_kernel(const mn_vertical_column* __restrict__ columns) {
    mn_pdl_prologue();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const mn_vertical_column col = columns[blockIdx.y];
    if (idx >= (long long)col.dh * col.dw) return;
    const int x = (int)(idx % col.dw), y = (int)(idx / col.dw);
    int sy, sx;
    if (!kUnlayout) {
        const int k = x / col.w;
        const int* t = col.cells + 3 * k;
        sy = t[0] + min(max(y - t[1], 0), t[2] - 1);
        sx = x - k * col.w;
    } else {
        int lo = 0, hi = col.n_cells - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (col.cells[5 * mid] <= y) lo = mid; else hi = mid - 1;
        }
        const int* t = col.cells + 5 * lo;
        sy = min(max(t[1] + y - t[0], t[1]), t[2] - 1);
        sx = min(max(t[3] + x, t[3]), t[4] - 1);
    }
    const uint8_t* s = col.src + (long long)sy * col.src_pitch + (long long)sx * 3;
    uint8_t* o = col.dst + (long long)y * col.dst_pitch + (long long)x * 3;
    o[0] = s[0];
    o[1] = s[1];
    o[2] = s[2];
}

}  // namespace

template <bool kUnlayout>
static int vertical_gather(const mn_vertical_column* columns, int n, long long max_pixels, void* stream, const char* what) {
    MN_REQUIRE(columns && n > 0 && n <= 65535 && max_pixels > 0, "%s: bad args", what);
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "%s: %lld pixels exceed the grid", what, max_pixels);
    MN_CUDA_CHECK((mn_launch(vertical_gather_kernel<kUnlayout>, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, columns)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_vertical_layout_u8_batched(const mn_vertical_column* columns, int n, long long max_pixels, void* stream) {
    return vertical_gather<false>(columns, n, max_pixels, stream, "mn_vertical_layout_u8_batched");
}

extern "C" int mn_vertical_unlayout_u8_batched(const mn_vertical_column* columns, int n, long long max_pixels, void* stream) {
    return vertical_gather<true>(columns, n, max_pixels, stream, "mn_vertical_unlayout_u8_batched");
}

extern "C" int mn_resize_cubic_u8_batched(const mn_resize_image* images, int n, int cn, long long max_pixels, void* stream) {
    MN_REQUIRE(images && n > 0 && n <= 65535 && cn > 0 && cn <= 4 && max_pixels > 0, "mn_resize_cubic_u8_batched: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_resize_cubic_u8_batched: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(resize_cubic_batched_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, images, cn)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_composite_regions_u8(const mn_region* regions, int n, long long max_pixels, void* stream) {
    MN_REQUIRE(regions && n > 0 && n <= 65535 && max_pixels > 0, "mn_composite_regions_u8: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_composite_regions_u8: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(composite_regions_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, regions)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_warp_affine_u8_batched(const mn_warp_image* images, int n, int cn, long long max_pixels, void* stream) {
    MN_REQUIRE(images && n > 0 && n <= 65535 && cn > 0 && cn <= 4 && max_pixels > 0, "mn_warp_affine_u8_batched: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_warp_affine_u8_batched: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(warp_affine_batched_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, images, cn)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_composite_regions_affine_u8(const mn_region_affine* regions, int n, long long max_pixels, void* stream) {
    MN_REQUIRE(regions && n > 0 && n <= 65535 && max_pixels > 0, "mn_composite_regions_affine_u8: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_composite_regions_affine_u8: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(composite_regions_affine_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, regions)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_warp_perspective_u8_batched(const mn_warp_perspective_image* images, int n, int cn, long long max_pixels,
                                              void* stream) {
    MN_REQUIRE(images && n > 0 && n <= 65535 && cn > 0 && cn <= 4 && max_pixels > 0, "mn_warp_perspective_u8_batched: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_warp_perspective_u8_batched: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(warp_perspective_batched_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, images, cn)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_composite_regions_quad_u8(const mn_region_quad* regions, int n, long long max_pixels, void* stream) {
    MN_REQUIRE(regions && n > 0 && n <= 65535 && max_pixels > 0, "mn_composite_regions_quad_u8: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_composite_regions_quad_u8: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(composite_regions_quad_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, regions)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_remap_curved_u8_batched(const mn_remap_curved_image* images, int n, int cn, long long max_pixels, void* stream) {
    MN_REQUIRE(images && n > 0 && n <= 65535 && cn > 0 && cn <= 4 && max_pixels > 0, "mn_remap_curved_u8_batched: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_remap_curved_u8_batched: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(remap_curved_batched_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, images, cn)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_composite_regions_curved_u8(const mn_region_curved* regions, int n, long long max_pixels, void* stream) {
    MN_REQUIRE(regions && n > 0 && n <= 65535 && max_pixels > 0, "mn_composite_regions_curved_u8: bad args");
    MN_REQUIRE(max_pixels < (1ll << 31) * 256, "mn_composite_regions_curved_u8: %lld pixels exceed the grid", max_pixels);
    MN_CUDA_CHECK((mn_launch(composite_regions_curved_kernel, dim3((unsigned)mn_cdiv64(max_pixels, 256), n), dim3(256), 0,
                             (cudaStream_t)stream, regions)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_preprocess_lq_u8(const uint8_t* img, int h, int w, int cn, double fx, double fy, int dh, int dw,
                                   float* lq, uint8_t* lq_u8, int out_h, int out_w, void* stream) {
    MN_REQUIRE(img && lq && h > 0 && w > 0 && cn > 0 && cn <= 4 && fx > 0.0 && fy > 0.0, "mn_preprocess_lq_u8: bad args");
    MN_REQUIRE(dh > 0 && dw > 0 && dh <= out_h && dw <= out_w, "mn_preprocess_lq_u8: resized image (%dx%d) does not fit the %dx%d canvas "
               "(test_sr.py:109 skips such images)", dh, dw, out_h, out_w);
    MN_REQUIRE((long long)out_h * out_w * cn < (1ll << 31), "mn_preprocess_lq_u8: canvas too large");
    const int total = out_h * out_w * cn;
    MN_CUDA_CHECK((mn_launch(preprocess_lq_kernel, dim3(mn_cdiv(total, 128)), dim3(128), 0, (cudaStream_t)stream, img, h, w, cn,
                             1.0 / fx, 1.0 / fy, dh, dw, lq, lq_u8, out_h, out_w)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_postprocess_sr_u8(const float* sr, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                                    uint8_t* out, int B, int C, int H, int W, void* stream) {
    MN_REQUIRE(sr && out && B > 0 && C > 0 && C <= 4 && H > 0 && W > 0, "mn_postprocess_sr_u8: bad args");
    const long long total = (long long)B * H * W;
    MN_CUDA_CHECK((mn_launch(postprocess_sr_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, (cudaStream_t)stream, sr, stride_n, stride_c,
                             stride_h, stride_w, out, B, C, H, W)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_preprocess_lq_u8_batched(const mn_lq_crop* crops, int n, int cn, float* lq, int out_h, int out_w, void* stream) {
    MN_REQUIRE(crops && lq && n > 0 && n <= 65535 && cn > 0 && cn <= 4 && out_h > 0 && out_w > 0, "mn_preprocess_lq_u8_batched: bad args");
    MN_REQUIRE((long long)out_h * out_w * cn < (1ll << 31), "mn_preprocess_lq_u8_batched: canvas too large");
    const int total = out_h * out_w * cn;
    MN_CUDA_CHECK((mn_launch(preprocess_lq_crops_kernel, dim3(mn_cdiv(total, 128), n), dim3(128), 0, (cudaStream_t)stream, crops, cn,
                             lq, out_h, out_w)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_postprocess_sr_u8_pieces(const float* sr, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                                           int C, int H, int W, const mn_sr_piece* pieces, int n_pieces, int max_width, void* stream) {
    MN_REQUIRE(sr && pieces && C > 0 && C <= 4 && H > 0 && W > 0 && n_pieces > 0 && n_pieces <= 65535 && max_width > 0 && max_width <= W,
               "mn_postprocess_sr_u8_pieces: bad args");
    const long long total = (long long)H * max_width;
    MN_CUDA_CHECK((mn_launch(postprocess_sr_pieces_kernel, dim3((unsigned)mn_cdiv64(total, 256), n_pieces), dim3(256), 0, (cudaStream_t)stream,
                             sr, stride_n, stride_c, stride_h, stride_w, C, H, pieces, max_width)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_figure_u8(const mn_figure_image* images, int n_images, int max_width, void* stream) {
    MN_REQUIRE(images && n_images > 0 && n_images <= 65535 && max_width > 0, "mn_figure_u8: bad args");
    const long long total = 128ll * max_width;
    MN_CUDA_CHECK((mn_launch(figure_kernel, dim3((unsigned)mn_cdiv64(total, 256), n_images), dim3(256), 0, (cudaStream_t)stream,
                             images, max_width)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_prior_tiles_u8(const float* priors, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                                 const mn_prior_tile* tiles, int n_rows, void* stream) {
    MN_REQUIRE(priors && tiles && n_rows > 0 && n_rows <= 65535, "mn_prior_tiles_u8: bad args");
    MN_CUDA_CHECK((mn_launch(prior_tiles_kernel, dim3(128 * 128 / 256, n_rows), dim3(256), 0, (cudaStream_t)stream, priors, stride_n,
                             stride_c, stride_h, stride_w, tiles)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
