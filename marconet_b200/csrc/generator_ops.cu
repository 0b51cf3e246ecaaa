// TSPGAN (StyleGAN-like structure-prior generator) helper operators.  HBM-bound elementwise /
// reduction kernels; see include/marconet_b200.h for the reference call sites they replace.
#include "mn_common.cuh"

namespace {

// ---------------------------------------------------------------- PixelNorm (networks.py:170-171)
__global__ void pixelnorm_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C) {
    mn_pdl_prologue();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= N) return;
    const float* xr = x + (size_t)row * C;
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) ss = fmaf(xr[c], xr[c], ss);
    ss = mn_warp_sum(ss);
    const float r = rsqrtf(ss / (float)C + 1e-8f);
    for (int c = lane; c < C; c += 32) y[(size_t)row * C + c] = xr[c] * r;
}

// ---------------------------------------------------------------- SelectText (networks.py:205-215)
__global__ void select_text_kernel(const float* __restrict__ emb, const int64_t* __restrict__ labels,
                                   const float* __restrict__ s, int s_stride, float* __restrict__ out,
                                   int N, int L, int C) {
    mn_pdl_prologue();
    // out: [N, 4, 4*L, C]; one thread per 4 channels of one output pixel
    const int c4 = C >> 2;
    const int64_t total = (int64_t)N * 16 * L * c4;
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;     // host guarantees total < 2^31: 32-bit div/mod only
    if (idx >= (uint32_t)total) return;
    const int c = (int)(idx % c4) * 4;
    uint32_t pix = idx / c4;
    const int xw = (int)(pix % (4 * L));
    pix /= (4 * L);
    const int n = (int)(pix / 4);
    const int l = xw >> 2;
    const int64_t lab = labels[(size_t)n * L + l];
    float4 e = *reinterpret_cast<const float4*>(emb + (size_t)lab * C + c);
    if (s) {
        const float* sn = s + (size_t)n * s_stride + c;
        e.x *= sn[0]; e.y *= sn[1]; e.z *= sn[2]; e.w *= sn[3];
    }
    *reinterpret_cast<float4*>(out + (size_t)idx * 4) = e;
}

// ---------------------------------------------------------------- demodulation (networks.py:284-287)
__global__ void demod_kernel(const float* __restrict__ s, int s_stride, const float* __restrict__ wsq,
                             float* __restrict__ demod, int N, int Cin, int Cout) {
    mn_pdl_prologue();
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = blockIdx.y;
    if (o >= Cout) return;
    const float* sn = s + (size_t)n * s_stride;
    float acc = 0.f;
    for (int c = 0; c < Cin; ++c) {
        const float sv = sn[c];
        acc = fmaf(sv * sv, wsq[(size_t)c * Cout + o], acc);
    }
    demod[(size_t)n * Cout + o] = rsqrtf(acc + 1e-8f);
}

// All demodulation tables of a generator pass in ONE launch: grid (cout tiles, N, layers), 64 columns x 4 k-slices.
__global__ void __launch_bounds__(256) demod_batched_kernel(const float* __restrict__ s_all, int s_stride, const mn_demod_desc* __restrict__ descs,
                                                            float* __restrict__ out_all, int out_stride) {
    mn_pdl_prologue();
    const mn_demod_desc d = descs[blockIdx.z];
    const int col = threadIdx.x & 63, ks = threadIdx.x >> 6;
    const int o = blockIdx.x * 64 + col;
    const int n = blockIdx.y;
    __shared__ float red[4][64];
    float acc = 0.f;
    if (o < d.cout) {
        const float* sn = s_all + (size_t)n * s_stride + d.s_off;
        const float* w = d.wsq + o;
#pragma unroll 4
        for (int c = ks; c < d.cin; c += 4) {
            const float sv = sn[c];
            acc = fmaf(sv * sv, w[(size_t)c * d.cout], acc);
        }
    }
    red[ks][col] = acc;
    __syncthreads();
    if (ks == 0 && o < d.cout)
        out_all[(size_t)n * out_stride + d.out_off + o] = rsqrtf((red[0][col] + red[1][col]) + (red[2][col] + red[3][col]) + 1e-8f);
}

// ---------------------------------------------------------------- bilinear x2 (+ per-sample channel scale)
// PyTorch upsample_bilinear2d, align_corners=False, scale 2: src = 0.5*(dst+0.5)-0.5 clamped at 0.
__device__ __forceinline__ void bilin_coords(int o, int size, int& i0, int& i1, float& l1) {
    float src = 0.5f * ((float)o + 0.5f) - 0.5f;
    src = src < 0.f ? 0.f : src;
    i0 = (int)src;
    i1 = i0 + (i0 < size - 1 ? 1 : 0);
    l1 = src - (float)i0;
}

__global__ void resample_modulate_kernel(const float* __restrict__ x, int x_cs, float* __restrict__ y, int y_cs,
                                         const float* __restrict__ s, int s_stride,
                                         int N, int H, int W, int C, int up) {
    mn_pdl_prologue();
    const int OH = up ? 2 * H : H, OW = up ? 2 * W : W;
    const int c4 = C >> 2;
    const int64_t total = (int64_t)N * OH * OW * c4;
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;     // host guarantees total < 2^31: 32-bit div/mod only
    if (idx >= (uint32_t)total) return;
    const int c = (int)(idx % c4) * 4;
    uint32_t pix = idx / c4;
    const int ox = (int)(pix % OW);
    pix /= OW;
    const int oy = (int)(pix % OH);
    const int n = (int)(pix / OH);
    const float* xn = x + (size_t)n * H * W * x_cs + c;
    float4 v;
    if (up) {
        int y0, y1, x0, x1; float ly, lx;
        bilin_coords(oy, H, y0, y1, ly);
        bilin_coords(ox, W, x0, x1, lx);
        const float hy = 1.f - ly, hx = 1.f - lx;
        const float4 a = *reinterpret_cast<const float4*>(xn + ((size_t)y0 * W + x0) * x_cs);
        const float4 b = *reinterpret_cast<const float4*>(xn + ((size_t)y0 * W + x1) * x_cs);
        const float4 cc = *reinterpret_cast<const float4*>(xn + ((size_t)y1 * W + x0) * x_cs);
        const float4 d = *reinterpret_cast<const float4*>(xn + ((size_t)y1 * W + x1) * x_cs);
        v.x = hy * (hx * a.x + lx * b.x) + ly * (hx * cc.x + lx * d.x);
        v.y = hy * (hx * a.y + lx * b.y) + ly * (hx * cc.y + lx * d.y);
        v.z = hy * (hx * a.z + lx * b.z) + ly * (hx * cc.z + lx * d.z);
        v.w = hy * (hx * a.w + lx * b.w) + ly * (hx * cc.w + lx * d.w);
    } else {
        v = *reinterpret_cast<const float4*>(xn + ((size_t)oy * W + ox) * x_cs);
    }
    if (s) {
        const float* sn = s + (size_t)n * s_stride + c;
        v.x *= sn[0]; v.y *= sn[1]; v.z *= sn[2]; v.w *= sn[3];
    }
    *reinterpret_cast<float4*>(y + (((size_t)n * OH + oy) * OW + ox) * y_cs + c) = v;
}


// Bilinear x2 specialisation.  One thread owns 4 channels of UP_RX consecutive input pixels of one input row and slides a
// 3x3 register window along the row: 3 new 128-bit loads (rows iy-1, iy, iy+1 of the next column, prefetched one column
// ahead) per 2x2 block of outputs, i.e. 0.75 loads per output instead of the generic kernel's 4 -- that kernel is bound by
// L1/L2 -> SM traffic (2.3 TB/s of HBM traffic where a 1-read : 4-write stream reaches 5.8 TB/s, tools/hbm_probe.cu).
// Coordinates, weights and the formula are resample_modulate_kernel's: hy*(hx*a + lx*b) + ly*(hx*c + lx*d).
constexpr int UP_RX = 4;
__device__ __forceinline__ float4 up_hblend(const float4& a, const float4& b, float hx, float lx) {
    return make_float4(hx * a.x + lx * b.x, hx * a.y + lx * b.y, hx * a.z + lx * b.z, hx * a.w + lx * b.w);
}
// RAGGED: sample n is the first valid_w[n] columns of its row (row pitch stays W): the source column clamps at valid_w[n]-1, the
// edge of that line's own tensor in the reference, and output columns >= 2*valid_w[n] are written as 0.  Each sample is then
// bit-identical to the non-ragged instantiation run on that sample alone at width valid_w[n].
template <bool RAGGED>
__global__ void __launch_bounds__(256) resample_up2_kernel(const float* __restrict__ x, int x_cs, float* __restrict__ y, int y_cs,
                                                           const float* __restrict__ s, int s_stride, int N, int H, int W_pitch, int C,
                                                           const int32_t* __restrict__ valid_w) {
    mn_pdl_prologue();
    const int c4 = C >> 2;
    const int runs = (W_pitch + UP_RX - 1) / UP_RX;
    const uint32_t total = (uint32_t)N * H * runs * c4;              // host guarantees the output (16x more) fits 31 bits
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % c4) * 4;
    uint32_t t = idx / c4;
    const int xs = (int)(t % runs) * UP_RX;
    t /= runs;
    const int iy = (int)(t % H);
    const int n = (int)(t / H);
    const int W = RAGGED ? min(valid_w[n], W_pitch) : W_pitch;       // clamp bound: the sample's own width
    const int OH = 2 * H, OW = 2 * W_pitch;
    float* y0p = y + ((size_t)n * OH + 2 * iy) * OW * y_cs + c;
    float* y1p = y0p + (size_t)OW * y_cs;
    if (RAGGED) {                                  // columns of this run beyond the sample's width: zeros
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        const int xe = min(xs + UP_RX, W_pitch);
        for (int ix = max(xs, W); ix < xe; ++ix)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                *reinterpret_cast<float4*>(y0p + (size_t)(2 * ix + dx) * y_cs) = z;
                *reinterpret_cast<float4*>(y1p + (size_t)(2 * ix + dx) * y_cs) = z;
            }
        if (xs >= W) return;
    }
    const float* xn = x + (size_t)n * H * W_pitch * x_cs + c;
    const float* row[3] = {xn + (size_t)(iy > 0 ? iy - 1 : 0) * W_pitch * x_cs, xn + (size_t)iy * W_pitch * x_cs,
                           xn + (size_t)(iy < H - 1 ? iy + 1 : iy) * W_pitch * x_cs};
    float4 sv = make_float4(1.f, 1.f, 1.f, 1.f);
    if (s) sv = *reinterpret_cast<const float4*>(s + (size_t)n * s_stride + c);
    // vertical taps of the two output rows (2iy, 2iy+1): which of {row above, this row, row below} and with what weight
    int ya0, ya1, yb0, yb1; float lya, lyb;
    bilin_coords(2 * iy, H, ya0, ya1, lya);
    bilin_coords(2 * iy + 1, H, yb0, yb1, lyb);
    const bool top = iy == 0;                      // even output row of the first input row: taps (row 0, row 1) with weight 0 on row 1
    const float hya = 1.f - lya, hyb = 1.f - lyb;

    float4 L[3], M[3], R[3], Nx[3];
    const int xl = xs > 0 ? xs - 1 : 0, xr = xs + 1 < W ? xs + 1 : W - 1;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        L[r] = *reinterpret_cast<const float4*>(row[r] + (size_t)xl * x_cs);
        M[r] = *reinterpret_cast<const float4*>(row[r] + (size_t)xs * x_cs);
        R[r] = *reinterpret_cast<const float4*>(row[r] + (size_t)xr * x_cs);
    }
#pragma unroll
    for (int j = 0; j < UP_RX; ++j) {
        const int ix = xs + j;
        if (ix >= W) break;
        if (j + 1 < UP_RX && ix + 1 < W) {         // prefetch the column after next before this column's arithmetic
            const int xn2 = ix + 2 < W ? ix + 2 : W - 1;
#pragma unroll
            for (int r = 0; r < 3; ++r) Nx[r] = *reinterpret_cast<const float4*>(row[r] + (size_t)xn2 * x_cs);
        }
        int xa0, xa1, xb0, xb1; float lxa, lxb;
        bilin_coords(2 * ix, W, xa0, xa1, lxa);     // even output column: taps (ix-1, ix), or (0, 1) with weight 0 at the left edge
        bilin_coords(2 * ix + 1, W, xb0, xb1, lxb); // odd output column: taps (ix, ix+1 clamped)
        const float hxa = 1.f - lxa, hxb = 1.f - lxb;
        const bool left = ix == 0;
        float4 he[3], ho[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            he[r] = left ? up_hblend(M[r], R[r], hxa, lxa) : up_hblend(L[r], M[r], hxa, lxa);
            ho[r] = up_hblend(M[r], R[r], hxb, lxb);
        }
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const float4* h = dx ? ho : he;
            const float4 a0 = top ? h[1] : h[0], a1 = top ? h[2] : h[1];       // even output row
            float4 o0 = make_float4(hya * a0.x + lya * a1.x, hya * a0.y + lya * a1.y, hya * a0.z + lya * a1.z, hya * a0.w + lya * a1.w);
            float4 o1 = make_float4(hyb * h[1].x + lyb * h[2].x, hyb * h[1].y + lyb * h[2].y, hyb * h[1].z + lyb * h[2].z,
                                    hyb * h[1].w + lyb * h[2].w);                 // odd output row: taps (iy, iy+1 clamped)
            if (s) {
                o0.x *= sv.x; o0.y *= sv.y; o0.z *= sv.z; o0.w *= sv.w;
                o1.x *= sv.x; o1.y *= sv.y; o1.z *= sv.z; o1.w *= sv.w;
            }
            *reinterpret_cast<float4*>(y0p + (size_t)(2 * ix + dx) * y_cs) = o0;
            *reinterpret_cast<float4*>(y1p + (size_t)(2 * ix + dx) * y_cs) = o1;
        }
#pragma unroll
        for (int r = 0; r < 3; ++r) { L[r] = M[r]; M[r] = R[r]; R[r] = Nx[r]; }
    }
}

// ---------------------------------------------------------------- ToRGB (networks.py:313-321)
// One warp walks pixels of one sample; the modulated 1x1 weights (3 x C) live in registers.
template <int CPL /* channels per lane = C/32 */>
__global__ void torgb_kernel(const float* __restrict__ x, int x_cs, const float* __restrict__ s, int s_stride,
                             const float* __restrict__ w, const float* __restrict__ bias,
                             const float* __restrict__ skip, float* __restrict__ out,
                             int N, int H, int W, int C) {
    mn_pdl_prologue();
    const int n = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int warp = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    // lane owns channels { q*128 + lane*4 + j }  (q < CPL/4)
    float wm[3][CPL];
#pragma unroll
    for (int q = 0; q < CPL / 4; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = q * 128 + lane * 4 + j;
            const float sv = s[(size_t)n * s_stride + c];
#pragma unroll
            for (int o = 0; o < 3; ++o) wm[o][q * 4 + j] = w[(size_t)o * C + c] * sv;
        }
    const int HW = H * W;
    const float* xn = x + (size_t)n * HW * x_cs;
    // TP pixels per trip: all loads of the trip are issued before the first FMA (memory-level parallelism; one pixel is only
    // C*4 bytes per warp), then 3 warp reductions per pixel.
    constexpr int TP = (CPL <= 4) ? 4 : 2;
    for (int p0 = warp * TP; p0 < HW; p0 += nwarps * TP) {
        float4 v[TP][CPL / 4];
#pragma unroll
        for (int t = 0; t < TP; ++t)
#pragma unroll
            for (int q = 0; q < CPL / 4; ++q)
                v[t][q] = (p0 + t < HW) ? *reinterpret_cast<const float4*>(xn + (size_t)(p0 + t) * x_cs + q * 128 + lane * 4)
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int t = 0; t < TP; ++t) {
            const int p = p0 + t;
            if (p >= HW) break;
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int q = 0; q < CPL / 4; ++q) {
                const float4 u = v[t][q];
                a0 = fmaf(u.x, wm[0][q * 4], a0); a0 = fmaf(u.y, wm[0][q * 4 + 1], a0);
                a0 = fmaf(u.z, wm[0][q * 4 + 2], a0); a0 = fmaf(u.w, wm[0][q * 4 + 3], a0);
                a1 = fmaf(u.x, wm[1][q * 4], a1); a1 = fmaf(u.y, wm[1][q * 4 + 1], a1);
                a1 = fmaf(u.z, wm[1][q * 4 + 2], a1); a1 = fmaf(u.w, wm[1][q * 4 + 3], a1);
                a2 = fmaf(u.x, wm[2][q * 4], a2); a2 = fmaf(u.y, wm[2][q * 4 + 1], a2);
                a2 = fmaf(u.z, wm[2][q * 4 + 2], a2); a2 = fmaf(u.w, wm[2][q * 4 + 3], a2);
            }
            a0 = mn_warp_sum(a0); a1 = mn_warp_sum(a1); a2 = mn_warp_sum(a2);
            if (lane < 3) {
                float r = lane == 0 ? a0 : (lane == 1 ? a1 : a2);
                r += bias[lane];
                if (skip) {
                    const int oy = p / W, ox = p - oy * W;
                    const int h2 = H >> 1, w2 = W >> 1;
                    int y0, y1, x0, x1; float ly, lx;
                    bilin_coords(oy, h2, y0, y1, ly);
                    bilin_coords(ox, w2, x0, x1, lx);
                    const float hy = 1.f - ly, hx = 1.f - lx;
                    const float* sk = skip + (size_t)n * h2 * w2 * 3 + lane;
                    const float a = sk[((size_t)y0 * w2 + x0) * 3], b = sk[((size_t)y0 * w2 + x1) * 3];
                    const float c = sk[((size_t)y1 * w2 + x0) * 3], d = sk[((size_t)y1 * w2 + x1) * 3];
                    r += hy * (hx * a + lx * b) + ly * (hx * c + lx * d);
                }
                out[((size_t)n * HW + p) * 3 + lane] = tanhf(r);
            }
        }
    }
}

// ---------------------------------------------------------------- label range check without a host round trip
// The reference indexes TextEmbeddings with the label (networks.py:211); an out-of-range label is an error there.
// For graph capture / pipelined callers the check runs on the device: bit 0 of *err is raised and the label is
// clamped so that the lookup stays in bounds.
__global__ void check_labels_kernel(const int64_t* __restrict__ labels, int64_t* __restrict__ clamped, int n, int classes,
                                    int32_t* __restrict__ err) {
    mn_pdl_prologue();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int64_t l = labels[i];
    if (l < 0 || l >= classes) { atomicOr(err, 1); l = l < 0 ? 0 : classes - 1; }
    clamped[i] = l;
}

// ---------------------------------------------------------------- font-style interpolation (test_w.py:107)
// One thread per (style row, 4 dims): new_w = w1*s + w2*t with each multiply and the add rounded on its own, as torch computes
// ``w1 * scale + w2 * (1 - scale)`` on fp32 tensors (explicit-rounding intrinsics: nvcc must not contract into an FMA).
__global__ void style_lerp_kernel(const float* __restrict__ w, int w_stride, const mn_lerp_row* __restrict__ rows, int n_rows,
                                  int dim, float* __restrict__ out, int out_stride) {
    mn_pdl_prologue();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int r = (int)(i / dim), d = (int)(i % dim);
    if (r >= n_rows) return;
    const mn_lerp_row row = rows[r];
    out[(long long)r * out_stride + d] = __fadd_rn(__fmul_rn(w[(long long)row.w1 * w_stride + d], row.s),
                                                   __fmul_rn(w[(long long)row.w2 * w_stride + d], row.t));
}

}  // namespace

extern "C" int mn_pixelnorm(const float* x, float* y, int N, int C, void* stream) {
    MN_REQUIRE(x && y && N > 0 && C > 0, "mn_pixelnorm: bad args");
    MN_CUDA_CHECK((mn_launch(pixelnorm_kernel, dim3(mn_cdiv(N, 4)), dim3(128), 0, (cudaStream_t)stream, x, y, N, C)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_select_text(const float* emb, const int64_t* labels, const float* s, int s_stride,
                              float* out, int N, int L, int C, void* stream) {
    MN_REQUIRE(emb && labels && out && N > 0 && L > 0 && C > 0 && (C & 3) == 0, "mn_select_text: bad args");
    const int64_t total = (int64_t)N * 16 * L * (C >> 2);
    MN_REQUIRE(total < (1ll << 31), "tensor too large for 32-bit indexing");
    MN_CUDA_CHECK((mn_launch(select_text_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, (cudaStream_t)stream, emb, labels, s, s_stride, out, N, L, C)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_demod(const float* s, int s_stride, const float* wsq, float* demod, int N, int Cin, int Cout, void* stream) {
    MN_REQUIRE(s && wsq && demod && N > 0 && Cin > 0 && Cout > 0, "mn_demod: bad args");
    dim3 grid(mn_cdiv(Cout, 128), N);
    MN_CUDA_CHECK((mn_launch(demod_kernel, dim3(grid), dim3(128), 0, (cudaStream_t)stream, s, s_stride, wsq, demod, N, Cin, Cout)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_resample_modulate(const float* x, int x_cs, float* y, int y_cs, const float* s, int s_stride,
                                    int N, int H, int W, int C, int up, void* stream) {
    MN_REQUIRE(x && y && N > 0 && H > 0 && W > 0 && C > 0, "mn_resample_modulate: bad args");
    MN_REQUIRE((C & 3) == 0 && (x_cs & 3) == 0 && (y_cs & 3) == 0, "mn_resample_modulate: channels must be multiples of 4");
    MN_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 15) == 0, "mn_resample_modulate: pointers must be 16B aligned");
    const int OH = up ? 2 * H : H, OW = up ? 2 * W : W;
    const int64_t total = (int64_t)N * OH * OW * (C >> 2);
    MN_REQUIRE(total < (1ll << 31), "tensor too large for 32-bit indexing");
    if (up && (!s || ((s_stride & 3) == 0 && ((uintptr_t)s & 15) == 0))) {
        MN_CUDA_CHECK((mn_launch(resample_up2_kernel<false>, dim3((unsigned)mn_cdiv64((int64_t)N * H * mn_cdiv(W, UP_RX) * (C >> 2), 256)), dim3(256), 0, (cudaStream_t)stream, x, x_cs, y, y_cs, s, s_stride, N, H, W, C,
                                 (const int32_t*)nullptr)));
        MN_LAUNCH_CHECK();
        return MN_OK;
    }
    MN_CUDA_CHECK((mn_launch(resample_modulate_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, (cudaStream_t)stream, x, x_cs, y, y_cs, s, s_stride, N, H, W, C, up)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_resample_modulate_ragged(const float* x, int x_cs, float* y, int y_cs, const float* s, int s_stride,
                                           const int32_t* valid_w, int N, int H, int W, int C, void* stream) {
    MN_REQUIRE(x && y && valid_w && N > 0 && H > 0 && W > 0 && C > 0, "mn_resample_modulate_ragged: bad args");
    MN_REQUIRE((C & 3) == 0 && (x_cs & 3) == 0 && (y_cs & 3) == 0, "mn_resample_modulate_ragged: channels must be multiples of 4");
    MN_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)y & 15) == 0 && (!s || ((s_stride & 3) == 0 && ((uintptr_t)s & 15) == 0)),
               "mn_resample_modulate_ragged: x, y and s must be 16B aligned (s_stride a multiple of 4)");
    const int64_t total = (int64_t)N * 2 * H * 2 * W * (C >> 2);
    MN_REQUIRE(total < (1ll << 31), "tensor too large for 32-bit indexing");
    MN_CUDA_CHECK((mn_launch(resample_up2_kernel<true>, dim3((unsigned)mn_cdiv64((int64_t)N * H * mn_cdiv(W, UP_RX) * (C >> 2), 256)), dim3(256), 0,
                             (cudaStream_t)stream, x, x_cs, y, y_cs, s, s_stride, N, H, W, C, valid_w)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_torgb(const float* x, int x_cs, const float* s, int s_stride, const float* w, const float* bias,
                        const float* skip, float* out, int N, int H, int W, int C, void* stream) {
    MN_REQUIRE(x && s && w && bias && out && N > 0 && H > 0 && W > 0, "mn_torgb: bad args");
    MN_REQUIRE(C % 128 == 0 && C <= 512 && (x_cs & 3) == 0 && ((uintptr_t)x & 15) == 0, "mn_torgb: C must be 128/256/384/512, 16B aligned");
    MN_REQUIRE(!skip || ((H & 1) == 0 && (W & 1) == 0), "mn_torgb: skip needs even H, W");
    const int HW = H * W;
    int blocks = mn_cdiv(HW, 8 * 4);           // 8 warps per block, >= 4 pixels per warp
    const int cap = mn_cdiv(mn_num_sms() * 8, N);
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    dim3 grid(blocks, N);
    cudaStream_t st = (cudaStream_t)stream;
    switch (C / 32) {
        case 4: MN_CUDA_CHECK((mn_launch(torgb_kernel<4>, dim3(grid), dim3(256), 0, st, x, x_cs, s, s_stride, w, bias, skip, out, N, H, W, C))); break;
        case 8: MN_CUDA_CHECK((mn_launch(torgb_kernel<8>, dim3(grid), dim3(256), 0, st, x, x_cs, s, s_stride, w, bias, skip, out, N, H, W, C))); break;
        case 12: MN_CUDA_CHECK((mn_launch(torgb_kernel<12>, dim3(grid), dim3(256), 0, st, x, x_cs, s, s_stride, w, bias, skip, out, N, H, W, C))); break;
        case 16: MN_CUDA_CHECK((mn_launch(torgb_kernel<16>, dim3(grid), dim3(256), 0, st, x, x_cs, s, s_stride, w, bias, skip, out, N, H, W, C))); break;
        default: mn_set_error("mn_torgb: unsupported C=%d", C); return MN_ERR_UNSUPPORTED;
    }
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_demod_batched(const float* s_all, int s_stride, const mn_demod_desc* descs, int n_layers, int max_cout,
                                float* out_all, int out_stride, int N, void* stream) {
    MN_REQUIRE(s_all && descs && out_all && n_layers > 0 && max_cout > 0 && N > 0, "mn_demod_batched: bad args");
    MN_CUDA_CHECK((mn_launch(demod_batched_kernel, dim3(dim3(mn_cdiv(max_cout, 64), N, n_layers)), dim3(256), 0, (cudaStream_t)stream, s_all, s_stride, descs, out_all, out_stride)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_check_labels(const int64_t* labels, int64_t* clamped, int n, int classes, int32_t* err, void* stream) {
    MN_REQUIRE(labels && clamped && err && n > 0 && classes > 0, "mn_check_labels: bad args");
    MN_CUDA_CHECK((mn_launch(check_labels_kernel, dim3(mn_cdiv(n, 128)), dim3(128), 0, (cudaStream_t)stream, labels, clamped, n, classes, err)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

extern "C" int mn_style_lerp(const float* w, int w_stride, const mn_lerp_row* rows, int n_rows, int dim, float* out, int out_stride,
                             void* stream) {
    MN_REQUIRE(w && rows && out && n_rows > 0 && dim > 0 && w_stride >= dim && out_stride >= dim, "mn_style_lerp: bad args");
    const long long total = (long long)n_rows * dim;
    MN_CUDA_CHECK((mn_launch(style_lerp_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, (cudaStream_t)stream, w, w_stride,
                             rows, n_rows, dim, out, out_stride)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}
