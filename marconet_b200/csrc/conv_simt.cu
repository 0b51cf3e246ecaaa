// fp32 CUDA-core implicit-GEMM convolution (NHWC), the exact-arithmetic path of
// mn_conv2d_nhwc (include/marconet_b200.h).  Replaces F.conv2d / nn.Linear call sites listed
// there.  GEMM view:  M = N*OH*OW pixels, N = Cout, K = KH*KW*Cin (tap-major, channel-minor).
//
// Tile 128 x BN x 16, 256 threads, 8 x (BN/16) register tile per thread, register-staged
// double buffering of shared memory (global loads for k-tile t+1 are in flight while tile t
// is multiplied).  Split-K over blockIdx.z for problems with too few output tiles to fill
// 132 SMs (4x4..16x16 generator layers, the 32768-deep patch embedding).
#include "mn_common.cuh"
#include "conv_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int BK = 16;
constexpr int NTHREADS = 256;

template <int BN, bool VEC_A, bool VEC_B>
__global__ void __launch_bounds__(NTHREADS, 2) conv_igemm_f32_kernel(const ConvGeom g) {
    mn_pdl_prologue();
    constexpr int TN = BN / 16;       // columns per thread (8 or 4)
    constexpr int NS = TN / 4;        // float4 strips per thread along N
    // one buffer: the A / B k-tiles during the K loop, then the staging area of the epilogue (64 rows x BN floats fit exactly)
    __shared__ __align__(16) float smem_buf[2 * BK * BM + 2 * BK * BN];
    float (*As)[BK][BM] = reinterpret_cast<float (*)[BK][BM]>(smem_buf);
    float (*Bs)[BK][BN] = reinterpret_cast<float (*)[BK][BN]>(smem_buf + 2 * BK * BM);
    static_assert(2 * BK * BM + 2 * BK * BN >= 64 * BN, "staging half-tile must fit");

    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int split = blockIdx.z;
    const int kt_begin = split * g.ktiles_per_split;
    const int kt_end = min(g.ktiles, kt_begin + g.ktiles_per_split);

    // ---- A loader state: one output pixel (row of the GEMM) per thread ----
    const int a_row = tid & (BM - 1);
    const int a_kc = (tid >> 7) * 8;
    const int a_m = m0 + a_row;
    const bool a_row_ok = a_m < g.M;
    int a_iy0 = 0, a_ix0 = 0;
    const float* a_base = g.x;
    {
        int mm = a_row_ok ? a_m : 0;
        int n = mm / (g.OH * g.OW);
        int r = mm - n * (g.OH * g.OW);
        int oy = r / g.OW, ox = r - oy * g.OW;
        a_iy0 = oy * g.sh - g.ph;
        a_ix0 = ox * g.sw - g.pw;
        a_base = g.x + (size_t)n * g.H * g.W * g.x_cs;
    }
    // ---- B loader state ----
    const int b_krow = tid >> 4;
    const int b_n = (tid & 15) * TN;

    float a_reg[8];
    float b_reg[TN];

    auto load_tiles = [&](int kt) {
        // A
        if (VEC_A) {
            const int cpt = g.Cin / BK;              // k-tiles per tap
            const int tap = kt / cpt;
            const int c0 = (kt - tap * cpt) * BK + a_kc;
            const int ky = tap / g.KW, kx = tap - ky * g.KW;
            const int iy = a_iy0 + ky, ix = a_ix0 + kx;
            const bool ok = a_row_ok && (unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W;
            if (ok) {
                const float4* p = reinterpret_cast<const float4*>(a_base + ((size_t)iy * g.W + ix) * g.x_cs + c0);
                float4 v0 = __ldg(p), v1 = __ldg(p + 1);
                a_reg[0] = v0.x; a_reg[1] = v0.y; a_reg[2] = v0.z; a_reg[3] = v0.w;
                a_reg[4] = v1.x; a_reg[5] = v1.y; a_reg[6] = v1.z; a_reg[7] = v1.w;
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) a_reg[j] = 0.f;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = kt * BK + a_kc + j;
                float v = 0.f;
                if (a_row_ok && k < g.K) {
                    const int tap = k / g.Cin, c = k - tap * g.Cin;
                    const int ky = tap / g.KW, kx = tap - ky * g.KW;
                    const int iy = a_iy0 + ky, ix = a_ix0 + kx;
                    if ((unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W)
                        v = __ldg(a_base + ((size_t)iy * g.W + ix) * g.x_cs + c);
                }
                a_reg[j] = v;
            }
        }
        // B
        const int k = kt * BK + b_krow;
        if (VEC_B) {
#pragma unroll
            for (int s = 0; s < TN / 4; ++s) {
                const int n = n0 + b_n + s * 4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (k < g.K && n < g.Cout) v = __ldg(reinterpret_cast<const float4*>(g.w + (size_t)k * g.Cout + n));
                b_reg[s * 4 + 0] = v.x; b_reg[s * 4 + 1] = v.y; b_reg[s * 4 + 2] = v.z; b_reg[s * 4 + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < TN; ++j) {
                const int n = n0 + b_n + j;
                b_reg[j] = (k < g.K && n < g.Cout) ? __ldg(g.w + (size_t)k * g.Cout + n) : 0.f;
            }
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int j = 0; j < 8; ++j) As[buf][a_kc + j][a_row] = a_reg[j];
#pragma unroll
        for (int s = 0; s < TN / 4; ++s)
            *reinterpret_cast<float4*>(&Bs[buf][b_krow][b_n + s * 4]) =
                make_float4(b_reg[s * 4], b_reg[s * 4 + 1], b_reg[s * 4 + 2], b_reg[s * 4 + 3]);
    };

    const int ty = tid >> 4, tx = tid & 15;
    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    if (kt_begin < kt_end) {
        load_tiles(kt_begin);
        store_tiles(0);
        __syncthreads();
        int buf = 0;
        for (int kt = kt_begin; kt < kt_end; ++kt) {
            const bool more = kt + 1 < kt_end;
            if (more) load_tiles(kt + 1);
#pragma unroll
            for (int k = 0; k < BK; ++k) {
                float a[8], b[TN];
                float4 t0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
                float4 t1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
                a[0] = t0.x; a[1] = t0.y; a[2] = t0.z; a[3] = t0.w;
                a[4] = t1.x; a[5] = t1.y; a[6] = t1.z; a[7] = t1.w;
#pragma unroll
                for (int s = 0; s < NS; ++s) {
                    float4 u = *reinterpret_cast<const float4*>(&Bs[buf][k][s * (BN / NS) + tx * 4]);
                    b[s * 4] = u.x; b[s * 4 + 1] = u.y; b[s * 4 + 2] = u.z; b[s * 4 + 3] = u.w;
                }
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            if (more) store_tiles(buf ^ 1);
            __syncthreads();
            buf ^= 1;
        }
    }

    // ---- epilogue ----
    // The accumulator tile goes through shared memory in two 64-row halves and ONE rolled loop runs the fused epilogue.  (Round 1
    // called the generic epilogue from the fully unrolled 8 x NS register loop: 7k .. 14k straight-line SASS instructions, each
    // executed once per warp -- the small layers this kernel serves spent their time on instruction-cache misses: 28 .. 70 us for
    // microseconds of arithmetic, ncu source page.)
    const bool vec_ok = (g.Cout & 3) == 0 && (!g.y || ((g.y_cs & 3) == 0 && (reinterpret_cast<uintptr_t>(g.y) & 15) == 0)) &&
                        (!g.y2 || ((g.y2_cs & 3) == 0 && (reinterpret_cast<uintptr_t>(g.y2) & 15) == 0)) &&
                        (!g.residual || ((g.res_cs & 3) == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0)) &&
                        (!g.out_scale || ((g.os_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(g.out_scale) & 15) == 0)) &&
                        (!g.y2_scale || ((g.y2s_stride & 3) == 0 && (reinterpret_cast<uintptr_t>(g.y2_scale) & 15) == 0)) &&
                        (!g.bias || (reinterpret_cast<uintptr_t>(g.bias) & 15) == 0) && (g.splits <= 1 || (reinterpret_cast<uintptr_t>(g.ws) & 15) == 0);
    const int hw = g.OH * g.OW;
    float* stg = smem_buf;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        if (half) __syncthreads();            // the first half has been read (the K loop ends with a barrier of its own)
#pragma unroll
        for (int ii = 0; ii < 4; ++ii)
#pragma unroll
            for (int s = 0; s < NS; ++s)
                *reinterpret_cast<float4*>(&stg[(ty * 4 + ii) * BN + s * (BN / NS) + tx * 4]) =
                    make_float4(acc[half * 4 + ii][s * 4], acc[half * 4 + ii][s * 4 + 1], acc[half * 4 + ii][s * 4 + 2], acc[half * 4 + ii][s * 4 + 3]);
        __syncthreads();
#pragma unroll 1
        for (int idx = tid; idx < 64 * (BN / 4); idx += NTHREADS) {
            const int row = idx / (BN / 4), c4 = idx - row * (BN / 4);
            const int m = m0 + half * 64 + row, o = n0 + c4 * 4;
            if (m >= g.M || o >= g.Cout) continue;
            const float4 u = *reinterpret_cast<const float4*>(&stg[row * BN + c4 * 4]);
            if (g.splits > 1) {
                float* dst = g.ws + ((size_t)split * g.M + m) * g.Cout + o;
                if (vec_ok) *reinterpret_cast<float4*>(dst) = u;
                else { const float v[4] = {u.x, u.y, u.z, u.w}; for (int j = 0; j < 4 && o + j < g.Cout; ++j) dst[j] = v[j]; }
            } else if (vec_ok) {
                const int n = m / hw;
                const bool masked = g.valid_w && (m % g.OW) >= g.valid_w[n];
                conv_epilogue_vec4(g, m, n, masked, o, u, g.bias ? ldg4(g.bias + o) : make_float4(0.f, 0.f, 0.f, 0.f));
            } else {
                float v[4] = {u.x, u.y, u.z, u.w};
                conv_epilogue4(g, m, o, v);
            }
        }
    }
}

__global__ void conv_splitk_reduce_kernel(const ConvGeom g) {
    mn_pdl_prologue();
    const int ngroups = (g.Cout + 3) >> 2;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)g.M * ngroups) return;
    const int m = (int)(idx / ngroups);
    const int o = (int)(idx - (int64_t)m * ngroups) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < g.splits; ++s) {
        const float* src = g.ws + ((size_t)s * g.M + m) * g.Cout + o;
        for (int j = 0; j < 4 && o + j < g.Cout; ++j) v[j] += src[j];
    }
    conv_epilogue4(g, m, o, v);
}

template <int BN>
int launch_simt(const ConvGeom& g, bool vec_a, bool vec_b, cudaStream_t st) {
    dim3 grid(mn_cdiv(g.M, BM), mn_cdiv(g.Cout, BN), g.splits);
    if (vec_a && vec_b) MN_CUDA_CHECK((mn_launch(conv_igemm_f32_kernel<BN, true, true>, dim3(grid), dim3(NTHREADS), 0, st, g)));
    else if (vec_a) MN_CUDA_CHECK((mn_launch(conv_igemm_f32_kernel<BN, true, false>, dim3(grid), dim3(NTHREADS), 0, st, g)));
    else if (vec_b) MN_CUDA_CHECK((mn_launch(conv_igemm_f32_kernel<BN, false, true>, dim3(grid), dim3(NTHREADS), 0, st, g)));
    else MN_CUDA_CHECK((mn_launch(conv_igemm_f32_kernel<BN, false, false>, dim3(grid), dim3(NTHREADS), 0, st, g)));
    MN_LAUNCH_CHECK();
    return MN_OK;
}

}  // namespace

int mn_conv_splitk_reduce_launch(const ConvGeom& g, cudaStream_t st) {
    const int64_t total = (int64_t)g.M * ((g.Cout + 3) / 4);
    MN_CUDA_CHECK((mn_launch(conv_splitk_reduce_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, st, g)));
    return MN_OK;
}

int mn_conv_simt_plan_splits(const ConvGeom& g0, int64_t ws_bytes, int requested) {
    const int bn = g0.Cout > 64 ? 128 : 64;
    const int tiles = mn_cdiv(g0.M, BM) * mn_cdiv(g0.Cout, bn);
    const int ktiles = mn_cdiv(g0.K, BK);
    int splits = 1;
    if (requested > 1) splits = requested;
    else if (requested == 0) {
        const int sms = mn_num_sms();
        if (tiles < sms && ktiles >= 16) {
            splits = mn_cdiv(2 * sms, tiles);
            if (splits > ktiles / 4) splits = ktiles / 4;
            if (splits > 64) splits = 64;
            if (splits < 1) splits = 1;
        }
    }
    if (splits > ktiles) splits = ktiles;
    if (splits > 1) {
        const int64_t per = (int64_t)g0.M * g0.Cout * 4;
        if (ws_bytes < per * 2) return 1;
        if (per * splits > ws_bytes) splits = (int)(ws_bytes / per);
    }
    if (splits < 1) splits = 1;
    // the count mn_conv_simt_launch runs: whole k-tiles per split, no empty split at the end
    return mn_cdiv(ktiles, mn_cdiv(ktiles, splits));
}

int mn_conv_simt_launch(ConvGeom g, cudaStream_t st) {
    g.ktiles = mn_cdiv(g.K, BK);
    g.ktiles_per_split = mn_cdiv(g.ktiles, g.splits);
    g.splits = mn_cdiv(g.ktiles, g.ktiles_per_split);
    const bool vec_a = (g.Cin % BK == 0) && (g.x_cs % 4 == 0) && ((reinterpret_cast<uintptr_t>(g.x) & 15) == 0);
    const bool vec_b = (g.Cout % 4 == 0) && ((reinterpret_cast<uintptr_t>(g.w) & 15) == 0);
    int rc = (g.Cout > 64) ? launch_simt<128>(g, vec_a, vec_b, st) : launch_simt<64>(g, vec_a, vec_b, st);
    if (rc != MN_OK) return rc;
    if (g.splits > 1) {
        const int64_t total = (int64_t)g.M * ((g.Cout + 3) / 4);
        MN_CUDA_CHECK((mn_launch(conv_splitk_reduce_kernel, dim3((unsigned)mn_cdiv64(total, 256)), dim3(256), 0, st, g)));
        MN_LAUNCH_CHECK();
    }
    return MN_OK;
}
