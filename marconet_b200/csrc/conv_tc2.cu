// conv_tc2.cu -- wgmma operand-split implicit-GEMM convolution for sm_90a, the tensor-core path of mn_conv2d_nhwc.
// x*w ~= xh*wh + (xh*wl + xl*wh) with 16-bit halves (three MMAs, cross terms in their own fp32 accumulator: the tensor core
// truncates when it adds into fp32, see the epilogue's dfix).  One work item = 128 pixels x NT channels (x one k-slice), NT = 64
// or 128 chosen per layer by the plan.
// HALO: one TMA box per 64-channel block brings the zero-padded (TH+2) x (TW+2) halo; the taps are shifted reads of it (shapes
// whose halo does not fit take one shifted 128-pixel box per tap: mn_conv_tc_*).  SPLIT: a warpgroup turns it into hi / lo planes
// in place (fused GroupNorm(+swish) here).  MMA: two consumer warpgroups ldmatrix the shifted rows into the register A fragments
// of wgmma.m64n{NT}k16, B = the 128B-swizzled weight tile, TMA-multicast to a 2-CTA cluster; a weight / A stage is released once
// per warpgroup.  Persistent CTAs; epilogue staged through shared memory in 64-column halves.  Warpgroups (setmaxnreg moves registers to the consumers): 0 split, 1 producers (warp 4 weights,
// warp 5 A tiles), 2 / 3 consumers (rows 0-63 / 64-127).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "conv_common.cuh"
#include "mn_common.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace tcptx;

constexpr int KB = 64;                          // channels per k-block
constexpr int NUM_THREADS2 = 512;               // 4 warpgroups: see the role list in the header comment
// registers per thread of each role after setmaxnreg (4 x 128 threads x 128 at launch = 128 x (SPLIT + PROD + 2 CONS))
constexpr int REG_SPLIT = 88, REG_PROD = 24, REG_CONS = 200;
static_assert(REG_SPLIT + REG_PROD + 2 * REG_CONS <= 4 * 128, "register budget");
constexpr int MAX_HS = 3;
constexpr int MAX_BSTAGES = 4;
__host__ __device__ constexpr int b_half(int nt) { return nt * 128; }   // one (hi or lo) weight tile: nt channels x 64 k x 2 B
__host__ __device__ constexpr int b_stage(int nt) { return 2 * b_half(nt); }
constexpr int STG_PITCH = 72;                   // floats per staged row (64 columns): conflict-free float2 stores of the accumulators
constexpr int STG_BYTES = 128 * STG_PITCH * 4;
constexpr int SMEM_LIMIT = 232448;              // 227 KB

template <int A> struct ActTag { static constexpr int value = A; };

// One thread's share of the epilogue GroupNorm statistics (sum and sum of squares of y per sample and group).  Summing y and y*y
// directly in fp32 loses the variance to cancellation when |mean| >> std (E[y^2] - mean^2: ~1e-3 relative at mean/std = 300):
// the values are summed about a pivot (the thread's first value) in fp32 and turned into sum / sum of squares in fp64, where
// the finaliser's E[y^2] - mean^2 has 29 more bits to cancel.
struct GnAcc {
    float p = 0.f, s = 0.f, q = 0.f;
    int c = 0;
    __device__ __forceinline__ void add(const float4 w) {
        if (c == 0) p = w.x;
        const float d0 = w.x - p, d1 = w.y - p, d2 = w.z - p, d3 = w.w - p;
        s += (d0 + d1) + (d2 + d3);
        q = fmaf(d0, d0, fmaf(d1, d1, fmaf(d2, d2, fmaf(d3, d3, q))));
        c += 4;
    }
    // sum y = c p + s ;  sum y^2 = q + 2 p s + c p^2
    __device__ __forceinline__ void sums(double& sum, double& sq) const {
        const double pd = p, cd = c;
        sum = cd * pd + s;
        sq = (double)q + 2.0 * pd * s + cd * pd * pd;
    }
};

// MODE: 0 = f16x3, 1 = bf16x3, 2 = f16x1 (a template parameter: the wgmma operand registers must not depend on a runtime branch)
template <bool GN, int MODE, int NT>
__global__ void __launch_bounds__(NUM_THREADS2, 1)
conv_tc2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
                const __grid_constant__ CUtensorMap tmBlo, const ConvGeom g, const Tc2Geom t) {
    constexpr int B_HALF = b_half(NT), B_STAGE = b_stage(NT);
    extern __shared__ uint8_t smem_raw[];
    // keep the pointer in the shared address space (offset arithmetic on the array) so loads compile to LDS, not generic LD
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t smem_base = smem_u32(smem);
    const int HS = t.hstages;
    const uint32_t off_b = HS * t.halo_stage_bytes;
    const uint32_t off_stg = off_b + t.bstages * B_STAGE;
    const uint32_t off_rowm = off_stg + STG_BYTES;
    const uint32_t off_bars = off_rowm + 1024;
    float* stg = reinterpret_cast<float*>(smem + off_stg);
    int* rowm = reinterpret_cast<int*>(smem + off_rowm);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + off_bars);
    constexpr int I_HF = 0, I_HE = MAX_HS, I_SD = 2 * MAX_HS, I_BF = 3 * MAX_HS, I_BE = I_BF + MAX_BSTAGES;
    auto bar = [&](int i) { return smem_u32(bars + i); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cs = t.cs;
    const uint32_t crank = cs > 1 ? cluster_ctarank() : 0u;
    const uint16_t cmask = (uint16_t)((1u << cs) - 1u);
    const int num_clusters = gridDim.x / cs;
    // first work item of this CTA's cluster; read inside each role, after its setmaxnreg, so that no register value has to live
    // across the register reallocation (ptxas spills such values)
    auto first_work = [&]() { return (int)(blockIdx.x / cs); };
    const int total_work = t.m_groups * t.n_tiles * t.ksplit;
    const int BS = t.bstages;
    const int units = t.per_tap ? t.cbps * t.taps : t.cbps;      // A tiles per work item
    const int unit_taps = t.per_tap ? 1 : t.taps;                 // k-blocks per A tile
    // work item -> (k-slice, channel tile, pixel-tile group); identical in every warp role
    auto work_ks = [&](int work) { return work % t.ksplit; };
    auto work_nt = [&](int work) { return (work / t.ksplit) % t.n_tiles; };
    auto work_mg = [&](int work) { return work / (t.ksplit * t.n_tiles); };

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBhi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBlo) : "memory");
        for (int s = 0; s < MAX_HS; ++s) { mbar_init(bar(I_HF + s), 1); mbar_init(bar(I_HE + s), 2); mbar_init(bar(I_SD + s), 128); }
        // B stage s of every CTA of the cluster is written by every CTA's multicast: one arrival per consumer warpgroup of each CTA
        for (int s = 0; s < MAX_BSTAGES; ++s) { mbar_init(bar(I_BF + s), 1); mbar_init(bar(I_BE + s), 2 * cs); }
        fence_barrier_init();
    }
    __syncthreads();
    if (cs > 1) cluster_sync_all();
    // Programmatic dependent launch: everything above may overlap the tail of the previous kernel in the stream; from here on we
    // read its results, so wait for it to complete and flush.  Let our own dependents start their prologue as soon as SMs free up.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    auto tile_origin = [&](int work, int& n0, int& oy0, int& ox0) {
        int m_tile = work_mg(work) * cs + (int)crank;
        if (m_tile >= t.m_tiles) { n0 = g.N + 1024; oy0 = 0; ox0 = 0; return; }   // padding CTA of a cluster: everything out of bounds
        const int tw_i = m_tile % t.tiles_w; m_tile /= t.tiles_w;
        const int th_i = m_tile % t.tiles_h; m_tile /= t.tiles_h;
        n0 = m_tile * t.TN; oy0 = th_i * t.TH; ox0 = tw_i * t.TW;
    };

    if (warp >= 4 && warp < 8) {
        setmaxnreg_dec<REG_PROD>();
        if (warp == 4) {
            // =========================== weight (B) producer ===========================
            uint32_t s = 0, ph = 0;
            const int rows = NT / cs;
            const uint32_t dst0 = smem_base + off_b + crank * rows * 128;
            for (int work = first_work(); work < total_work; work += num_clusters) {
                const int row0 = work_nt(work) * NT + (int)crank * rows;
                const int cb0 = work_ks(work) * t.cbps;
                for (int cb = cb0; cb < cb0 + t.cbps; ++cb) {
                    for (int tap = 0; tap < t.taps; ++tap) {
                        mbar_wait(bar(I_BE + s), ph ^ 1);
                        if (elect_one_sync()) {
                            const uint32_t dst = dst0 + s * B_STAGE;
                            mbar_expect_tx(bar(I_BF + s), B_STAGE);
                            if (cs > 1) {
                                tma_load_3d_mc(&tmBhi, bar(I_BF + s), dst, cb * KB, row0, tap, cmask);
                                tma_load_3d_mc(&tmBlo, bar(I_BF + s), dst + B_HALF, cb * KB, row0, tap, cmask);
                            } else {
                                tma_load_3d(&tmBhi, bar(I_BF + s), dst, cb * KB, row0, tap);
                                tma_load_3d(&tmBlo, bar(I_BF + s), dst + B_HALF, cb * KB, row0, tap);
                            }
                        }
                        __syncwarp();
                        if (++s == (uint32_t)BS) { s = 0; ph ^= 1; }
                    }
                }
            }
        } else if (warp == 5) {
            // =========================== A (halo or per-tap box) producer ===========================
            uint32_t hs = 0, ph = 0;
            for (int work = first_work(); work < total_work; work += num_clusters) {
                int n0, oy0, ox0;
                tile_origin(work, n0, oy0, ox0);
                const int cb0 = work_ks(work) * t.cbps;
                for (int u = 0; u < units; ++u) {
                    const int cb = cb0 + (t.per_tap ? u / t.taps : u);
                    const int tap = t.per_tap ? u % t.taps : 0;
                    const int ky = tap / t.KW, kx = tap - ky * t.KW;
                    mbar_wait(bar(I_HE + hs), ph ^ 1);
                    if (elect_one_sync()) {
                        mbar_expect_tx(bar(I_HF + hs), 2u * t.halo_rows * 128u);
                        const uint32_t dst = smem_base + hs * t.halo_stage_bytes;
                        tma_load_4d(&tmA, bar(I_HF + hs), dst, cb * KB, ox0 + kx - t.pw, oy0 + ky - t.ph, n0);
                        tma_load_4d(&tmA, bar(I_HF + hs), dst + t.box_bytes, cb * KB + 32, ox0 + kx - t.pw, oy0 + ky - t.ph, n0);
                    }
                    __syncwarp();
                    if (++hs == (uint32_t)HS) { hs = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp < 4) {
        // =========================== split warps: fp32 A tile -> (hi, lo) 16-bit planes, in place ===========================
        setmaxnreg_dec<REG_SPLIT>();
        const int sidx = threadIdx.x;
        const bool bf = t.prec == MN_PREC_BF16X3_TC;
        const uint32_t mask = bf ? 0xFFFF0000u : 0xFFFFE000u;
        const float xs = g.x_scale;
        float amax = 0.f;                                    // max |x * x_scale| this thread has split (range guard)
        uint32_t hs = 0, hph = 0;
        const int G = g.Cin >> 5;
        const int qs = sidx & 3, rs0 = sidx >> 2;            // 16-channel slice of the block, first halo row of this lane
        const int rows_up = (t.halo_rows + 31) & ~31;        // whole warps run every trip (__syncwarp inside)
        for (int work = first_work(); work < total_work; work += num_clusters) {
            int hn0 = 0, hoy0 = 0, hox0 = 0, gvw = 0x7fffffff;
            if (GN) {
                tile_origin(work, hn0, hoy0, hox0);
                if (g.valid_w && hn0 < g.N) gvw = g.valid_w[hn0];
            }
            const int cb0 = work_ks(work) * t.cbps;
            for (int u = 0; u < units; ++u) {
                const int cb = cb0 + (t.per_tap ? u / t.taps : u);
                // Fused GroupNorm instantiation -- four lanes per halo row: lane slice qs owns fp32 chunks 2qs, 2qs+1 of both 128-byte
                // boxes = channels [8qs, 8qs+8) and [32+8qs, 32+8qs+8) of the block, i.e. exactly the 16-byte fp16 chunks qs and 4+qs
                // of the hi and of the lo plane.  The GroupNorm constants of the lane's 16 channels live in registers, loaded before
                // the wait on the halo so that their latency overlaps the TMA.
                float gm0 = 0.f, gm1 = 0.f, ga[16], gb[16];
                if (GN) {
#pragma unroll
                    for (int e = 0; e < 16; ++e) { ga[e] = 0.f; gb[e] = 0.f; }
                    if (hn0 < g.N) {
                        const float2 mr0 = g.gn_mr[(size_t)hn0 * G + cb * 2], mr1 = g.gn_mr[(size_t)hn0 * G + cb * 2 + 1];
                        gm0 = mr0.x; gm1 = mr1.x;
#pragma unroll
                        for (int hlf = 0; hlf < 2; ++hlf)
#pragma unroll
                            for (int f = 0; f < 2; ++f) {
                                const int c0 = cb * KB + hlf * 32 + qs * 8 + f * 4;
                                const float4 gg = ldg4(g.gn_gamma + c0), be = ldg4(g.gn_beta + c0);
                                const float rs = hlf ? mr1.y : mr0.y;
                                ga[hlf * 8 + f * 4 + 0] = rs * gg.x; ga[hlf * 8 + f * 4 + 1] = rs * gg.y;
                                ga[hlf * 8 + f * 4 + 2] = rs * gg.z; ga[hlf * 8 + f * 4 + 3] = rs * gg.w;
                                gb[hlf * 8 + f * 4 + 0] = be.x; gb[hlf * 8 + f * 4 + 1] = be.y; gb[hlf * 8 + f * 4 + 2] = be.z; gb[hlf * 8 + f * 4 + 3] = be.w;
                            }
                    }
                }
                mbar_wait(bar(I_HF + hs), hph);
                uint8_t* halo = smem + hs * t.halo_stage_bytes;
                if constexpr (!GN) {
                    // Plain split: one lane per halo row, stored as it converts.  row0 (channels 0-31) becomes the hi plane and row1
                    // (channels 32-63) the lo plane, chunks 0-3 of each holding channels 0-31: once row0 is in registers its hi words
                    // can overwrite it, but its lo words have to wait until row1 has been read.
                    auto load8 = [&](const uint8_t* src, int sw, float4 (&v)[8]) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const float4*>(src + ((j ^ sw) << 4));
                    };
                    auto split16 = [&](float4 (&vv)[8], uint32_t (&hi)[16], uint32_t (&lo)[16]) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            float4 v = vv[j];
                            v.x *= xs; v.y *= xs; v.z *= xs; v.w *= xs;
                            amax = fmaxf(fmaxf(amax, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
                            const float h0 = __uint_as_float(__float_as_uint(v.x) & mask), h1 = __uint_as_float(__float_as_uint(v.y) & mask);
                            const float h2 = __uint_as_float(__float_as_uint(v.z) & mask), h3 = __uint_as_float(__float_as_uint(v.w) & mask);
                            if (bf) {
                                hi[2 * j] = pack_bf16(h0, h1); hi[2 * j + 1] = pack_bf16(h2, h3);
                                lo[2 * j] = pack_bf16(v.x - h0, v.y - h1); lo[2 * j + 1] = pack_bf16(v.z - h2, v.w - h3);
                            } else {
                                hi[2 * j] = pack_f16(h0, h1); hi[2 * j + 1] = pack_f16(h2, h3);
                                lo[2 * j] = pack_f16(v.x - h0, v.y - h1); lo[2 * j + 1] = pack_f16(v.z - h2, v.w - h3);
                            }
                        }
                    };
                    auto store4 = [&](uint8_t* dst, int sw, int jj0, const uint32_t (&w)[16]) {
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj)
                            *reinterpret_cast<uint4*>(dst + (((jj0 + jj) ^ sw) << 4)) = make_uint4(w[4 * jj], w[4 * jj + 1], w[4 * jj + 2], w[4 * jj + 3]);
                    };
                    for (int rho = sidx; rho < t.halo_rows; rho += 128) {
                        uint8_t* row0 = halo + rho * 128;
                        uint8_t* row1 = row0 + t.box_bytes;
                        const int sw = rho & 7;
                        float4 v[8];
                        uint32_t hi[16], lo[16];
                        load8(row0, sw, v);
                        split16(v, hi, lo);
                        store4(row0, sw, 0, hi);
                        load8(row1, sw, v);
                        store4(row1, sw, 0, lo);
                        split16(v, hi, lo);
                        store4(row0, sw, 4, hi);
                        store4(row1, sw, 4, lo);
                    }
                } else
                for (int rho = rs0; rho < rows_up; rho += 32) {
                    const bool live = rho < t.halo_rows;
                    uint8_t* row0 = halo + rho * 128;
                    uint8_t* row1 = row0 + t.box_bytes;
                    const int sw = rho & 7;
                    const uint32_t o0 = (uint32_t)((2 * qs) ^ sw) << 4, o1 = (uint32_t)((2 * qs + 1) ^ sw) << 4;
                    float4 v[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (live) {
                        v[0] = *reinterpret_cast<const float4*>(row0 + o0); v[1] = *reinterpret_cast<const float4*>(row0 + o1);
                        v[2] = *reinterpret_cast<const float4*>(row1 + o0); v[3] = *reinterpret_cast<const float4*>(row1 + o1);
                    }
                    // which pixel is this halo row, is it inside the image / the valid window?  (one sample per tile: plan TN == 1)
                    const int hy = rho / t.HWd, hx = rho - hy * t.HWd;
                    const int y = hoy0 - t.ph + hy, x = hox0 - t.pw + hx;
                    const bool inside = hn0 < g.N && (unsigned)y < (unsigned)g.H && (unsigned)x < (unsigned)g.W && x < gvw;
                    uint32_t hw[8], lw[8];          // hi / lo words: [0..3] = chunk qs, [4..7] = chunk 4+qs
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float tt[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
                        const float mean = (k >> 1) ? gm1 : gm0;
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float uu = fmaf(tt[e] - mean, ga[k * 4 + e], gb[k * 4 + e]);
                            if (g.gn_swish) uu = __fdividef(uu, 1.f + __expf(-uu));     // ex2.approx + rcp.approx: ~2e-7 relative on the sigmoid
                            tt[e] = inside ? uu * xs : 0.f;
                        }
                        amax = fmaxf(fmaxf(amax, fabsf(tt[0])), fmaxf(fabsf(tt[1]), fmaxf(fabsf(tt[2]), fabsf(tt[3]))));
                        const float h0 = __uint_as_float(__float_as_uint(tt[0]) & mask), h1 = __uint_as_float(__float_as_uint(tt[1]) & mask);
                        const float h2 = __uint_as_float(__float_as_uint(tt[2]) & mask), h3 = __uint_as_float(__float_as_uint(tt[3]) & mask);
                        if (bf) {
                            hw[2 * k] = pack_bf16(h0, h1); hw[2 * k + 1] = pack_bf16(h2, h3);
                            lw[2 * k] = pack_bf16(tt[0] - h0, tt[1] - h1); lw[2 * k + 1] = pack_bf16(tt[2] - h2, tt[3] - h3);
                        } else {
                            hw[2 * k] = pack_f16(h0, h1); hw[2 * k + 1] = pack_f16(h2, h3);
                            lw[2 * k] = pack_f16(tt[0] - h0, tt[1] - h1); lw[2 * k + 1] = pack_f16(tt[2] - h2, tt[3] - h3);
                        }
                    }
                    // the four lanes of a row (same warp) have read all 256 bytes of it: overwrite in place (row0 <- hi plane, row1 <- lo plane).
                    // Odd rows store their upper chunk first: the two rows of a quarter-warp then hit disjoint banks.
                    __syncwarp();
                    if (live) {
                        const uint32_t ca = (uint32_t)(qs ^ sw) << 4, cb2 = (uint32_t)((4 + qs) ^ sw) << 4;
                        const uint4 ha = make_uint4(hw[0], hw[1], hw[2], hw[3]), hb = make_uint4(hw[4], hw[5], hw[6], hw[7]);
                        const uint4 la = make_uint4(lw[0], lw[1], lw[2], lw[3]), lb = make_uint4(lw[4], lw[5], lw[6], lw[7]);
                        const bool odd = (rho & 1) != 0;
                        const uint32_t c1 = odd ? cb2 : ca, c2 = odd ? ca : cb2;
                        const uint4 h1 = odd ? hb : ha, h2 = odd ? ha : hb, l1 = odd ? lb : la, l2 = odd ? la : lb;
                        *reinterpret_cast<uint4*>(row0 + c1) = h1; *reinterpret_cast<uint4*>(row1 + c1) = l1;
                        *reinterpret_cast<uint4*>(row0 + c2) = h2; *reinterpret_cast<uint4*>(row1 + c2) = l2;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // these generic writes precede the next TMA refill
                mbar_arrive(bar(I_SD + hs));
                if (++hs == (uint32_t)HS) { hs = 0; hph ^= 1; }
            }
        }
        conv_range_report(g, __float_as_uint(amax), t.prec == MN_PREC_F16X3_TC || t.prec == MN_PREC_F16X1_TC);
    } else {
        // =========================== consumer warpgroups: ldmatrix A fragments + wgmma + epilogue ===========================
        setmaxnreg_inc<REG_CONS>();
        const int wg = (warp - 8) >> 2, wq = warp & 3;       // warpgroup (pixel rows 64wg..), warp within it (16 rows each)
        const int wtid = threadIdx.x - 256 - wg * 128;        // 0..127 inside the warpgroup
        constexpr bool bf = MODE == 1, three = MODE != 2;
        // the tile row this lane addresses for ldmatrix (rows 0-15 of the warp's 16-row slice, k-chunk lane >> 4)
        const int r = wg * 64 + wq * 16 + (lane & 15);
        const int tn = r / (t.TH * t.TW);
        const int rem = r - tn * (t.TH * t.TW);
        const int th = rem / t.TW, tw = rem - th * t.TW;
        const int rho0 = tn < t.TN ? (tn * t.HHt + th) * t.HWd + tw : 0;   // A-tile row of tap (0,0); unused MMA rows read row 0
        const uint32_t kchunk = (uint32_t)(lane >> 4);
        const uint64_t desc0 = make_b_desc(smem_base + off_b);
        const float wscale = (t.wscale ? *t.wscale : 1.f) / g.x_scale;      // x_scale is a power of two: exact
        // The tensor core truncates (toward zero) every time it adds into the fp32 accumulator: measured mean shrink of the main
        // accumulator = 1.5e-8 per accumulation step, sign-symmetric, independent of K (tools/probe_tc_bias.py).  Undo the
        // expected shrink of D (K/16 steps); Dc is 2^-11 of the result and needs nothing.
        const float dfix = 1.f + 1.5e-8f * (float)(t.taps * t.cbps * (KB / 16));
        float* wstg = stg + wg * 64 * STG_PITCH;
        // Stage releases, once per warpgroup, after the wgmma group that read the stage has retired (the group's completion covers
        // every warp's ldmatrix and B reads).  A weight stage is filled by the multicast of every CTA of the cluster: warp c of the
        // warpgroup arrives on CTA c's barrier.
        auto release_b = [&](uint32_t s) {
            if (cs > 1) { if (lane == 0 && wq < cs) mbar_arrive_cluster(mapa_u32(bar(I_BE + s), (uint32_t)wq)); }
            else if (wtid == 0) mbar_arrive(bar(I_BE + s));
        };
        auto release_a = [&](uint32_t s) { if (wtid == 0) mbar_arrive(bar(I_HE + s)); };
        constexpr int ND = NT / 2;                            // accumulator registers per thread (64 rows x NT columns / 128 threads)
        uint32_t hs = 0, hph = 0, bs = 0, bph = 0;
        for (int work = first_work(); work < total_work; work += num_clusters) {
            float d[ND], dc[ND];
#pragma unroll
            for (int i = 0; i < ND; ++i) { d[i] = 0.f; dc[i] = 0.f; }
            auto fence_acc = [&]() {
#pragma unroll
                for (int i = 0; i < ND; ++i) { wg_fence_operand(d[i]); if (three) wg_fence_operand(dc[i]); }
            };
            // One wgmma group per tap, drained with wait_group 0: ptxas serializes register-A wgmmas (C7513) when ldmatrix writes
            // fragment registers while a group is still in flight, so within a warpgroup the taps stay sequential and the overlap
            // comes from the other consumer warpgroup (128-wide items give it twice the MMA time per tap to cover).
            int kb = 0;
            for (int u = 0; u < units; ++u) {
                mbar_wait(bar(I_SD + hs), hph);
                const uint32_t abase = smem_base + hs * t.halo_stage_bytes;
                int ky = 0, kx = 0;
                for (int tap = 0; tap < unit_taps; ++tap, ++kb) {
                    const int rho = rho0 + ky * t.HWd + kx;
                    if (++kx == t.KW) { kx = 0; ++ky; }
                    const uint32_t arow = abase + rho * 128;
                    const uint32_t sw = (uint32_t)(rho & 7);
                    uint32_t ah[4][4], al[4][4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t off = ((2u * j + kchunk) ^ sw) << 4;
                        ldsm_x4(arow + off, ah[j]);
                        if (three) ldsm_x4(arow + t.box_bytes + off, al[j]);
                    }
                    mbar_wait(bar(I_BF + bs), bph);
                    const uint64_t dh0 = desc0 + (uint64_t)((bs * B_STAGE) >> 4);   // start-address field is in 16-byte units
                    const uint64_t dl0 = dh0 + (uint64_t)(B_HALF >> 4);
                    fence_acc();
                    wg_fence();
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t acc = (kb | j) != 0;
                        wgmma_k16_rs<NT, bf>(d, ah[j], dh0 + 2 * j, acc);
                        if (three) { wgmma_k16_rs<NT, bf>(dc, ah[j], dl0 + 2 * j, acc); wgmma_k16_rs<NT, bf>(dc, al[j], dh0 + 2 * j, 1); }
                    }
                    wg_commit();
                    wg_wait<0>();
                    fence_acc();
                    release_b(bs);
                    if (++bs == (uint32_t)BS) { bs = 0; bph ^= 1; }
                }
                release_a(hs);                                        // every tap of this A tile has been read
                if (++hs == (uint32_t)HS) { hs = 0; hph ^= 1; }
            }

            // ---- epilogue, per 64-column half: accumulators -> staging rows (this warpgroup's 64 rows) -> fused epilogue with
            // float4 row stores ----
#pragma unroll
            for (int i = 0; i < ND; ++i) d[i] = three ? fmaf(d[i], dfix, dc[i]) * wscale : d[i] * wscale;
            const int nt_i = work_nt(work);
            const int ks = work_ks(work);
            int n0, oy0, ox0;
            tile_origin(work, n0, oy0, ox0);
#pragma unroll 1
            for (int h = 0; h < NT / 64; ++h) {
                named_bar_sync(1 + wg, 128);                              // the previous half's / item's rows have been stored
                if (h == 0 && wtid < 64) {
                    const int rr = wg * 64 + wtid;
                    const int tn2 = rr / (t.TH * t.TW), rem2 = rr - tn2 * (t.TH * t.TW);
                    const int th2 = rem2 / t.TW, tw2 = rem2 - th2 * t.TW;
                    const int n = n0 + tn2, oy = oy0 + th2, ox = ox0 + tw2;
                    const bool ok = tn2 < t.TN && n < g.N && oy < g.OH && ox < g.OW;
                    rowm[rr] = ok ? (n * g.OH + oy) * g.OW + ox : -1;
                    rowm[128 + rr] = ok ? (n | ((g.valid_w && ox >= g.valid_w[n]) ? (1 << 30) : 0)) : 0;
                }
                {
                    // accumulator layout of wgmma m64nN: d[4i + {0,1}] = row (lane >> 2), cols 8i + 2(lane & 3) + {0,1}; d[4i + {2,3}] = row + 8
                    const int row = wq * 16 + (lane >> 2), col = 2 * (lane & 3);
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int i1 = ND - 32 + 4 * i;                   // columns 64 + 8i.. of the second half (== 4i when NT == 64)
                        const float v0 = h ? d[i1] : d[4 * i], v1 = h ? d[i1 + 1] : d[4 * i + 1];
                        const float v2 = h ? d[i1 + 2] : d[4 * i + 2], v3 = h ? d[i1 + 3] : d[4 * i + 3];
                        *reinterpret_cast<float2*>(wstg + row * STG_PITCH + 8 * i + col) = make_float2(v0, v1);
                        *reinterpret_cast<float2*>(wstg + (row + 8) * STG_PITCH + 8 * i + col) = make_float2(v2, v3);
                    }
                }
                named_bar_sync(1 + wg, 128);
                {
                    const int col = (lane & 15) * 4;
                    const int o = nt_i * NT + h * 64 + col;
                    const int rbase = wg * 64 + wq * 16 + (lane >> 4);   // tile rows rbase + 2i, i < 8
                    if (t.ksplit > 1) {
                        // raw partial sum of this k-slice; conv_splitk_reduce_kernel adds the slices and runs the epilogue
#pragma unroll 4
                        for (int i = 0; i < 8; ++i) {
                            const int row = rbase + 2 * i;
                            const int m = rowm[row];
                            if (m >= 0)
                                *reinterpret_cast<float4*>(g.ws + ((size_t)ks * g.M + m) * g.Cout + o) =
                                    *reinterpret_cast<const float4*>(stg + row * STG_PITCH + col);
                        }
                    } else {
                        const float4 bias4 = g.bias ? ldg4(g.bias + o) : make_float4(0.f, 0.f, 0.f, 0.f);
                        // one sample per tile (every layer except the 4x4 .. 8x8 maps): its per-sample scale vectors are loaded once
                        const bool one_n = t.TN == 1;
                        float4 os4 = make_float4(1.f, 1.f, 1.f, 1.f), y2s4 = os4;
                        float* y2base = g.y2;
                        if (one_n && n0 < g.N) {
                            if (g.out_scale) os4 = ldg4(g.out_scale + (size_t)n0 * g.os_stride + o);
                            if (g.y2 && g.y2_scale) y2s4 = ldg4(g.y2_scale + (size_t)n0 * g.y2s_stride + o);
                            // per-sample (possibly peer-GPU) destination of the second output, rebased so that row index m addresses it
                            if (g.y2_ptrs) y2base = g.y2_ptrs[n0] - (size_t)n0 * g.OH * g.OW * g.y2_cs;
                        }
                        GnAcc ga;                       // GroupNorm statistics of this thread's 8 rows x 4 channels (one group)
                        // One sample per tile, the tile inside the tensor (the plans guarantee H % TH == 0, W % TW == 0 and a power-of-two
                        // TW) and 128 pixels in it: every row is valid and its pixel index is arithmetic -- no rowm look-ups, no per-row
                        // branch.  Tiles of one sample with fewer pixels (4x16, 2x32, 1x64 maps: the halo cap of plan_tc2 leaves TN = 1
                        // with TH * TW = 64) take the rowm path, which drops the MMA rows past the tile.
                        const bool dense_tile = one_n && n0 < g.N && t.TH * t.TW == 128;
                        const int tws = __ffs(t.TW) - 1;
                        const int m00 = (n0 * g.OH + oy0) * g.OW + ox0;
                        const int vwn = (dense_tile && g.valid_w) ? g.valid_w[n0] : 0x7fffffff;
                        auto rows_dense = [&](auto tag) {
                            constexpr int ACT = decltype(tag)::value;
#pragma unroll 4     // 8 spills once the per-row path also serves one-sample tiles (ptxas -v)
                            for (int i = 0; i < 8; ++i) {
                                const int row = rbase + 2 * i;
                                const int th3 = row >> tws, tw3 = row & (t.TW - 1);
                                const int m = m00 + th3 * g.OW + tw3;
                                const float4 uv = *reinterpret_cast<const float4*>(stg + row * STG_PITCH + col);
                                const bool masked = ox0 + tw3 >= vwn;
                                const float4 w4 = conv_epilogue_row4<ACT>(g, m, n0, masked, o, uv, bias4, true, os4, true, y2s4, y2base);
                                if (g.gn_stats_out && !masked) ga.add(w4);
                            }
                        };
                        auto rows = [&](auto tag) {
                            constexpr int ACT = decltype(tag)::value;
                            if (dense_tile) { rows_dense(tag); return; }
                            if (one_n && n0 >= g.N) return;          // padding CTA of a cluster: nothing to store
#pragma unroll 4
                            for (int i = 0; i < 8; ++i) {
                                const int row = rbase + 2 * i;
                                const int m = rowm[row];
                                if (m >= 0) {
                                    const int nn = rowm[128 + row];
                                    const float4 uv = *reinterpret_cast<const float4*>(stg + row * STG_PITCH + col);
                                    const bool masked = (nn >> 30) != 0;
                                    const float4 w4 = conv_epilogue_row4<ACT>(g, m, nn & 0x3FFFFFFF, masked, o, uv, bias4, one_n, os4, one_n, y2s4, y2base);
                                    if (g.gn_stats_out && !masked) ga.add(w4);
                                }
                            }
                        };
                        switch (g.act) {
                            case MN_ACT_NONE: rows(ActTag<MN_ACT_NONE>{}); break;
                            case MN_ACT_RELU: rows(ActTag<MN_ACT_RELU>{}); break;
                            case MN_ACT_LRELU02: rows(ActTag<MN_ACT_LRELU02>{}); break;
                            default: rows(ActTag<-1>{}); break;
                        }
                        if (g.gn_stats_out) {
                            double gs, gq;
                            ga.sums(gs, gq);
                            // lanes 0-7 / 8-15 (and 16-23 / 24-31, the odd rows) hold the two 32-channel groups of this 64-column half
#pragma unroll
                            for (int sh = 1; sh <= 4; sh <<= 1) { gs += __shfl_xor_sync(0xffffffffu, gs, sh); gq += __shfl_xor_sync(0xffffffffu, gq, sh); }
                            gs += __shfl_xor_sync(0xffffffffu, gs, 16); gq += __shfl_xor_sync(0xffffffffu, gq, 16);
                            if ((lane & 23) == 0 && n0 < g.N) {        // lanes 0 and 8
                                double* dst = g.gn_stats_out + ((size_t)n0 * (g.Cout >> 5) + (o >> 5)) * 2;
                                atomicAdd(dst, gs);
                                atomicAdd(dst + 1, gq);
                            }
                        }
                    }
                }
            }
        }
    }
    __syncthreads();
    if (cs > 1) cluster_sync_all();     // no CTA leaves while its peer may still multicast into it or arrive on its barriers
}

// ------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode2() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// checks shared by both tilings; fills the fields that do not depend on the pixel tile
bool plan_common(const ConvGeom& g, Tc2Plan& p) {
    auto fail = [&](const char* w) { p.ok = false; p.why = w; return false; };
    if (g.sh != 1 || g.sw != 1) return fail("stride != 1");
    const bool k3 = g.KH == 3 && g.KW == 3 && g.ph == 1 && g.pw == 1, k1 = g.KH == 1 && g.KW == 1 && g.ph == 0 && g.pw == 0;
    if (!k3 && !k1) return fail("only 3x3/pad1 and 1x1/pad0");
    if (g.Cin % KB != 0) return fail("Cin % 64 != 0");
    if (g.Cout % 64 != 0) return fail("Cout % 64 != 0");
    if (g.x_cs % 4 != 0 || (reinterpret_cast<uintptr_t>(g.x) & 15)) return fail("x alignment");
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if ((g.y && (g.y_cs % 4 || !al16(g.y))) || (g.y2 && (g.y2_cs % 4 || !al16(g.y2))) || (g.residual && (g.res_cs % 4 || !al16(g.residual))) ||
        (g.out_scale && (g.os_stride % 4 || !al16(g.out_scale))) || (g.y2_scale && (g.y2s_stride % 4 || !al16(g.y2_scale))) ||
        (g.bias && !al16(g.bias)))
        return fail("epilogue operands must be 16-byte aligned with channel strides that are multiples of 4");
    p.t.KW = g.KW;
    p.t.cblocks = g.Cin / KB; p.t.taps = g.KH * g.KW;
    return true;
}

// split-K, the shared-memory rings and the plan's size for work items of nt output channels
void plan_nt(const ConvGeom& g, Tc2Plan& p, bool allow_ksplit, int nt) {
    Tc2Geom& t = p.t;
    t.nt = nt;
    t.n_tiles = g.Cout / nt;
    // split-K: few tiles but a deep K loop (4x4 / 8x8 generator layers, ResNet stages at batch 1) -> spread the channel blocks of
    // a tile over several CTAs; partial sums go to the caller's workspace and conv_splitk_reduce_kernel finishes the job.
    t.ksplit = 1;
    if (allow_ksplit) {
        const int items = t.m_groups * t.n_tiles, slots = mn_num_sms() / t.cs;
        while (t.ksplit * 2 * items <= slots && t.cblocks % (t.ksplit * 2) == 0 && t.ksplit < 8) t.ksplit *= 2;
        while (t.ksplit > 1 && (int64_t)t.ksplit * g.M * g.Cout * 4 > g.ws_bytes) t.ksplit >>= 1;
        if (t.ksplit > 1 && (!g.ws || g.gn_mr || (g.Cout & 3) || g.y2_ptrs || g.gn_stats_out)) t.ksplit = 1;
    }
    t.cbps = t.cblocks / t.ksplit;
    // A ring: a third stage when it still leaves >= 3 weight stages and the K loop per A tile is short
    const int other = STG_BYTES + 1024 + 256 + 1024;
    const int units = t.per_tap ? t.cbps * t.taps : t.cbps;
    t.hstages = 2;
    if (3 * t.halo_stage_bytes + other + 3 * b_stage(nt) <= SMEM_LIMIT && (t.per_tap || (units <= 4 && units >= 2))) t.hstages = 3;
    const int fixed = t.hstages * t.halo_stage_bytes + other;
    int bs = (SMEM_LIMIT - fixed) / b_stage(nt);
    if (bs > MAX_BSTAGES) bs = MAX_BSTAGES;
    t.bstages = bs;
    p.smem = fixed + bs * b_stage(nt);
}

// persistent-grid makespan of a plan in units of one 64-channel x 64-k x tap block per pixel tile
int64_t plan_cost(const Tc2Geom& t) {
    const int clusters = mn_num_sms() / t.cs;
    const int64_t waves = (t.m_groups * t.n_tiles * t.ksplit + clusters - 1) / clusters;
    return waves * (t.nt / 64) * t.cbps;
}

// cluster pairing, the work-item width, split-K and the shared-memory rings, once the pixel tile is known
bool plan_finish(const ConvGeom& g, Tc2Plan& p, bool allow_ksplit) {
    Tc2Geom& t = p.t;
    t.box_bytes = (t.halo_rows * 128 + 1023) & ~1023;
    t.halo_stage_bytes = 2 * t.box_bytes;
    t.m_tiles = t.tiles_w * t.tiles_h * t.tiles_n;
    t.cs = t.m_tiles >= 2 ? 2 : 1;
    t.m_groups = (t.m_tiles + t.cs - 1) / t.cs;
    // 128-channel work items read each A fragment and split each halo for twice the outputs.  Take them unless they leave
    // fewer than 3 weight stages or halving the number of items lengthens the persistent grid's makespan (Cout = 64 layers,
    // few-tile layers at batch 1).  Equal makespans go to the wider items only if they need no deeper split-K: on small layers
    // the extra partial sums and reduce launch cost more than the wider tile saves.
    plan_nt(g, p, allow_ksplit, 64);
    if (g.Cout % 128 == 0) {
        Tc2Plan wide = p;
        plan_nt(g, wide, allow_ksplit, 128);
        const int64_t cw = plan_cost(wide.t), cn = plan_cost(p.t);
        if (wide.t.bstages >= 3 && (cw < cn || (cw == cn && wide.t.ksplit <= p.t.ksplit))) p = wide;
    }
    if (t.bstages < 2) { p.ok = false; p.why = "not enough shared memory for 2 weight stages"; return false; }
    p.ok = true;
    return true;
}

// halo tiling ("version 2"): one (TH+2) x (TW+2) halo per channel block; drops the optional requests of tiles of several samples
Tc2Plan plan_tc2(ConvGeom& g) {
    Tc2Plan p{};
    auto fail = [&](const char* w) { p.ok = false; p.why = w; return p; };
    if (!plan_common(g, p)) return p;
    Tc2Geom& t = p.t;
    t.per_tap = 0;
    t.TH = g.H < 8 ? g.H : 8;
    if (!is_pow2(t.TH) || g.H % t.TH) return fail("H must be a multiple of 8 (or a power of two below 8)");
    const int maxw = 128 / t.TH;
    t.TW = g.W < maxw ? g.W : maxw;
    if (!is_pow2(t.TW) || g.W % t.TW) return fail("W must be a multiple of 128/TH (or a power of two below it)");
    t.TN = 128 / (t.TH * t.TW);
    t.ph = g.ph; t.pw = g.pw;
    t.HHt = t.TH + 2 * g.ph; t.HWd = t.TW + 2 * g.pw;
    // tiny images (4x4): 8 whole images per tile would need a 288-row halo; use fewer images per tile and leave the upper
    // MMA rows unused (their rows map outside the tensor and are masked in the epilogue).
    while (t.TN > 1 && t.TN * t.HHt * t.HWd > 208) t.TN >>= 1;
    t.halo_rows = t.TN * t.HHt * t.HWd;
    if (t.halo_rows > 208) return fail("halo tile too large for shared memory");
    if (g.y2_ptrs && t.TN != 1) return fail("per-sample output pointers need samples of at least one whole pixel tile (OH*OW >= 128)");
    if (t.TN != 1) { g.gn_mr = nullptr; g.gn_stats_out = nullptr; }    // both work per sample: one sample per tile or not at all
    if (t.HWd > 256 || t.HHt > 256 || t.TN > 256) return fail("TMA box dim");
    t.tiles_w = g.W / t.TW; t.tiles_h = g.H / t.TH; t.tiles_n = (g.N + t.TN - 1) / t.TN;
    plan_finish(g, p, true);
    return p;
}

// per-tap tiling ("version 1"): a 128-pixel box per (channel block, tap); covers the maps the halo tiling cannot
Tc2Plan plan_tc1(const ConvGeom& g) {
    Tc2Plan p{};
    auto fail = [&](const char* w) { p.ok = false; p.why = w; return p; };
    if (!plan_common(g, p)) return p;
    Tc2Geom& t = p.t;
    t.per_tap = 1;
    int TW, TH, TN;
    if (g.W >= 128) { if (g.W % 128) return fail("W % 128"); TW = 128; TH = 1; TN = 1; }
    else {
        if (128 % g.W) return fail("W does not divide 128");
        TW = g.W;
        const int rows = 128 / TW;
        if (g.H >= rows) { if (g.H % rows) return fail("H % tile rows"); TH = rows; TN = 1; }
        else { if (rows % g.H) return fail("H does not divide tile rows"); TH = g.H; TN = rows / g.H; }
    }
    t.TW = TW; t.TH = TH; t.TN = TN;
    t.HWd = TW; t.HHt = TH; t.ph = g.ph; t.pw = g.pw;
    t.halo_rows = 128;
    t.tiles_w = g.W / TW; t.tiles_h = g.H / TH; t.tiles_n = (g.N + TN - 1) / TN;
    plan_finish(g, p, false);
    return p;
}

template <bool GN, int MODE, int NT>
int launch_tc2(const CUtensorMap& ma, const CUtensorMap& mbh, const CUtensorMap& mbl, const ConvGeom& g, const Tc2Plan& p, cudaStream_t st) {
    static unsigned long long smem_done = 0;
    MN_CUDA_CHECK(mn_ensure_dyn_smem(conv_tc2_kernel<GN, MODE, NT>, SMEM_LIMIT, &smem_done));
    const Tc2Geom& t = p.t;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(mn_conv_tc_ctas(t), 1, 1);
    cfg.blockDim = dim3(NUM_THREADS2, 1, 1);
    cfg.dynamicSmemBytes = p.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = t.cs; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = mn_pdl_enabled() ? 2 : 1;
    MN_CUDA_CHECK(cudaLaunchKernelEx(&cfg, conv_tc2_kernel<GN, MODE, NT>, ma, mbh, mbl, g, t));
    return MN_OK;
}

template <bool GN, int MODE>
int launch_tc2_nt(const CUtensorMap& ma, const CUtensorMap& mbh, const CUtensorMap& mbl, const ConvGeom& g, const Tc2Plan& p, cudaStream_t st) {
    return p.t.nt == 128 ? launch_tc2<GN, MODE, 128>(ma, mbh, mbl, g, p, st) : launch_tc2<GN, MODE, 64>(ma, mbh, mbl, g, p, st);
}

}  // namespace

int mn_conv_tc_ctas(const Tc2Geom& t) {
    const int total_work = t.m_groups * t.n_tiles * t.ksplit;
    int sms = mn_num_sms();
    if (mn_max_ctas() > 0 && mn_max_ctas() < sms) sms = mn_max_ctas();
    int clusters = sms / t.cs;
    if (clusters < 1) clusters = 1;
    if (clusters > total_work) clusters = total_work;
    return clusters * t.cs;
}

Tc2Plan mn_conv_tc_plan(ConvGeom& g) {
    const Tc2Plan halo = plan_tc2(g);
    if (halo.ok) return halo;
    if (g.y2_ptrs) {
        mn_set_error("mn_conv2d_nhwc: per-sample output pointers (y2_ptrs) exist only in the tensor-core halo tiling, which does not run this shape (%s)", halo.why);
        return halo;
    }
    g.gn_mr = nullptr; g.gn_stats_out = nullptr;      // requests of the halo tiling only
    const Tc2Plan per_tap = plan_tc1(g);
    if (!per_tap.ok)
        mn_set_error("tensor-core path unsupported: halo tiling: %s; per-tap tiling: %s", halo.why, per_tap.why);
    return per_tap;
}

int mn_conv_tc_launch(const ConvGeom& g, Tc2Plan& p, const void* w_hi, const void* w_lo, const float* w_scale, int prec, cudaStream_t st) {
    if (!w_hi || !w_lo || !w_scale) { mn_set_error("mn_conv2d_nhwc: tensor-core precision needs packed w_tc_hi/w_tc_lo/w_tc_scale"); return MN_ERR_INVALID; }
    PFN_encodeTiled enc = get_encode2();
    if (!enc) { mn_set_error("cuTensorMapEncodeTiled not available from the driver"); return MN_ERR_CUDA; }
    CUtensorMap ma, mbh, mbl;
    Tc2Geom& t = p.t;
    {
        cuuint64_t dims[4] = {(cuuint64_t)g.Cin, (cuuint64_t)g.W, (cuuint64_t)g.H, (cuuint64_t)g.N};
        cuuint64_t strides[3] = {(cuuint64_t)g.x_cs * 4, (cuuint64_t)g.W * g.x_cs * 4, (cuuint64_t)g.H * g.W * g.x_cs * 4};
        cuuint32_t box[4] = {32, (cuuint32_t)t.HWd, (cuuint32_t)t.HHt, (cuuint32_t)t.TN};
        cuuint32_t es[4] = {1, 1, 1, 1};
        CUresult r = enc(&ma, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(g.x), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { mn_set_error("cuTensorMapEncodeTiled(A) failed: %d", (int)r); return MN_ERR_CUDA; }
    }
    const CUtensorMapDataType dt = (prec == MN_PREC_BF16X3_TC) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    for (int which = 0; which < 2; ++which) {
        cuuint64_t dims[3] = {(cuuint64_t)g.Cin, (cuuint64_t)g.Cout, (cuuint64_t)(g.KH * g.KW)};
        cuuint64_t strides[2] = {(cuuint64_t)g.Cin * 2, (cuuint64_t)g.Cin * g.Cout * 2};
        cuuint32_t box[3] = {64, (cuuint32_t)(t.nt / t.cs), 1};
        cuuint32_t es[3] = {1, 1, 1};
        CUresult r = enc(which ? &mbl : &mbh, dt, 3, const_cast<void*>(which ? w_lo : w_hi), dims, strides, box, es,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { mn_set_error("cuTensorMapEncodeTiled(B) failed: %d", (int)r); return MN_ERR_CUDA; }
    }
    t.wscale = w_scale + 1;
    t.prec = prec;
    int rc;
    if (prec == MN_PREC_BF16X3_TC) rc = g.gn_mr ? launch_tc2_nt<true, 1>(ma, mbh, mbl, g, p, st) : launch_tc2_nt<false, 1>(ma, mbh, mbl, g, p, st);
    else if (prec == MN_PREC_F16X1_TC) rc = g.gn_mr ? launch_tc2_nt<true, 2>(ma, mbh, mbl, g, p, st) : launch_tc2_nt<false, 2>(ma, mbh, mbl, g, p, st);
    else rc = g.gn_mr ? launch_tc2_nt<true, 0>(ma, mbh, mbl, g, p, st) : launch_tc2_nt<false, 0>(ma, mbh, mbl, g, p, st);
    if (rc != MN_OK || t.ksplit == 1) return rc;
    ConvGeom gr = g;
    gr.splits = t.ksplit;
    return mn_conv_splitk_reduce_launch(gr, st);
}
