// mn_conv2d_nhwc / mn_conv2d_plan: argument validation and the one dispatch decision between the convolution kernels.
#include "mn_common.cuh"
#include "conv_common.cuh"

static int make_geom(const mn_conv_params* p, ConvGeom& g) {
    MN_REQUIRE(p != nullptr, "mn_conv2d_nhwc: null params");
    MN_REQUIRE(p->x && p->w && (p->y || p->y2), "mn_conv2d_nhwc: null x/w/y");
    MN_REQUIRE(p->N > 0 && p->H > 0 && p->W > 0 && p->Cin > 0 && p->Cout > 0, "mn_conv2d_nhwc: non-positive dims");
    MN_REQUIRE(p->KH > 0 && p->KW > 0 && p->stride_h > 0 && p->stride_w > 0 && p->pad_h >= 0 && p->pad_w >= 0,
               "mn_conv2d_nhwc: bad kernel/stride/pad");
    MN_REQUIRE(p->x_cs >= p->Cin, "mn_conv2d_nhwc: x_cs < Cin");
    g.x = p->x; g.w = p->w; g.y = p->y; g.y2 = p->y2;
    g.bias = p->bias; g.out_scale = p->out_scale; g.residual = p->residual; g.y2_scale = p->y2_scale;
    g.valid_w = p->valid_w; g.ws = p->workspace; g.ws_bytes = p->workspace ? p->workspace_bytes : 0;
    g.gn_mr = reinterpret_cast<const float2*>(p->gn_mean_rstd); g.gn_gamma = p->gn_gamma; g.gn_beta = p->gn_beta; g.gn_swish = p->gn_swish;
    MN_REQUIRE(!p->gn_mean_rstd || (p->gn_gamma && p->gn_beta), "mn_conv2d_nhwc: fused GroupNorm needs gamma and beta");
    g.N = p->N; g.H = p->H; g.W = p->W; g.Cin = p->Cin; g.x_cs = p->x_cs;
    g.KH = p->KH; g.KW = p->KW; g.sh = p->stride_h; g.sw = p->stride_w; g.ph = p->pad_h; g.pw = p->pad_w; g.Cout = p->Cout;
    g.OH = (p->H + 2 * p->pad_h - p->KH) / p->stride_h + 1;
    g.OW = (p->W + 2 * p->pad_w - p->KW) / p->stride_w + 1;
    MN_REQUIRE(g.OH > 0 && g.OW > 0, "mn_conv2d_nhwc: empty output");
    g.y_cs = p->y_cs; g.y2_cs = p->y2_cs; g.res_cs = p->res_cs; g.res_bcast = p->res_broadcast_n;
    MN_REQUIRE(!p->y || p->y_cs >= p->Cout, "mn_conv2d_nhwc: y_cs < Cout");
    MN_REQUIRE(!p->y2 || p->y2_cs >= p->Cout, "mn_conv2d_nhwc: y2_cs < Cout");
    MN_REQUIRE(!p->residual || p->res_cs >= p->Cout, "mn_conv2d_nhwc: res_cs < Cout");
    g.os_stride = p->out_scale_stride > 0 ? p->out_scale_stride : p->Cout;
    g.y2s_stride = p->y2_scale_stride > 0 ? p->y2_scale_stride : p->Cout;
    g.act = p->act; g.gain = p->act_gain;
    const int64_t M = (int64_t)p->N * g.OH * g.OW;
    MN_REQUIRE(M < (1ll << 31) && (int64_t)p->KH * p->KW * p->Cin < (1ll << 31), "mn_conv2d_nhwc: problem too large");
    g.M = (int)M; g.K = p->KH * p->KW * p->Cin;
    g.ktiles = g.ktiles_per_split = 0; g.splits = 1;
    g.x_scale = p->x_scale > 0.f ? p->x_scale : 1.f; g.x_absmax = p->x_absmax; g.range_flag = p->range_flag; g.range_tag = p->range_tag;
    g.y2_ptrs = p->y2_ptrs; g.gn_stats_out = p->gn_stats_out;
    MN_REQUIRE(!p->gn_stats_out || p->y, "mn_conv2d_nhwc: gn_stats_out needs the y output");
    MN_REQUIRE(!p->y2_ptrs || p->y2, "mn_conv2d_nhwc: y2_ptrs needs the second output enabled (y2 != NULL)");
    return MN_OK;
}

// The one dispatch decision: which kernel runs *p, with which tile and split count, and which of the optional requests of the
// halo tiling (fused GroupNorm input, epilogue statistics) it honours; the ones it drops are cleared in g.  mn_conv2d_nhwc launches
// what it returns and mn_conv2d_plan reports it, so the two cannot disagree.
static int plan_conv(const mn_conv_params* p, ConvGeom& g, mn_conv_plan* r, Tc2Plan* tc) {
    const int rc = make_geom(p, g);
    if (rc != MN_OK) return rc;
    *r = mn_conv_plan{};
    r->precision = p->precision;
    r->splits = 1;
    switch (p->precision) {
        case MN_PREC_FP32_SIMT:
            if (g.y2_ptrs) {
                mn_set_error("mn_conv2d_nhwc: per-sample output pointers (y2_ptrs) exist only in the tensor-core halo tiling");
                return MN_ERR_UNSUPPORTED;
            }
            g.gn_mr = nullptr; g.gn_stats_out = nullptr;
            if (mn_conv_small_supported(g)) {
                r->kernel = MN_CONV_KERNEL_SMALL;
            } else {
                r->kernel = MN_CONV_KERNEL_SIMT;
                r->splits = mn_conv_simt_plan_splits(g, g.ws_bytes, p->split_k);
            }
            break;
        case MN_PREC_F16X3_TC:
        case MN_PREC_BF16X3_TC:
        case MN_PREC_F16X1_TC:
            *tc = mn_conv_tc_plan(g);
            if (!tc->ok) return MN_ERR_UNSUPPORTED;
            r->kernel = tc->t.per_tap ? MN_CONV_KERNEL_TC1 : MN_CONV_KERNEL_TC2;
            r->nt = tc->t.nt; r->TN = tc->t.TN; r->TH = tc->t.TH; r->TW = tc->t.TW; r->splits = tc->t.ksplit;
            r->cs = tc->t.cs; r->m_tiles = tc->t.m_tiles; r->work_items = tc->t.m_groups * tc->t.n_tiles * tc->t.ksplit;
            r->hstages = tc->t.hstages; r->bstages = tc->t.bstages; r->ctas = mn_conv_tc_ctas(tc->t);
            break;
        default:
            mn_set_error("mn_conv2d_nhwc: unknown precision mode %d", p->precision);
            return MN_ERR_UNSUPPORTED;
    }
    r->gn_fused = g.gn_mr != nullptr;
    r->gn_stats_out = g.gn_stats_out != nullptr;
    return MN_OK;
}

extern "C" int mn_conv2d_plan(const mn_conv_params* p, mn_conv_plan* out) {
    MN_REQUIRE(out != nullptr, "mn_conv2d_plan: null output");
    ConvGeom g;
    mn_conv_plan r;
    Tc2Plan tc;
    const int rc = plan_conv(p, g, &r, &tc);
    if (rc == MN_OK) *out = r;
    return rc;
}

extern "C" int mn_conv2d_nhwc(const mn_conv_params* p, void* stream) {
    ConvGeom g;
    mn_conv_plan r;
    Tc2Plan tc;
    const int rc = plan_conv(p, g, &r, &tc);
    if (rc != MN_OK) return rc;
    // a request the plan drops is refused, not ignored: the caller would get an input never normalised or statistics never written
    if ((p->gn_mean_rstd && !r.gn_fused) || (p->gn_stats_out && !r.gn_stats_out)) {
        mn_set_error("mn_conv2d_nhwc: the fused GroupNorm input (gn_mean_rstd) and the epilogue statistics (gn_stats_out) need the "
                     "tensor-core halo tiling with one sample per pixel tile; mn_conv2d_plan drops them for this problem");
        return MN_ERR_UNSUPPORTED;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (r.kernel) {
        case MN_CONV_KERNEL_SMALL: return mn_conv_small_launch(g, st);
        case MN_CONV_KERNEL_SIMT: g.splits = r.splits; return mn_conv_simt_launch(g, st);
        default: return mn_conv_tc_launch(g, tc, p->w_tc_hi, p->w_tc_lo, p->w_tc_scale, p->precision, st);
    }
}
