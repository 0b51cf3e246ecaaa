/*
 * marconet_b200.h -- C ABI of libmarconet_b200.so (sm_90a).
 *
 * The reference (csxmli2016/MARCONet) has no FFI/plugin boundary of its own: its hot
 * path is Python modules in models/networks.py that call torch.nn.functional ops
 * (cuDNN / cuBLAS / ATen kernels) plus one third-party CUDA extension
 * (basicsr.ops.fused_act, models/networks.py:10).  This header is the boundary a
 * maintainer would bind instead of those calls: every entry point names the
 * reference call site(s) it replaces.  All functions
 *   - take raw DEVICE pointers and sizes (no torch types),
 *   - are asynchronous on the given stream (a cudaStream_t passed as void*),
 *   - never allocate persistent device memory (the caller owns every buffer,
 *     including workspaces),
 *   - return 0 on success or a negative mn_status; mn_last_error() returns a
 *     message for the calling thread.
 *
 * Activation layout everywhere: NHWC, fp32, channel stride given explicitly as
 * `*_cs` (floats per pixel in the underlying buffer) so that operators can read
 * from / write into channel slices of concatenated buffers without copies.
 */
#ifndef MARCONET_B200_H
#define MARCONET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    MN_OK = 0,
    MN_ERR_INVALID = -1,   /* bad argument (shape, alignment, null pointer)      */
    MN_ERR_CUDA = -2,      /* a CUDA runtime/driver call failed (see last error) */
    MN_ERR_UNSUPPORTED = -3,
    MN_ERR_WORKSPACE = -4  /* workspace too small                                 */
} mn_status;

typedef enum {
    MN_ACT_NONE = 0,
    MN_ACT_RELU = 1,       /* models/resnet.py:24,29                              */
    MN_ACT_LRELU02 = 2,    /* nn.LeakyReLU(0.2) / fused_leaky_relu slope          */
    MN_ACT_TANH = 3,       /* models/networks.py:321,375                          */
    MN_ACT_GELU = 4,       /* exact erf GELU, models/textvit_arch.py:47,87        */
    MN_ACT_SIGMOID = 5,    /* models/textvit_arch.py:50                           */
    MN_ACT_RSQRT_EPS = 6   /* rsqrt(v + 1e-8): demodulation, networks.py:286      */
} mn_act;

typedef enum {
    MN_PREC_FP32_SIMT = 0,   /* CUDA-core fp32 FMA implicit GEMM                       */
    MN_PREC_F16X3_TC = 1,    /* wgmma fp16, fp16 hi/lo split, 3 MMAs (~fp32)            */
    MN_PREC_BF16X3_TC = 2,   /* wgmma bf16, bf16 hi/lo split, 3 MMAs                    */
    MN_PREC_F16X1_TC = 3     /* wgmma single pass fp16 (NOT parity grade)              */
} mn_precision;

const char* mn_last_error(void);
int mn_version(void);
/* Cap the number of CTAs the persistent tensor-core kernels launch (0 = one per SM).  Leaving a few SMs free lets NCCL's
 * copy kernels run beside them, so an asynchronous all-gather overlaps the next chunk of compute.  Returns the old value. */
int mn_set_max_ctas(int n);

/* Programmatic dependent launch (every kernel is launched with the programmatic-stream-serialization attribute so that its
 * launch overlaps the previous kernel's tail).  mn_set_pdl(0) turns the attribute off process-wide (returns the old
 * setting); the environment variable MN_PDL=0 does the same at load time. */
int mn_set_pdl(int on);
/* 1 when the current device is compute capability 9.x (wgmma/TMA paths usable). */
int mn_device_is_sm90(void);

/* ------------------------------------------------------------------------------------
 * Implicit-GEMM convolution / linear layer.
 *
 * Replaces: every F.conv2d / nn.Conv2d / nn.Linear / F.linear on the path
 *   models/resnet.py:5-8,36,21-30 ; models/networks.py:294,299 (ModulatedConv2d, via the
 *   shared-weight reformulation y = demod[n,o] * sum_k W[o,k] * (s[n,c(k)] * x[n,k]) ),
 *   :336-408,501-505 (TSPSRNet convs, spectral norm folded at pack time),
 *   models/textvit_arch.py:34,42,46-51,57,61,86-88,101-102 (Linear = 1x1 conv on [M,1,1,K]),
 *   and the fused bias+leaky-relu of basicsr fused_act (networks.py:195,244-245).
 *
 *   y[n,oy,ox,o] = act( out_scale[n,o] * sum_{ky,kx,c} x[n,oy*sh+ky-ph,ox*sw+kx-pw,c] * w[(ky*KW+kx)*Cin+c][o]
 *                       + bias[o] + residual[n,oy,ox,o] ) * act_gain
 *   y2[n,oy,ox,o] = y[n,oy,ox,o] * y2_scale[n,o]      (optional second output: the
 *                   pre-modulated operand of the next modulated conv)
 *   Columns ox >= valid_w[n] are written as 0 when valid_w != NULL (ragged per-character
 *   windows keep their zero padding, models/networks.py:442-447).
 * ------------------------------------------------------------------------------------ */
typedef struct {
    const float* x;  int N, H, W, Cin, x_cs;
    const float* w;  int KH, KW, stride_h, stride_w, pad_h, pad_w, Cout;   /* w: [KH*KW*Cin][Cout] */
    float* y;        int y_cs;                 /* may be NULL when only y2 is wanted           */
    const float* bias;                         /* [Cout] or NULL                               */
    const float* out_scale; int out_scale_stride; /* [N][stride] (stride 0 -> Cout) or NULL      */
    const float* residual; int res_cs;         /* NHWC [N,OH,OW,res_cs] or NULL                */
    int res_broadcast_n;                       /* 1: residual has no batch dim (positional emb) */
    int act;  float act_gain;
    float* y2;       int y2_cs;  const float* y2_scale; int y2_scale_stride;   /* optional      */
    const int32_t* valid_w;                    /* [N] or NULL                                   */
    float* workspace; int64_t workspace_bytes; /* split-K partial sums; may be NULL (no split)  */
    int split_k;                               /* 0 = choose automatically, 1 = never split     */
    int precision;                             /* mn_precision                                  */
    /* tensor-core precisions only: weights pre-split by mn_conv_pack_weights_tc()                */
    const void* w_tc_hi; const void* w_tc_lo;  /* 16-bit [KH*KW][Cout][Cin] (K-major)            */
    const float* w_tc_scale;                   /* the 2-float scale record written by the packer */
    /* optional input transform fused into the halo-tiled tensor-core kernel's operand-split stage: a request, which
     * mn_conv2d_plan reports as gn_fused (dropped by every other kernel and by tiles of several samples):
     *   x' = swish( (x - mean[n,g]) * rstd[n,g] * gamma[c] + beta[c] ),  zero outside the image / beyond valid_w[n]
     * i.e. GroupNorm(32 channels per group) + swish of models/networks.py:508-512 applied while the A operand is built (its own
     * kernel instantiation: four lanes per halo row, constants in registers).  Needs OH*OW >= 128 (one sample per 128-pixel tile);
     * the sigmoid uses ex2.approx / rcp.approx (~2e-7 relative).  */
    const float* gn_mean_rstd;                 /* [N][Cin/32][2] from mn_groupnorm_stats, or NULL                          */
    const float* gn_gamma; const float* gn_beta;   /* [Cin]                                                                */
    int gn_swish;
    /* fp16-range management of the tensor-core precisions (the fp16 hi/lo split needs |x * x_scale| < 65504; the reference
     * computes in fp32, models/networks.py:294,299 / F.conv2d everywhere, and has no such limit):
     *   x_scale   power of two applied to the A operand before it is split and undone exactly in the epilogue (0 -> 1);
     *   x_absmax  optional DEVICE float: atomic max of |x * x_scale| over every element the kernel consumed (calibration);
     *   range_flag optional int32 the kernel STORES range_tag into when an operand element left the representable range
     *             (fp16 modes: |x * x_scale| >= 65504; every mode: Inf).  May point to pinned host memory (plain store). */
    float x_scale;
    float* x_absmax;
    int32_t* range_flag;
    int32_t range_tag;
    /* Per-sample base pointers of the SECOND output: sample n's [OH][OW][y2_cs] block is written at y2_ptrs[n] instead of
     * y2 + n*OH*OW*y2_cs (y2 must still be non-NULL to enable the output; it is not dereferenced).  The pointers may address the
     * memory of PEER GPUs (NVLink-mapped symmetric memory): the epilogue's stores then deliver every character's prior features
     * straight into the buffer of the rank that runs that character's SR decoder, tile by tile, while the MMAs of the next tile run
     * -- the exchange of the character-sharded path (reference consumer: models/networks.py:442-445, 475-478) without a separate
     * collective.  halo-tiled tensor-core kernel only, layers whose samples are whole pixel tiles (OH*OW >= 128), no split-K. */
    float* const* y2_ptrs;
    /* GroupNorm statistics of the OUTPUT accumulated by the epilogue (models/networks.py:508-512: the tensor this convolution writes
     * is normalised next): per (sample, group of 32 output channels) sum and sum of squares of y, fp32 partials per warp and tile
     * added into [N][Cout/32][2] doubles with atomics (the caller zeroes the buffer; columns beyond valid_w contribute 0).
     * halo-tiled tensor-core kernel, whole-tile samples (OH*OW >= 128), no split-K: a request, like gn_mean_rstd, which
     * mn_conv2d_plan reports as gn_stats_out; finish with mn_groupnorm_finalize. */
    double* gn_stats_out;
} mn_conv_params;

int mn_conv2d_nhwc(const mn_conv_params* p, void* stream);

typedef enum {
    MN_CONV_KERNEL_SMALL = 0,   /* direct 3x3 kernel for Cout <= 4 (fp32)                       */
    MN_CONV_KERNEL_SIMT = 1,    /* fp32 CUDA-core implicit GEMM (+ split-K reduce)              */
    MN_CONV_KERNEL_TC1 = 2,     /* tensor-core per-tap tiling                                   */
    MN_CONV_KERNEL_TC2 = 3      /* tensor-core halo tiling (+ split-K reduce)                   */
} mn_conv_kernel;

/* What mn_conv2d_nhwc would launch for *p, filled in without launching anything or reading memory. */
typedef struct {
    int kernel;                 /* mn_conv_kernel                                               */
    int precision;              /* the precision that runs (MN_PREC_FP32_SIMT for small / simt) */
    int nt;                     /* tensor-core kernels: output channels per work item (64/128)  */
    int TN, TH, TW;             /* tensor-core kernels: samples x rows x columns of a pixel tile */
    int splits;                 /* split-K factor of the simt or halo-tiled kernel (1: none)    */
    int gn_fused;               /* 1: the kernel applies the gn_mean_rstd input transform       */
    int gn_stats_out;           /* 1: the kernel accumulates the gn_stats_out statistics        */
    /* tensor-core kernels only (0 for the fp32 kernels): */
    int cs;                     /* CTAs per cluster (2: the weight tile is multicast to a pair)  */
    int m_tiles;                /* pixel tiles                                                  */
    int work_items;             /* (pixel tiles / cs, rounded up) x (Cout / nt) x splits         */
    int hstages, bstages;       /* depths of the A-tile and weight-tile rings                   */
    int ctas;                   /* grid of the launch under the current mn_set_max_ctas cap      */
} mn_conv_plan;
/* The one dispatch decision: MN_OK and *out filled in, or the status and message mn_conv2d_nhwc would return for *p.
 * A tensor-core precision picks the halo tiling when it runs the geometry, else the per-tap tiling; it fails
 * (MN_ERR_UNSUPPORTED, mn_last_error() says why) when neither does.  The optional requests gn_mean_rstd and gn_stats_out
 * never make it fail: where they cannot be honoured (fp32 kernels, per-tap tiling, tiles of several samples; the halo
 * tiling's Cin / Cout % 64 covers the groups of 32 channels) they are dropped -- gn_fused / gn_stats_out = 0 -- and the
 * problem is planned as if they had never been made (split-K allowed again).  Only their NULL-ness is read.
 * mn_conv2d_nhwc refuses a request its plan drops.  y2_ptrs is no request: without the halo tiling the plan fails. */
int mn_conv2d_plan(const mn_conv_params* p, mn_conv_plan* out);
/* Split fp32 weights w:[taps*Cin][Cout] (the layout mn_conv2d_nhwc takes) into hi/lo 16-bit planes
 * [taps][Cout][Cin], pre-scaled by a power of two so the lo plane stays in the fp16 normal range.
 * hi, lo: taps*Cin*Cout 16-bit elements each; scale2: 2 floats {abs-max, 2^-S}. */
int mn_conv_pack_weights_tc(const float* w, int taps, int Cin, int Cout, int precision, void* hi, void* lo,
                            float* scale2, void* stream);

/* ------------------------------------------------------------------------------------
 * Generator (TSPGAN) operators
 * ------------------------------------------------------------------------------------ */
/* PixelNorm, models/networks.py:170-171:  y = x * rsqrt(mean(x^2, dim=1) + 1e-8), x:[N][C]. */
int mn_pixelnorm(const float* x, float* y, int N, int C, void* stream);

/* SelectText (models/networks.py:205-215) fused with the first conv's input modulation:
 *   out[n, yy, l*4+xx, c] = emb[labels[n*L+l]][c] * s[n*s_stride + c],   yy,xx in [0,4)
 * labels are int64 on the DEVICE and must already be range-checked by the host. */
int mn_select_text(const float* emb, const int64_t* labels, const float* s, int s_stride,
                   float* out, int N, int L, int C, void* stream);

/* Device-side range check of the character labels (the reference fails on the empty embedding slice at
 * models/networks.py:211): clamped[i] = clamp(labels[i], 0, classes-1); bit 0 of *err is raised when any label was out
 * of range.  For callers that must not touch the host between launches (CUDA-graph capture, SURVEY 8f n1). */
int mn_check_labels(const int64_t* labels, int64_t* clamped, int n, int classes, int32_t* err, void* stream);

/* Demodulation factors, models/networks.py:284-287 restated on the shared weight:
 *   demod[n][o] = rsqrt( sum_c s[n][c]^2 * wsq[c][o] + 1e-8 ),
 *   wsq[c][o] = scale^2 * sum_{ky,kx} W[o][c][ky][kx]^2 (packed once at load time). */
int mn_demod(const float* s, int s_stride, const float* wsq, float* demod, int N, int Cin, int Cout, void* stream);

/* All demodulation tables of one generator pass in a single launch.  descs: DEVICE array of n_layers records;
 * demod of layer l lands in out_all[n*out_stride + out_off .. + cout). */
typedef struct {
    const float* wsq;   /* [cin][cout] */
    int32_t s_off;      /* column offset of this layer's style inside s_all rows */
    int32_t cin, cout;
    int32_t out_off;
} mn_demod_desc;
int mn_demod_batched(const float* s_all, int s_stride, const mn_demod_desc* descs, int n_layers, int max_cout,
                     float* out_all, int out_stride, int N, void* stream);

/* y = (bilinear x2 upsample, align_corners=False, of x) * s[n][c]   (up=1)
 * y = x * s[n][c]                                                   (up=0);  s may be NULL.
 * Replaces nn.Upsample / F.interpolate(scale_factor=2, mode='bilinear') at
 * models/networks.py:268,293,318,360,370,415-416 (and the per-sample style multiply of :284). */
int mn_resample_modulate(const float* x, int x_cs, float* y, int y_cs, const float* s, int s_stride,
                         int N, int H, int W, int C, int up, void* stream);
/* Ragged-width bilinear x2 of the SR decoder (models/networks.py:360,370,415-416 -- the trunk's two up-samples, conv_up.0 and
 * conv_final.2 -- for a batch whose lines have their own widths): sample n is the first valid_w[n] <= W columns of its W-wide
 * rows.  The source column clamps at valid_w[n]-1 (the right edge of that line's own tensor in the reference) instead of W-1;
 * output columns >= 2*valid_w[n] of the [N, 2H, 2W, C] output are written as 0.  s (may be NULL; 16B aligned, s_stride % 4 == 0)
 * is the per-sample channel scale of mn_resample_modulate.  Each sample equals mn_resample_modulate(up=1) run on it alone at its
 * exact width, bit for bit. */
int mn_resample_modulate_ragged(const float* x, int x_cs, float* y, int y_cs, const float* s, int s_stride,
                                const int32_t* valid_w, int N, int H, int W, int C, void* stream);

/* ToRGB, models/networks.py:313-321: 1x1 modulated conv to 3 channels WITHOUT demodulation
 * + bias + bilinear-x2(skip) + tanh.
 *   out[n,p,o] = tanh( sum_c x[n,p,c]*s[n][c]*w[o][c] + bias[o] + up2(skip)[n,p,o] )
 * w:[3][C] already multiplied by 1/sqrt(C); skip:[N,H/2,W/2,3] or NULL; out:[N,H,W,3]. */
int mn_torgb(const float* x, int x_cs, const float* s, int s_stride, const float* w, const float* bias,
             const float* skip, float* out, int N, int H, int W, int C, void* stream);

/* ------------------------------------------------------------------------------------
 * SR decoder (TSPSRNet) operators
 * ------------------------------------------------------------------------------------ */
/* GroupNorm(32 channels/group, eps) + optional swish, models/networks.py:487-493,508-512.
 * Statistics run over H x valid_w[n] pixels per sample (valid_w NULL -> W); columns beyond
 * valid_w[n] are written as 0.  stats_ws: >= N*(C/cpg)*3 doubles of scratch. */
int mn_groupnorm_swish(const float* x, int x_cs, float* y, int y_cs, const float* gamma, const float* beta,
                       int N, int H, int W, int C, int cpg, float eps, int swish,
                       const int32_t* valid_w, double* stats_ws, void* stream);
/* The two halves of mn_groupnorm_swish, for fusing the normalisation into the consuming convolution:
 * statistics -> mean_rstd [N][C/cpg][2] fp32 (stats_ws: >= 2*N*(C/cpg) doubles), and the elementwise apply. */
int mn_groupnorm_stats(const float* x, int x_cs, int N, int H, int W, int C, int cpg, float eps,
                       const int32_t* valid_w, double* stats_ws, float* mean_rstd, void* stream);
/* Second half of mn_groupnorm_stats alone: sums [N][C/cpg][2] (sum, sum of squares; fp64) -> mean_rstd.  Used when the PRODUCING
 * convolution accumulated the sums in its epilogue (mn_conv_params.gn_stats_out): no separate read pass over the tensor. */
int mn_groupnorm_finalize(const double* stats_ws, int N, int H, int W, int C, int cpg, float eps, const int32_t* valid_w,
                          float* mean_rstd, void* stream);
int mn_groupnorm_apply(const float* x, int x_cs, float* y, int y_cs, const float* gamma, const float* beta,
                       const float* mean_rstd, int N, int H, int W, int C, int cpg, int swish,
                       const int32_t* valid_w, void* stream);

/* Per-character window table entry (host computes the integers bit-exactly like
 * models/networks.py:426-441 / :460-474). */
typedef struct {
    int32_t line;     /* b: which LR line the character belongs to                          */
    int32_t x1, x2;   /* window [x1,x2) in the line feature map                              */
    int32_t y1;       /* first column of the centred crop of the character prior            */
} mn_window;

/* AdaIN + concat, models/networks.py:442-445,518-533:
 *   out[i,:,:wv,0:C]  = (prior[i,:,y1:y1+wv,:] - mean_p)/std_p * std_l + mean_l
 *   out[i,:,:wv,C:2C] = feat[line,:,x1:x2,:]
 *   out[i,:,wv:,:]    = 0                        (wv = x2-x1, slot width = Wp)
 * std uses the unbiased variance + 1e-5.  prior:[Nc,H,Wp,C], feat:[B,H,W,C], out:[Nc,H,Wp,2C].
 * stats_ws: >= 6*Nc*C doubles of scratch. */
int mn_adain_concat(const float* prior, int prior_cs, const float* feat, int feat_cs, const mn_window* win,
                    float* out, int Nc, int H, int Wp, int W, int C, double* stats_ws, void* stream);

/* Write-back of the per-character modulation, models/networks.py:448-449 / :481-482:
 *   out[b,:,x,:] = feat + (feat*scale[i,:,x-x1,:] + shift[i,:,x-x1,:])  if column x of line b is
 *   owned by character i = owner[b*W + x] (the LAST character in program order whose window
 *   covers x; -1: none -> out = feat).  scale/shift:[Nc,H,Wp,C]. */
int mn_window_scatter(const float* feat, int feat_cs, const float* scale, const float* shift,
                      const int32_t* owner, const mn_window* win, float* out, int out_cs,
                      int B, int H, int W, int Wp, int C, void* stream);

/* The window integers of models/networks.py:426-441 / :460-474 computed on the device (no host round trip):
 *   center = (int)(locs[b*locs_stride + 2c] * W)   (fp32 multiply, truncation), x1 = max(center-half,0) as coded,
 *   x2 = min(center+half, W), y1 = half - (x2-x1)/2; valid[i] = x2-x1; owner[b*W+x] = last character whose window
 *   covers column x, else -1.  Characters of line b are win[line_first[b] .. line_first[b+1]) (device int32[B+1]);
 *   max_chars >= the longest line.  An empty window (reference: error at networks.py:443) raises bit 1 of *err and
 *   becomes a zero-width window. */
int mn_char_windows(const float* locs, int locs_stride, const int32_t* line_first, int B, int max_chars, int W, int half,
                    mn_window* win, int32_t* valid, int32_t* owner, int32_t* err, void* stream);
/* mn_char_windows for lines of their own widths (device int32 line_w[B], each <= W), models/networks.py:426-441 / :460-474 run on
 * each line's own tensor: center = (int)(locs[b*locs_stride + 2c] * line_w[b]), x2 = min(center+half, line_w[b]); owner[b*W+x]
 * is filled for x < line_w[b] and -1 beyond.  Error bits as in mn_char_windows.  A width larger than W is not reported: it is
 * clamped to W (the caller guarantees line_w[b] <= W). */
int mn_char_windows_ragged(const float* locs, int locs_stride, const int32_t* line_first, const int32_t* line_w, int B, int max_chars,
                           int W, int half, mn_window* win, int32_t* valid, int32_t* owner, int32_t* err, void* stream);

/* The reference module's standalone helper functions on NCHW-contiguous tensors (rows = B*C, len = H*W); the hot path uses
 * the fused NHWC kernels above.
 *   mn_swish         x * sigmoid(x)                                                models/networks.py:492-493
 *   mn_row_mean_std  mean, sqrt(unbiased var + eps) of every row                   calc_mean_std_4D, :518-525
 *   mn_adain_rows    (prior - prior_mean)/prior_std * lq_std + lq_mean per row     adaptive_instance_normalization, :528-533 */
int mn_swish(const float* x, float* y, long long n, void* stream);
int mn_row_mean_std(const float* x, float* mean, float* stdv, int rows, int len, float eps, void* stream);
int mn_adain_rows(const float* prior, const float* prior_mean, const float* prior_std, const float* lq_mean,
                  const float* lq_std, float* out, int rows, int len, void* stream);

/* ------------------------------------------------------------------------------------
 * TextViT operators
 * ------------------------------------------------------------------------------------ */
/* nn.LayerNorm over the last dim (eps 1e-5), models/textvit_arch.py:41,46,53,58,85,99. */
int mn_layernorm(const float* x, float* y, const float* gamma, const float* beta, int rows, int dim,
                 float eps, void* stream);

/* nn.Linear for M <= 64 rows (the tokens of one text line), models/textvit_arch.py:42,46-51,57,61,86-88,101-102:
 *   y[M][N] = act(x[M][K] w[K][N] + bias[N] + residual[M][N]) * gain, K % 32 == 0, N % 16 == 0.  (Note: residual is added
 *   BEFORE the activation, like mn_conv2d_nhwc.) */
int mn_linear_small_m(const float* x, const float* w, const float* bias, const float* residual, float* y,
                      int M, int K, int N, int act, float gain, void* stream);

/* The same layer over a GATHERED x and `batches` independent row blocks (text lines): element (r, k) of batch z is
 *   x[z*x_batch_stride + r*x_row_stride + (k / x_seg_len)*x_seg_stride + k % x_seg_len]      (x_seg_len % 32 == 0),
 * y is dense [batches][M][N]; residual (optional) is [M][N] per batch at residual + z*res_batch_stride (0 = shared).
 * This is the TextViT patch embedding (models/textvit_arch.py:33-36: Rearrange 'b c (h p1) (w p2) -> b h w (p1 p2 c)' +
 * Linear(32768, 512) + positional embedding) reading the NHWC ResNet feature map [B,8,512,512] in place:
 *   M = 64 tokens, K = 8*8*512, x_row_stride = 8*512, x_seg_len = 8*512, x_seg_stride = 512*512, x_batch_stride = 8*512*512. */
int mn_linear_small_m_ex(const float* x, long long x_row_stride, long long x_batch_stride, int x_seg_len, long long x_seg_stride,
                         const float* w, const float* bias, const float* residual, long long res_batch_stride, float* y,
                         int batches, int M, int K, int N, int act, float gain, void* stream);

/* mn_linear_small_m_ex with a caller-owned scratch: deep-K layers (the patch embedding, K = 32768) are additionally split into
 * outer K slices whose raw partial tiles go to `workspace` (>= slices*batches*M*N floats are used when available) and are added
 * in slice order by a second kernel that runs the bias / residual / activation epilogue -- deterministic, no atomics.
 * workspace may be NULL (then identical to mn_linear_small_m_ex). */
int mn_linear_small_m_ws(const float* x, long long x_row_stride, long long x_batch_stride, int x_seg_len, long long x_seg_stride,
                         const float* w, const float* bias, const float* residual, long long res_batch_stride, float* y,
                         int batches, int M, int K, int N, int act, float gain, float* workspace, long long workspace_bytes,
                         void* stream);

/* LayerNorm over the TOKEN axis followed by Linear(T -> To) over the token axis, i.e. the
 * `x.permute(0,2,1)` -> LayerNorm(T) -> Linear -> permute(0,2,1) idiom at
 * models/textvit_arch.py:154 (T=64 -> 16) and :72 (64 -> 1).  x:[B,T,D] -> out:[B,To,D]. */
int mn_token_mix(const float* x, const float* gamma, const float* beta, const float* w, const float* bias,
                 float* out, int B, int T, int To, int D, float eps, void* stream);

/* Fused multi-head attention, models/textvit_arch.py:104-111: softmax(q k^T * scale) v for every
 * (batch, head) in one CTA.  qkv:[B,S,3*heads*dh] (q|k|v thirds, head-major inside), out:[B,S,heads*dh].
 * S <= 64, dh == 64. */
int mn_attention(const float* qkv, float* out, int B, int S, int heads, int dh, float scale, void* stream);

/* ------------------------------------------------------------------------------------
 * Layout conversion at the module boundary (the reference API is NCHW, models/networks.py:42,61,411)
 * ------------------------------------------------------------------------------------ */
int mn_nchw_to_nhwc(const float* x, float* y, int N, int C, int H, int W, int y_cs, void* stream);
int mn_nhwc_to_nchw(const float* x, int x_cs, float* y, int N, int C, int H, int W, void* stream);

/* ------------------------------------------------------------------------------------
 * Script pre/post-processing on the device (SURVEY 8f n2; the reference does this on the host with cv2 / torchvision)
 * ------------------------------------------------------------------------------------ */
/* test_sr.py:98-111:  LQ = cv2.resize(img, (0,0), fx, fy, INTER_CUBIC)  (8-bit HWC image, OpenCV's own algorithm, bit-exact:
 * see csrc/image_ops.cu), pasted into a zero out_h x out_w canvas, ToTensor, Normalize((.5,.5,.5),(.5,.5,.5)).
 *   img:[h][w][cn] uint8 (device), dh = round_half_even(h*fy), dw = round_half_even(w*fx) (computed by the caller, as cv::resize
 *   does), lq:[cn][out_h][out_w] fp32, lq_u8 (optional): the resized bytes [dh][dw][cn].  Fails when dw > out_w (the script skips
 *   such images, test_sr.py:107-109). */
int mn_preprocess_lq_u8(const uint8_t* img, int h, int w, int cn, double fx, double fy, int dh, int dw,
                        float* lq, uint8_t* lq_u8, int out_h, int out_w, void* stream);

/* test_sr.py:198-201 (+ the uint8 rounding of cv2.imwrite, :231):
 *   out[b][y][x][C-1-c] = saturate_u8(round_half_even(clip(sr[b,c,y,x]*0.5 + 0.5, 0, 1) * 255)).
 * sr is addressed through element strides so that the channels_last view the SR module returns is read in place. */
int mn_postprocess_sr_u8(const float* sr, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                         uint8_t* out, int B, int C, int H, int W, void* stream);

/* Text lines wider than the canvas (and batches of lines of any width): test_sr.py:98-111 applied to many crops in one launch.
 * Each crop is an image of its own: `img` points at row 0, first column of the crop inside a larger uint8 [.][.][cn] image whose
 * rows are `row_pitch` bytes apart; the crop is h x w pixels and the cubic taps replicate ITS border, never reading outside it
 * (= cv2.resize(img[:, a:b], (0,0), fx, fy, INTER_CUBIC), what a user who crops by hand gets).  dh = round_half_even(h*fy),
 * dw = round_half_even(w*fx) <= out_w.  crops: DEVICE array of n records (the caller validates them before copying them over).
 * lq: [n][cn][out_h][out_w] fp32, crop i bit-identical to mn_preprocess_lq_u8 on a contiguous copy of crop i. */
typedef struct {
    const uint8_t* img;
    int64_t row_pitch;          /* bytes between rows of the source image */
    int h, w, cn;
    double fx, fy;
    int dh, dw;
} mn_lq_crop;
int mn_preprocess_lq_u8_batched(const mn_lq_crop* crops, int n, int cn, float* lq, int out_h, int out_w, void* stream);

/* test_sr.py:198-201 (the bytes of mn_postprocess_sr_u8, channel flip included) for column ranges of several SR lines, written
 * into several destination images in one launch -- the stitch of a line restored crop by crop:
 *   dst[y*dst_pitch + x*C + (C-1-c)] = u8(sr[line, c, y, src_x0 + x]),   y < H, x < width, src_x0 + width <= W.
 * sr is addressed through element strides (the channels_last view TSPSRNet returns is read in place).  pieces: DEVICE array of
 * n_pieces records (validated by the caller); max_width >= every piece's width. */
typedef struct {
    int32_t line, src_x0, width;
    uint8_t* dst;               /* row 0, first column of the piece inside its image */
    int64_t dst_pitch;          /* bytes between rows of the destination image */
} mn_sr_piece;
int mn_postprocess_sr_u8_pieces(const float* sr, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                                int C, int H, int W, const mn_sr_piece* pieces, int n_pieces, int max_width, void* stream);

/* The figure test_sr.py writes per image (:206-231, cv2.imwrite of vstack(ShowLQ[:,:,::-1], ShowLocs[:,:,::-1], ShowSR, prior)),
 * panels 1, 2 and 4 for a batch of images in one launch (DESIGN.md section 7b).  The figure is uint8 [512][W][3]; every panel is
 * computed at the ShowLQ width S = round_half_even(w*128/h) and cropped to W <= S:
 *   rows   0-127  ShowLQ[:, :, ::-1], ShowLQ = cv2.resize(img, (0,0), fx=128/h, fy=128/h, INTER_CUBIC) (:98; OpenCV's own cubic,
 *                 the arithmetic of mn_preprocess_lq_u8);
 *   rows 128-255  ShowLocs[:, :, ::-1] (:214-230): ShowLQ with (255, 0, 0) in rows 0-63 of the `n_top` marker column ranges and
 *                 (0, 0, 255) in rows 64-127 of the `n_bot` ranges -- [start, stop) pairs, top ranges first, computed by the caller
 *                 with the script's Python slice rules on a width-S row;
 *   rows 256-383  not written (ShowSR: mn_postprocess_sr_u8_pieces with dst at row 256);
 *   rows 384-511  prior (:206-211, not flipped): cv2.resize(hstack(prior_k*0.5+0.5 for k < n_chars), (S, 128), INTER_LINEAR)*255,
 *                 OpenCV's float linear resize, then cvRound with saturation (cv2.imwrite).  Each character's [3][128][128] fp32
 *                 prior is read in place through element strides (the channels_last generator output).
 * images: DEVICE array of n_images records; marks and priors are DEVICE arrays (validated by the caller); max_width >= every W. */
typedef struct {
    const float* img;           /* [3][128][128] generator image in [-1, 1] */
    int64_t stride_c, stride_h, stride_w;
} mn_figure_prior;
typedef struct {
    const uint8_t* img;         /* row 0 of the h x w x 3 source image */
    int64_t row_pitch;          /* bytes between rows of the source image */
    uint8_t* fig;               /* row 0 of the [512][W][3] figure */
    int64_t fig_pitch;          /* bytes between rows of the figure */
    const int32_t* marks;       /* n_top + n_bot column ranges [start, stop), 0 <= start < stop <= S */
    const mn_figure_prior* priors;
    int32_t h, w, S, W, n_top, n_bot, n_chars;
} mn_figure_image;
int mn_figure_u8(const mn_figure_image* images, int n_images, int max_width, void* stream);

/* Characters predicted by TextContextEncoderV2 on detection windows (DESIGN.md section 7b, "Predicted characters"), one CTA per
 * encoder row b < n_rows, the record rows[b] telling where the window lies and where its result goes:
 *   1. idx[t] = argmax over the C classes of logits[b][t] (t < T <= 64), torch.max(dim) semantics: the first maximal index wins,
 *      a NaN is larger than any number (the first NaN wins);
 *   2. CTC collapse (test_w.py:34-40): keep t iff (t == 0 || idx[t] != idx[t-1]) && idx[t] < n_alphabet; the first
 *      MN_PRED_SLOTS kept indices are the decoded characters, character j taking box slot j;
 *   3. box: l = locs_lr[b][2j], r = locs_lr[b][2j+1]; c = (r+l)/2, hw = (r-l)/2 in fp32 (tspgan_model.py:331-337); in fp64
 *      x1 = a + (c - hw)*scale, x2 = a + (c + hw)*scale, each operation rounded on its own (no contraction);
 *   4. core: the character is kept iff lo <= (x1+x2)/2 < hi (a NaN centre is never kept).
 * out receives the kept characters compacted in decode order (label, x1, x2; unused slots label -1, x1 = x2 = 0), n_kept and
 * n_decoded (the decoded count before the core test).  logits: fp32 rows `logits_row_stride` elements apart, each [T][C] dense,
 * C % 4 == 0 and 16-byte aligned; locs_lr: fp32 rows `locs_row_stride` apart, 2*MN_PRED_SLOTS values each.  rows: DEVICE
 * array (validated by the caller). */
#define MN_PRED_SLOTS 16
typedef struct {
    double x1[MN_PRED_SLOTS];
    double x2[MN_PRED_SLOTS];
    int32_t label[MN_PRED_SLOTS];
    int32_t n_kept, n_decoded;
} mn_char_pred;
typedef struct {
    double a;                   /* source column of the window's first column */
    double scale;               /* source columns per unit of canvas width: 16*h for a 32x512 canvas */
    double lo, hi;              /* the window's core [lo, hi) in source columns (+-inf at the line's ends) */
    mn_char_pred* out;
} mn_pred_row;
int mn_decode_predictions(const float* logits, long long logits_row_stride, int T, int C, const float* locs_lr, long long locs_row_stride,
                          const mn_pred_row* rows, int n_rows, int n_alphabet, void* stream);
/* Every character the encoder reads on a line that fits the canvas (test_w.py:34-40, 99: all of clear_labels(logits[0]), no cap):
 * steps 1-2 of mn_decode_predictions (the same argmax and CTC collapse) over all T <= 64 timesteps of row b < n_rows of logits,
 * one CTA per row.  out[b] receives the count n and the labels in timestep order (unused slots -1); the first
 * min(n, MN_PRED_SLOTS) labels are the characters mn_decode_predictions decodes on the same row. */
#define MN_LABEL_SLOTS 64
typedef struct {
    int32_t n;
    int32_t label[MN_LABEL_SLOTS];
} mn_label_row;
int mn_decode_labels(const float* logits, long long logits_row_stride, int T, int C, mn_label_row* out, int n_rows, int n_alphabet,
                     void* stream);

/* Font-style interpolation (test_w.py:107, new_w = w1*scale + w2*(1-scale)) for every style row of a sweep in one launch:
 *   out[r*out_stride + d] = fl(fl(w[w1*w_stride + d] * s) + fl(w[w2*w_stride + d] * t)),   d < dim,
 * each multiply and the add rounded on its own (no FMA): the bits of torch's fp32 ``w1 * s + w2 * (1 - s)`` for s = float32(scale)
 * and t = float32(1 - scale), 1 - scale computed in double.  rows: DEVICE array of n_rows records (indices validated by the
 * caller); w: the encoder style rows. */
typedef struct {
    int32_t w1, w2;             /* rows of w: the content character's style and the donor's */
    float s, t;
} mn_lerp_row;
int mn_style_lerp(const float* w, int w_stride, const mn_lerp_row* rows, int n_rows, int dim, float* out, int out_stride, void* stream);

/* The 8-bit strip test_w.py writes per style (:109-114, cv2.imwrite(hstack(prior*0.5+0.5)*255.0)), tile by tile: generator image
 * n < n_rows (fp32 [3][128][128] in [-1, 1], addressed through element strides: the channels_last output is read in place) goes
 * to the 128 x 128 x 3 tile at tiles[n].dst, rows tiles[n].dst_pitch bytes apart:
 *   dst[y*pitch + x*3 + c] = saturate_u8(cvRound(fl(fl(fl(p*0.5) + 0.5) * 255))),   not channel-flipped,
 * the arithmetic of panel 4 of mn_figure_u8 at its identity width.  tiles: DEVICE array (validated by the caller). */
typedef struct {
    uint8_t* dst;               /* row 0, first column of the tile */
    int64_t dst_pitch;          /* bytes between rows of the strip */
} mn_prior_tile;
int mn_prior_tiles_u8(const float* priors, long long stride_n, long long stride_c, long long stride_h, long long stride_w,
                      const mn_prior_tile* tiles, int n_rows, void* stream);

/* Text regions in whole images (DESIGN.md section 7b, "Text regions in whole images").
 * OpenCV's own 8-bit INTER_CUBIC resize (the arithmetic of mn_preprocess_lq_u8) of n images in one launch, blockIdx.y = image:
 * images[i].dst [dh][dw][cn] = cv2.resize(src [h][w][cn], (dw, dh), INTER_CUBIC) computed at scale_x / scale_y (cv::resize's
 * 1/fx, 1/fy: 1/s for the fx = fy = s background, 1/((double)dw/w) for the dsize form).  Pixels are addressed by row and column
 * with 64-bit byte offsets, so a destination may exceed 2^31 bytes.  max_pixels >= every dh*dw.  images: DEVICE array of
 * records (validated by the caller). */
typedef struct {
    const uint8_t* src;         /* row 0 of the source image */
    int64_t src_pitch;          /* bytes between rows of the source image */
    int32_t h, w;
    uint8_t* dst;               /* row 0 of the destination image */
    int64_t dst_pitch;          /* bytes between rows of the destination */
    int32_t dh, dw;
    double scale_x, scale_y;
} mn_resize_image;
int mn_resize_cubic_u8_batched(const mn_resize_image* images, int n, int cn, long long max_pixels, void* stream);

/* The restored regions of whole images composed over their cubic backgrounds, every region of every page in one launch,
 * blockIdx.y = region, one thread per output pixel (X, Y) of its rectangle [x0, x1) x [y0, y1) (output pixels).  P = the cubic
 * resize (mn_resize_cubic_u8_batched's arithmetic, dsize form, split at the rectangle's width) of the region's restored bytes
 * sr [sr_h][sr_w][3] (cv2.imwrite order; channel c of P reads channel 2 - c) onto the rectangle; a = min(1, fl((float)d + 0.5)/F),
 * d the distance to the nearest side not on the page border (a = 1 when F = 0 or every side lies on it); then
 *   page = sat_u8(rint_half_even(fl(fl(a*P) + fl(fl(1 - a)*page)))),   every operation rounded on its own.
 * A pixel is written by exactly one thread: the one of the last region of its chain that contains it, which composes the
 * background through every containing region of the chain in order.  chain: the indices (into `regions`) of every region of the
 * same page whose rectangle meets this one, itself included, increasing.  regions: DEVICE array of records whose chains point
 * into device memory (validated by the caller); max_pixels >= every rectangle's pixel count. */
typedef struct {
    uint8_t* page;              /* row 0 of the page [page_h][page_w][3], holding its background */
    int64_t page_pitch;
    const uint8_t* sr;          /* row 0 of the region's restored bytes */
    int64_t sr_pitch;
    const int32_t* chain;
    int32_t page_h, page_w, sr_h, sr_w;
    int32_t x0, y0, x1, y1;
    int32_t feather, n_chain;
} mn_region;
int mn_composite_regions_u8(const mn_region* regions, int n, long long max_pixels, void* stream);

/* Oriented text regions (DESIGN.md section 7b, "Oriented text regions").
 * cv2.warpAffine(src, M, (dw, dh), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE), OpenCV's own 8-bit path (IPP off), of n
 * images in one launch, blockIdx.y = image, one thread per destination pixel.  m = M row by row: destination pixel (x, y) ->
 * source pixel (m[0] x + m[1] y + m[2], m[3] x + m[4] y + m[5]).  OpenCV's fixed-point coordinates in 1/32 pixel,
 * Xq = (cvRound(fl(fl(m[1] y) + m[2]) * 1024) + 16 + cvRound(fl(m[0] x) * 1024)) >> 5 (fp64, no contraction), then remap's
 * 2-D cubic table (fp32 interpolateCubic at i/32, rint(fl(vy vx) 32768) saturated to int16, the sum's excess moved onto the
 * taps at rows and columns 2..3), the 16 taps with replicated borders and (sum + 2^14) >> 15 saturated.  cv2 keeps the integer
 * source coordinates as int16; with h, w <= 32767 that saturation changes no value, and callers keep every
 * |fixed-point coordinate| below 2^30.  Byte offsets are 64-bit.  max_pixels >= every dh*dw.  images: DEVICE array of records
 * (validated by the caller). */
typedef struct {
    const uint8_t* src;         /* row 0 of the source image */
    int64_t src_pitch;
    int32_t h, w;
    uint8_t* dst;               /* row 0 of the destination image */
    int64_t dst_pitch;
    int32_t dh, dw;
    double m[6];
} mn_warp_image;
int mn_warp_affine_u8_batched(const mn_warp_image* images, int n, int cn, long long max_pixels, void* stream);

/* mn_composite_regions_u8 for pages that hold oriented regions: every region of every page in one launch, blockIdx.y = region,
 * one thread per output pixel of r's rectangle [x0, x1) x [y0, y1).  kind MN_REGION_RECT: r is an mn_region record, composed
 * exactly as mn_composite_regions_u8 composes it (the same device functions).  kind MN_REGION_AFFINE: r's rectangle is the
 * bounding box of the region's footprint; n maps page pixel (X, Y) to pixel indices of the restored bytes T = sr [sr_h][sr_w][3]
 * (cv2.imwrite order), (Xq, Yq) are mn_warp_affine_u8_batched's fixed-point coordinates of (X, Y) under n, and the pixel
 * belongs to the region iff -16 <= Xq < 32 sr_w - 16 and -16 <= Yq < 32 sr_h - 16.  There
 *   P = mn_warp_affine_u8_batched's value of T[..., ::-1] at (Xq, Yq),
 *   u = (Xq + 16)/32, v = (Yq + 16)/32,  a = min(1, fl(min(fl(kx min(u, sr_w - u)), fl(ky min(v, sr_h - v))) / F)), 1 when F = 0,
 * and the blend and the owner rule are mn_composite_regions_u8's; chains index this array. */
#define MN_REGION_RECT 0
#define MN_REGION_AFFINE 1
typedef struct {
    mn_region r;
    int32_t kind;
    float kx, ky;               /* feather slopes of an affine region, output pixels per T pixel across its sides */
    int32_t pad;
    double n[6];                /* affine region: page pixel -> T pixel, row by row */
} mn_region_affine;
int mn_composite_regions_affine_u8(const mn_region_affine* regions, int n, long long max_pixels, void* stream);

/* Perspective text regions (DESIGN.md section 7b, "Perspective text regions").
 * cv2.warpPerspective(src, M, (dw, dh), INTER_CUBIC | WARP_INVERSE_MAP, BORDER_REPLICATE), OpenCV's own 8-bit path (IPP off), of
 * n images in one launch, blockIdx.y = image, one thread per destination pixel.  m = M row by row: destination pixel (x, y) ->
 * source pixel ((m[0] x + m[1] y + m[2]) / w, (m[3] x + m[4] y + m[5]) / w), w = m[6] x + m[7] y + m[8].  OpenCV's fixed-point
 * coordinates in 1/32 pixel (fp64, no contraction), formed in column blocks of bw = min(1024 / min(16, dh), dw): at the block's
 * first column xb, X0 = fl(fl(fl(m[0] xb) + fl(m[1] y)) + m[2]), Y0 and W0 likewise; with x1 = x - xb, W = fl(W0 + fl(m[6] x1)),
 * W = W ? fl(32 / W) : 0, Xq = cvRound(clamp(fl(fl(X0 + fl(m[0] x1)) W), INT_MIN, INT_MAX)) and likewise Yq; then remap's cubic
 * sampler exactly as mn_warp_affine_u8_batched uses it.  Byte offsets are 64-bit.  max_pixels >= every dh*dw.  images: DEVICE
 * array of records (validated by the caller). */
typedef struct {
    const uint8_t* src;         /* row 0 of the source image */
    int64_t src_pitch;
    int32_t h, w;
    uint8_t* dst;               /* row 0 of the destination image */
    int64_t dst_pitch;
    int32_t dh, dw;
    double m[9];
} mn_warp_perspective_image;
int mn_warp_perspective_u8_batched(const mn_warp_perspective_image* images, int n, int cn, long long max_pixels, void* stream);

/* mn_composite_regions_affine_u8 for pages that also hold perspective regions: every region of every page in one launch,
 * blockIdx.y = region.  Kinds MN_REGION_RECT and MN_REGION_AFFINE (n[0..5] = the affine N) are composed exactly as
 * mn_composite_regions_affine_u8 composes them (the same device functions).  Kind MN_REGION_PERSPECTIVE: r's rectangle is the
 * bounding box of the region's footprint; n (3 x 3) maps page pixel (X, Y) to pixel indices of the restored bytes T, (Xq, Yq) are
 * mn_warp_perspective_u8_batched's fixed-point coordinates of (X, Y) under n with the whole page [page_h][page_w] as the
 * destination (its column blocks start at page column 0), and the footprint test, the feather, P, the blend
 * and the owner rule are the affine kind's; chains index this array. */
#define MN_REGION_PERSPECTIVE 2
typedef struct {
    mn_region r;
    int32_t kind;
    float kx, ky;               /* feather slopes of an affine or perspective region */
    int32_t pad;
    double n[9];                /* affine region: n[0..5], page pixel -> T pixel, row by row; perspective region: all nine */
} mn_region_quad;
int mn_composite_regions_quad_u8(const mn_region_quad* regions, int n, long long max_pixels, void* stream);

/* Vertical text columns (DESIGN.md section 7b, "Vertical text columns").  Two integer gathers of 3-byte pixels, each over every
 * column of a call in one launch, blockIdx.y = column, one thread per destination pixel of its [dh][dw][3] destination, those
 * past its dh*dw pixels exit.  Byte offsets are 64-bit; max_pixels >= every dh*dw.  cells points at n_cells records of
 * int32 values built on the host; clamp(v, lo, hi) = min(max(v, lo), hi).  columns: DEVICE array of records whose cell tables
 * point into device memory (validated by the caller: every pixel read lies inside src).
 * mn_vertical_layout_u8_batched: src = the column crop C [h_r][w][3], dst = its line L [H_L][n_cells w][3], cells 3 per cell
 * (c_k, p_k, t_k): L[i][k w + j] = C[c_k + clamp(i - p_k, 0, t_k - 1)][j].
 * mn_vertical_unlayout_u8_batched: src = the restored line T [128][W_T][3], dst = the restored column T_col [H_c][W_c][3],
 * cells 5 per cell (R(c_k), R(p_k), R(p_k + t_k), R(k w_r), min(R((k+1) w_r), W_T)), R(0) = 0: row i belongs to the last cell k
 * with R(c_k) <= i, and T_col[i][j] = T[clamp(R(p_k) + i - R(c_k), R(p_k), R(p_k + t_k) - 1)]
 * [clamp(R(k w_r) + j, R(k w_r), min(R((k+1) w_r), W_T) - 1)]; w is unused. */
typedef struct {
    const uint8_t* src;         /* row 0 of the source: C (layout) or T (unlayout) */
    int64_t src_pitch;
    uint8_t* dst;               /* row 0 of the destination: L (layout) or T_col (unlayout) */
    int64_t dst_pitch;
    const int32_t* cells;       /* the column's cell table */
    int32_t dh, dw;
    int32_t n_cells, w;         /* w: the column's width w_r (layout) */
} mn_vertical_column;
int mn_vertical_layout_u8_batched(const mn_vertical_column* columns, int n, long long max_pixels, void* stream);
int mn_vertical_unlayout_u8_batched(const mn_vertical_column* columns, int n, long long max_pixels, void* stream);

/* Curved text regions (DESIGN.md section 7b, "Curved text regions").  A curve table is an fp64 array built on the host
 * (pipeline.curved_maps): curve[0] = s, the page's scale (unused by the rectify kernel); curve[1 .. k+1] = the column fractions
 * c_0 = 0, ..., c_k = 1; then the top curve's 3k+1 (x, y) points and the bottom curve's 3k+1 points, x and y interleaved.
 * Segment m of a curve is the cubic Bezier of its points 3m .. 3m+3, evaluated by de Casteljau per coordinate with s = 1 - t and
 * three levels of lerps fl(fl(s A) + fl(t B)), every fp64 operation rounded on its own.
 * mn_remap_curved_u8_batched: cv2.remap(src, mapx, mapy, INTER_CUBIC, BORDER_REPLICATE) with fp32 maps, OpenCV's own 8-bit path
 * (IPP off), of n images in one launch, blockIdx.y = image, one thread per destination pixel (x, y) of the [dh][dw][cn] crop
 * (w_r = dw, h_r = dh): a = (x + 0.5)/w_r, b = (y + 0.5)/h_r, m the last segment with c_m <= a (at most k - 1),
 * t = (a - c_m)/(c_{m+1} - c_m), mapx = fl(fl(fl(1 - b) T_m(t).x) + fl(b B_m(t).x)) - 0.5 and mapy likewise (fp64), then
 * Xq = rint(fl32(mapx) 32), Yq = rint(fl32(mapy) 32) and remap's cubic sampler exactly as mn_warp_affine_u8_batched uses it.
 * Callers keep every |map value| below 2^14.  Byte offsets are 64-bit.  max_pixels >= every dh*dw.  images: DEVICE array of
 * records whose curve tables point into device memory (validated by the caller). */
typedef struct {
    const uint8_t* src;         /* row 0 of the source image */
    int64_t src_pitch;
    int32_t h, w;
    uint8_t* dst;               /* row 0 of the destination crop */
    int64_t dst_pitch;
    int32_t dh, dw;
    const double* curve;        /* the region's curve table */
    int32_t n_seg, pad;         /* k */
} mn_remap_curved_image;
int mn_remap_curved_u8_batched(const mn_remap_curved_image* images, int n, int cn, long long max_pixels, void* stream);

/* mn_composite_regions_quad_u8 for pages that also hold curved regions: every region of every page in one launch, blockIdx.y =
 * region.  Kinds MN_REGION_RECT, MN_REGION_AFFINE and MN_REGION_PERSPECTIVE (q as mn_region_quad) are composed exactly as
 * mn_composite_regions_quad_u8 composes them (the same device functions).  Kind MN_REGION_CURVED: q.r's rectangle is the
 * bounding box of the region's control points in page pixels, widened by one pixel; page pixel (X, Y) is the point
 * p = ((X + 0.5)/s, (Y + 0.5)/s).  The segments m = 0 .. k-1 are tried in order, skipping one whose 8 control points' bounding box
 * does not hold p; with d = B_m(t) - T_m(t), r = p - T_m(t) and g(t) = fl(fl(d.x r.y) - fl(d.y r.x)), a segment whose g(0) < 0
 * and g(1) < 0 agree has no root; otherwise 48 bisection steps (mid = fl(0.5 fl(lo + hi)), lo keeps g(0)'s sign), then
 * t* = fl(0.5 fl(lo + hi)) and b = fl(dot(r, d) / dot(d, d)) at t*.  The first segment with 0 <= b <= 1 gives
 * a = c_m + t* (c_{m+1} - c_m), u = fl(a sr_w) - 0.5, v = fl(b sr_h) - 0.5, Xq = rint(fl32(u) 32), Yq = rint(fl32(v) 32); the
 * pixel belongs to the region iff a segment was accepted and -16 <= Xq < 32 sr_w - 16, -16 <= Yq < 32 sr_h - 16.  The feather
 * (q.kx, q.ky), P, the blend and the owner rule are the affine kind's; chains index this array. */
#define MN_REGION_CURVED 3
typedef struct {
    mn_region_quad q;           /* q.kind MN_REGION_CURVED: q.kx, q.ky are its feather slopes and q.n is unused */
    const double* curve;        /* curved region: its curve table */
    int32_t n_seg, pad;         /* curved region: k */
} mn_region_curved;
int mn_composite_regions_curved_u8(const mn_region_curved* regions, int n, long long max_pixels, void* stream);

/* Text blocks split into lines (DESIGN.md section 7b, "Text blocks").  Block i reads the crop C = img[y0:y1][x0:x1] (h x w,
 * three channels, in place through the image's pitch) and runs on the transposed crop when `vertical` is set: L = h, M = w
 * (horizontal) or L = w, M = h (vertical) are the lengths across and along its lines.  mn_find_lines_u8 issues four launches for
 * every block of a call, whatever their number:
 *   1. histogram: hist[g] = #{g(x, y) = g}, g = (c0 + c1 + c2 + 1) / 3, tiles of 32 x 32 pixels, blockIdx.y = block;
 *   2. threshold, one thread per block: t = OpenCV's Otsu threshold of hist (getThreshVal_Otsu_8u's fp64 loop, every operation
 *      rounded on its own, over the n = h w pixels the histogram counts), D = #{g <= t}; ink = polarity, or for MN_INK_AUTO
 *      dark (g <= t) iff 2 D <= n, else light (g > t); t = 0 when n = 0;
 *   3. profile over the tiles: for every index l < L, prof[l] = the ink count, prof[L + l] = M - (the least ink index along the
 *      line), prof[2 L + l] = the largest ink index along the line + 1 (0 where there is no ink);
 *   4. segmentation, one CTA per block: the runs of indices with prof[l] >= m (m = min_ink, default max(1, M / 128)), merged
 *      across gaps <= G (gap, default max(1, Hm / 4), Hm the lower median of the run lengths), those shorter than min_height
 *      dropped (default max(2, Hm' / 3), Hm' the lower median of the merged lengths), each kept line padded by
 *      p = (b - a + 3) / 4 and bounded by its neighbours' midpoints, its extent along the line the ink's over [a, b) padded by p.
 * out->rect[k] is line k in image pixels (x0, y0, x1, y1) in reading order: top to bottom, right to left for a vertical block.
 * out->n_lines is the number of lines, or minus it when it exceeds MN_BLOCK_MAX_LINES (then no rectangle is written).
 * hist, prof and scratch are device memory of 256, 3 L and 2 L + 4 int32 values; work (work_bytes) covers every hist and prof
 * of the call and is zeroed by the call.  max_tiles >= every block's ceil(w / 32) ceil(h / 32).  blocks: DEVICE array
 * (validated by the caller: 1 <= w, h <= 32767, the crop inside its image). */
#define MN_BLOCK_MAX_LINES 256
#define MN_INK_AUTO 0
#define MN_INK_DARK 1
#define MN_INK_LIGHT 2
typedef struct {
    int32_t n_lines;
    int32_t threshold;
    int32_t ink;                /* MN_INK_DARK or MN_INK_LIGHT */
    int32_t pad;
    int32_t rect[MN_BLOCK_MAX_LINES][4];
} mn_block_lines;
typedef struct {
    const uint8_t* img;         /* row 0 of the image */
    int64_t pitch;
    int32_t x0, y0, w, h;       /* the crop */
    int32_t vertical, polarity; /* polarity: MN_INK_AUTO, MN_INK_DARK or MN_INK_LIGHT */
    int32_t min_ink, gap, min_height, pad;   /* 0: the default */
    int32_t* hist;
    int32_t* prof;
    int32_t* scratch;
    mn_block_lines* out;
} mn_text_block;
int mn_find_lines_u8(const mn_text_block* blocks, int n, long long max_tiles, void* work, long long work_bytes, void* stream);

/* Skewed text blocks (DESIGN.md section 7b, "Skewed blocks").  Block i is searched over the angle table table[0 .. n_ang) of
 * fp64 (c, s) pairs uploaded by the host (a given angle is a one-entry table; no device trigonometry).  The frame is the
 * crop's, transposed for a vertical block (wt x ht): X = x + 0.5 - wt / 2, Y = y + 0.5 - ht / 2, u = fl(fl(X c) - fl(Y s)),
 * v = fl(fl(X s) + fl(Y c)), v_min / v_max and u_min / u_max over the four corner pixel centres, L = floor(v_max - v_min) + 1,
 * M = floor(u_max - u_min) + 1, bin k = clamp(floor(v - v_min), 0, L - 1), index j = clamp(floor(u - u_min), 0, M - 1).
 * mn_find_lines_skewed_u8 issues six launches for every block of a call, whatever their number:
 *   1, 2. mn_find_lines_u8's histogram and threshold over blocks[];
 *   3. angle profiles over 32 x 32 tiles (n_ang > 1 only): profiles[a stride + k] = #{ink pixels in bin k at angle a};
 *   4. scores, one CTA per block: scores[a] = sum_k (r_a[k + 1] - r_a[k])^2 (int64), the chosen index the largest score,
 *      ties to the least |a - (n_ang - 1) / 2|, then the least a; the chosen frame goes into chosen, L, M, u_min, v_min, c, s.
 *      When s != 0 it also rewrites blocks[i] as the frame's record (x0 = y0 = 0, w = M, h = L, vertical = 0);
 *   5. the chosen frame's profile into b.prof (3 L values laid out as mn_find_lines_u8's);
 *   6. mn_find_lines_u8's segmentation over blocks[].
 * out->rect[k] is therefore (c0, l0, c1, l1) in frame indices top to bottom when s != 0, and mn_find_lines_u8's rectangle
 * otherwise.  blocks[i] and skew[i].b are the same crop record on entry.  work (work_bytes) covers every hist, prof, profiles
 * and scores of the call and is zeroed by the call; prof and profiles hold 3 stride and n_ang stride int32, stride >= every
 * L of the table; b.scratch 2 stride + 4 int32.  skew, blocks: DEVICE arrays (validated by the caller, |angle| < 45 degrees). */
typedef struct {
    mn_text_block b;            /* the crop record; b.prof receives the chosen frame's profile */
    const double* table;        /* n_ang (c, s) pairs */
    int64_t* scores;            /* n_ang values (written when n_ang > 1) */
    int32_t* profiles;          /* n_ang x stride values (n_ang > 1) */
    int32_t n_ang, stride;
    int32_t chosen, L, M, pad;  /* written by the call */
    double u_min, v_min, c, s;  /* written by the call: the chosen frame */
} mn_skew_block;
int mn_find_lines_skewed_u8(mn_text_block* blocks, mn_skew_block* skew, int n, long long max_tiles, void* work, long long work_bytes,
                            void* stream);

/* Curled text blocks (DESIGN.md section 7b, "Curled blocks").  Block i is a horizontal crop b (h x w) cut into n_strips column
 * strips [x_j, x_{j+1}), x_j = j w / n_strips, each at least 32 pixels wide when n_strips > 1.  mn_find_lines_curved_u8 issues
 * seven launches for every block of a call, whatever the number of blocks and strips:
 *   1-4. mn_find_lines_u8's histogram, threshold, profile and segmentation over blocks[] (the lines of curve=None into b.out);
 *   5. strip profiles over 32 x 32 tiles: sprof[(3 j + q) h + y], q = 0 the ink count of row y in strip j, q = 1 w - its least
 *      ink column, q = 2 its largest ink column + 1 (0 where the row has no ink in the strip);
 *   6. strip runs, one CTA per (strip, block): steps 1-3 of mn_find_lines_u8's segmentation on strip j's count with the strip's
 *      width as M; the kept runs into runs[(j MN_CURVE_RUN_CAP + k) 4 ..] as (a, b, least ink column, largest ink column) and
 *      their number into nruns[j] (minus it when it exceeds MN_CURVE_RUN_CAP, then no run is written);
 *   7. link, one CTA per block: strip by strip, a run continues the line whose last run overlaps it most (rows
 *      min(b, b') - max(a, a') > 0; ties to the least last a, then the least line) when that line's largest overlap in the strip
 *      is this run (ties to the upper run); other runs start lines; a line whose last run lies more than MN_CURVE_MAX_GAP strips
 *      back is closed.  Lines of fewer than (n_strips + 3) / 4 runs are dropped, the rest ordered by (their first run's a, line)
 *      into cout: header = (status, n_lines, Hm, strip, count, 0, 0, 0), Hm the lower median of the kept runs' heights, and per
 *      line (first strip, last strip, runs, least ink column, largest ink column, sample mask, 0, 0, then (a_j, b_j) for
 *      j < MN_CURVE_MAX_STRIPS, (-1, -1) without a run); bit j of the mask is set when 2 (b_j - a_j) <= 3 Hm.  status is
 *      MN_CURVE_ERR_RUNS (strip `strip` holds `count` runs) or MN_CURVE_ERR_LINES (`count` lines) over a limit.
 * hist, b.prof, sprof and nruns lie in work (work_bytes, zeroed by the call); b.scratch (2 h + 4), sscratch (n_strips (2 h + 4)),
 * runs and link (n_strips MN_CURVE_RUN_CAP 7 int32) need no zeroing.  max_tiles >= every block's tile count, max_strips >= every
 * n_strips.  blocks[i] and curves[i].b are the same crop record (vertical = 0).  blocks, curves: DEVICE arrays. */
#define MN_CURVE_MAX_STRIPS 32
#define MN_CURVE_RUN_CAP 256
#define MN_CURVE_MAX_GAP 2
#define MN_CURVE_LINE_INTS (8 + 2 * MN_CURVE_MAX_STRIPS)
#define MN_CURVE_ERR_RUNS 1
#define MN_CURVE_ERR_LINES 2
typedef struct {
    int32_t header[8];
    int32_t line[MN_BLOCK_MAX_LINES][MN_CURVE_LINE_INTS];
} mn_curve_lines;
typedef struct {
    mn_text_block b;            /* the crop record: hist, prof, scratch and out as mn_find_lines_u8's */
    int32_t* sprof;             /* 3 n_strips h */
    int32_t* nruns;             /* n_strips */
    int32_t* runs;              /* n_strips MN_CURVE_RUN_CAP 4 */
    int32_t* sscratch;          /* n_strips (2 h + 4) */
    int32_t* link;              /* n_strips MN_CURVE_RUN_CAP 7 */
    mn_curve_lines* cout;
    int32_t n_strips, pad;
} mn_curve_block;
int mn_find_lines_curved_u8(const mn_text_block* blocks, const mn_curve_block* curves, int n, long long max_tiles, int max_strips,
                            void* work, long long work_bytes, void* stream);

/* Text pages: blocks found by a recursive XY-cut (DESIGN.md section 7b, "Text pages").  Page i is the crop of blocks[i] (h x w,
 * vertical = a vertical page) and pages[i] holds the same record in pages[i].b.  A node is a rectangle of the crop and the axis
 * it tries next; each level runs one attempt on every open node of every page.  mn_find_blocks_u8 issues
 * 5 + 6 MN_PAGE_LEVELS launches for every page of a call, whatever the number of pages and nodes:
 *   1, 2. mn_find_lines_u8's histogram and threshold over blocks[];
 *   3. the ink bitmap (bit x & 31 of bits[y wpitch + x / 32] = ink at (x, y)) and the root node, gaps (1, 1);
 *   4-6. per level (MN_PAGE_LEVELS times): the attempt counts per node (nch, nopen), the per-page scan (off, the next list's
 *        count, the limit), and the ordered emit into the other list; leaves are carried forward, so each list is in reading
 *        order.  Pages without open nodes return at once;
 *   7. text size S (the lower median of max(h, w) >= 2 over the leaves) and the gaps of pass 2 into res, the root again;
 *   8-10. the levels again with those gaps;
 *   11. the leaves classified (MN_PAGE_REJECTED) and each block grown by q = (min(gx, gy) - 1) / 2, clipped, into leaves[].
 * res->error is MN_PAGE_ERR_NODES when a level's list would exceed MN_PAGE_MAX_NODES (or cap) nodes, MN_PAGE_ERR_BLOCKS when
 * the page has more than MN_PAGE_MAX_BLOCKS blocks.  hist, bits, list[2], leaves, nch, nopen, off, b.out (threshold and ink)
 * and res are device memory inside work (work_bytes, zeroed by the call); list[k], leaves, nch, nopen and off hold cap entries, with
 * cap <= min(MN_PAGE_MAX_NODES, (h + 1) (w + 1) / 4).  The state fields are zero on entry.  blocks, pages: DEVICE arrays
 * (validated by the caller: 1 <= w, h <= 32767, the crop inside its image).
 * Ruled pages (DESIGN.md section 7b, "Ruled pages"): a page with rbits (inside work) has rule pixels U, the ink pixels in a
 * maximal row or column run of at least rule_length.  flags holds MN_PAGE_RULES, MN_PAGE_FIGURES, MN_PAGE_DIRECTIONS and
 * MN_PAGE_PANELS for the options below that some page of the call has.  A call with MN_PAGE_RULES issues 3 more launches
 * after the bitmap, whatever the number of pages: the bitmap transposed into rbits' scratch, the long runs of every row of
 * both planes, and the column runs transposed back into rbits, U cleared from bits and |U| counted into res->rule_pixels.
 * In such a page's XY-cut an index whose U count is at least half the node's extent is white, and a white run holding one
 * cuts whatever its length; a block grows by q on each side only up to the nearest row (column) of its margin with U in its
 * columns (rows).  Pages without rbits take the path of a call without MN_PAGE_RULES, and a call without it issues exactly
 * the launches above.
 * Figures (DESIGN.md section 7b, "Figures"): a page with fbits (inside work) has figures: at 7, its pass-1 leaves whose
 * shorter side is at least f go, in leaf order, into figs (MN_PAGE_MAX_FIGURES entries; st = the rows of the figures before
 * it), with f = figure_size, or 3 S when figure_size is 0; res->figure_size = f and res->n_figures = their number, or
 * res->error = MN_PAGE_ERR_FIGURES over the limit.
 * A call with MN_PAGE_FIGURES issues 1 more launch after 7, whatever the number of pages: each figure row of every figure page
 * painted into fbits (F, the union of the figure rectangles) and cleared from bits, so that pass 2 and the leaf rules see
 * I'' = I' and not F.  F takes no part in the rule-index cut; a block's growth stops at U or F as it does at U alone.  The rule
 * launches skip a page with fbits and no rbits, the figure launch a page without fbits, and a call without MN_PAGE_FIGURES
 * issues exactly the launches above.
 * Mixed directions (DESIGN.md section 7b, "Mixed directions"): a page with dirs != 0 has its blocks' directions tested.  A call
 * with MN_PAGE_DIRECTIONS issues 1 more launch after 11, whatever the number of pages: every kept leaf of such a page (its
 * ungrown rectangle in list[src]) has its row and column bands counted and its leaves[] entry marked MN_PAGE_VERTICAL when
 * its direction is vertical, and MN_PAGE_UNDECIDED (with the page's direction) when the test is undecided.  The launch skips
 * pages without dirs and pages with an error; a call without MN_PAGE_DIRECTIONS issues exactly the launches above.
 * Reversed panels (DESIGN.md section 7b, "Reversed panels"): a page with pans (inside work) has panels, and rbits (U's plane,
 * h x wpitch words, with its scratch only when rule_length != 0) even without rules; the rule launches skip a page with
 * rule_length 0.  At 7, such a page keeps its pass-1 leaves (no root yet) with p = panel_size, or S when it is 0, in
 * res->panel_size.  A call with MN_PAGE_PANELS issues 2 more launches after 7, whatever the number of pages:
 *   a. the panel test, one CTA per pass-1 leaf whose shorter side is at least p: a panel iff 2 |I' & leaf| > h w and more than
 *      half of its pixels have a grey within 8 of its modal grey (ties to the smaller); such a leaf's st gains MN_PAGE_PANEL.
 *      The last CTA of each page lists the panels in leaf order in pans (MN_PAGE_MAX_PANELS entries; st = the rows of the
 *      panels before it; res->n_panels, or res->error = MN_PAGE_ERR_PANELS over the limit), selects the figures among the other
 *      leaves and writes the root of pass 2;
 *   b. every panel row painted, one warp per row: the interior inverted in bits (J = not I), the 1-pixel outline cleared from
 *      bits and OR'd into rbits, so that the rule-index cut and the growth stops see it as a rule.
 * A call without MN_PAGE_PANELS issues exactly the launches above.
 * Page turns (DESIGN.md section 7b, "Page turns"): a page with dirs & MN_PAGE_DIRS_TURN (and dirs & 1: its blocks' directions
 * are tested) has a vote table of cap mn_page_turn entries inside work, at the first 16-byte boundary after its leaves table.
 * A call with MN_PAGE_TURNS (and MN_PAGE_DIRECTIONS) issues 1 more launch after the direction launch, whatever the number of
 * pages: every kept leaf i of such a page writes entry i, from the bands along its direction (rows when its leaves[] st lacks
 * MN_PAGE_VERTICAL, else columns), the maximal runs of non-white indices of the direction test: n_bands, e_lo = the sum over
 * bands of lo_k - min lo and e_hi = the sum of max hi - hi_k, lo_k and hi_k the least and largest index across of an ink bit
 * of band k's rows (columns) inside the leaf; all 0 without a band.  Rejected leaves keep a zero entry.  The launch skips pages
 * without the table and pages with an error; a call without MN_PAGE_TURNS issues exactly the launches above. */
#define MN_PAGE_RULES 1
#define MN_PAGE_FIGURES 2
#define MN_PAGE_DIRECTIONS 4
#define MN_PAGE_PANELS 8
#define MN_PAGE_TURNS 16
#define MN_PAGE_DIRS_TURN 2     /* dirs bit: a turn page, with a vote table */
typedef struct {
    int32_t n_bands, pad;
    int64_t e_lo, e_hi;
} mn_page_turn;
#define MN_PAGE_MAX_FIGURES 1024
#define MN_PAGE_MAX_PANELS 1024
#define MN_PAGE_LEVELS 24
#define MN_PAGE_MAX_BLOCKS 1024
#define MN_PAGE_MAX_NODES 65536
#define MN_PAGE_ROWS 1          /* node st: tries rows next (else columns) */
#define MN_PAGE_FAILED 2        /* node st: its previous attempt made no cut */
#define MN_PAGE_LEAF 4          /* node st: closed */
#define MN_PAGE_REJECTED 8      /* node st: a leaf that is not text */
#define MN_PAGE_VERTICAL 16     /* leaf st: a block of a direction page whose direction is vertical */
#define MN_PAGE_UNDECIDED 32    /* leaf st: a block of a direction page that took the page's direction, its test undecided */
#define MN_PAGE_PANEL 64        /* pass-1 leaf st: a panel of a panel page */
#define MN_PAGE_ERR_NODES 1
#define MN_PAGE_ERR_BLOCKS 2
#define MN_PAGE_ERR_FIGURES 3
#define MN_PAGE_ERR_PANELS 4
typedef struct {
    int16_t x0, y0, x1, y1;     /* in the crop */
    int32_t st;
} mn_page_node;
typedef struct {
    int32_t error, n_leaves, n_blocks, text_size;
    int32_t gap_x, gap_y, threshold, ink;
    int32_t rule_pixels;        /* |U| of a ruled page (DESIGN.md section 7b, "Ruled pages"), else 0 */
    int32_t figure_size, n_figures;        /* f and the number of figures of a figure page with a text size, else 0 */
    int32_t panel_size, n_panels, pad;     /* p and the number of panels of a panel page with a text size, else 0 */
} mn_page_result;
typedef struct {
    mn_text_block b;            /* the crop record (b.hist, b.out as mn_find_lines_u8's) */
    uint32_t* bits;             /* h x wpitch words */
    mn_page_node* list[2];
    mn_page_node* leaves;       /* the result: n_leaves leaves in reading order, blocks grown */
    int32_t* nch;
    int32_t* nopen;
    int32_t* off;
    mn_page_result* res;
    int32_t wpitch, cap, gap_x, gap_y;   /* gap_x, gap_y: 0 = the default */
    int32_t src, active, open, gx, gy, pad, n[2];   /* state, written by the call */
    uint32_t* rbits;            /* null, or a ruled page's h x wpitch words of U followed by w x ceil(h / 32) words of scratch */
    int32_t rule_length;        /* a ruled page's rule length, 2 <= rule_length <= 32767 */
    int32_t dirs;               /* 1: a direction page, its blocks' directions tested; else 0.  | MN_PAGE_DIRS_TURN: a turn page */
    uint32_t* fbits;            /* null, or a figure page's h x wpitch words of F */
    mn_page_node* figs;         /* a figure page's table of MN_PAGE_MAX_FIGURES figures */
    int32_t figure_size;        /* a figure page's f in [2, 32767], or 0 for 3 S */
    int32_t frows;              /* state: the rows of all of its figures */
    mn_page_node* pans;         /* null, or a panel page's table of MN_PAGE_MAX_PANELS panels */
    int32_t panel_size;         /* a panel page's p in [2, 32767], or 0 for S */
    int32_t prows;              /* state: the rows of all of its panels */
    int32_t pdone, pad3;        /* state: the panel test's CTAs done with the page */
} mn_text_page;
int mn_find_blocks_u8(const mn_text_block* blocks, mn_text_page* pages, int n, long long max_tiles, int flags, void* work,
                      long long work_bytes, void* stream);

/* Skewed pages (DESIGN.md section 7b, "Skewed pages").  Page i is searched as a skewed block on skew[i] (skew[i].b, blocks[i] and
 * pages[i].b the same crop record on entry; a page without skew the one-entry table (1, 0)), and the XY-cut of
 * mn_find_blocks_u8 runs on a bitmap of frame cells.  mn_find_blocks_skewed_u8 issues 7 + 6 MN_PAGE_LEVELS launches for every
 * page of a call, whatever the number of pages and nodes:
 *   1-4. mn_find_lines_skewed_u8's histogram, threshold, angle profiles and scores (the chosen frame into skew[i]);
 *   5. the frame bitmap: bit j & 31 of bits[k wpitch + j / 32] is set iff an ink pixel has cell (k, j) in the frame at (c, s),
 *      or for a vertical page at (c, -s) on the untransposed crop (the transposed search frame with its axes swapped); the root
 *      node, and pages[i].b.w = M, pages[i].b.h = L;
 *   6-13. mn_find_blocks_u8's levels, text size and leaves, in frame cells (with its 3 rule launches under MN_PAGE_RULES,
 *         its figure launch under MN_PAGE_FIGURES, its direction launch under MN_PAGE_DIRECTIONS and its 2 panel launches
 *         under MN_PAGE_PANELS; a ruled, figure, direction or panel page has skew None, so its frame bitmap is
 *         mn_find_blocks_u8's).
 * bits holds max L x wpitch words, wpitch >= max M / 32, and cap entries per list, max over the page's table; the angle
 * profiles and scores are as mn_find_lines_skewed_u8's (b.prof unused).  work (work_bytes) is zeroed by the call. */
int mn_find_blocks_skewed_u8(mn_text_block* blocks, mn_skew_block* skew, mn_text_page* pages, int n, long long max_tiles, int flags,
                             void* work, long long work_bytes, void* stream);

/* Windowed blocks (DESIGN.md section 7b, "Skewed pages").  Block i is the set of pixels of the crop wins[i].b whose frame cell
 * (k, j) at (c, s) (the frame of "Skewed blocks", transposed crop for a vertical block) lies in [c0, c1) x [l0, l1).
 * blocks[i] is its frame record: x0 = y0 = 0, w = c1 - c0, h = l1 - l0, vertical = 0, with hist, prof, scratch, out and the
 * knobs shared with wins[i].b.  mn_find_lines_window_u8 issues four launches for every block of a call: the histogram of the
 * set and the profile in bins k - l0 and indices j - c0, both over the tiles of the footprint [px0, px0 + pw) x
 * [py0, py0 + ph) of crop pixels (which holds the set), and mn_find_lines_u8's threshold and segmentation over blocks[].
 * out->rect[k] is therefore (c0', l0', c1', l1') in window cells, top to bottom.  max_tiles >= every footprint's tile count;
 * work (work_bytes) covers every hist and prof of the call and is zeroed by the call. */
typedef struct {
    mn_text_block b;            /* the crop record */
    double c, s;                /* the frame's angle */
    int32_t c0, l0, c1, l1;     /* the window, in frame cells */
    int32_t px0, py0, pw, ph;   /* its footprint, in crop pixels */
} mn_window_block;
int mn_find_lines_window_u8(const mn_text_block* blocks, const mn_window_block* wins, int n, long long max_tiles, void* work,
                            long long work_bytes, void* stream);

/* Page corners (DESIGN.md section 7b, "Perspective pages").  Page i is the whole image of blocks[i] (x0 = y0 = 0, w x h, its
 * polarity); pages[i].b is the same record.  mn_find_page_quads_u8 issues 8 launches for every page of a call:
 *   1, 2. mn_find_lines_u8's histogram and threshold over blocks[] (Otsu's t into b.out);
 *   3. per 32 x 32 tile, the 4-connected components of the paper mask (grey > t; grey <= t for MN_INK_LIGHT) merged in
 *      shared memory: label[y w + x] = the raster index of the tile-local root, -1 off the paper;
 *   4. the merge across tile borders, by union-find with atomicMin;
 *   5. path compression (label = the component's smallest raster index) and each component's pixels into count[label];
 *   6. the page: the most pixels, ties to the smallest label, into *best as (count << 32) | ~label (0: no paper);
 *   7. each row's extent of the page, ext[2 y] = max(w - x), ext[2 y + 1] = max(x + 1) (0: none);
 *   8. one CTA per page: the monotone-chain hull of the rows' pixel-square corners into hull (x, y pairs, cross products in
 *      int64, collinear points dropped) and the four hull vertices of the largest doubled area, ties to the smallest index
 *      tuple, ordered clockwise on screen from tl (the smallest x + y, then y) into res.
 * label and count hold h w values, ext 2 h, hull 2 (4 h + 8); every one of them, best and res lie in work (work_bytes, zeroed
 * by the call).  blocks, pages: DEVICE arrays (validated by the caller: 1 <= w, h <= 32767). */
typedef struct {
    int32_t threshold;          /* Otsu's t of the image */
    int32_t label;              /* the page's label (its smallest raster index), -1 when no pixel is paper */
    int32_t size;               /* its pixels */
    int32_t n_hull;             /* hull vertices */
    int64_t area2;              /* the quad's doubled area */
    int32_t idx[4];             /* the quad's hull vertices, i < a < j < b */
    int32_t quad[8];            /* tl, tr, br, bl as (x, y) pixel-square corners */
} mn_page_quad;
typedef struct {
    mn_text_block b;
    int32_t* label;
    int32_t* count;
    int32_t* ext;
    unsigned long long* best;
    int32_t* hull;
    mn_page_quad* res;
} mn_quad_page;
int mn_find_page_quads_u8(const mn_text_block* blocks, const mn_quad_page* pages, int n, long long max_tiles, void* work,
                          long long work_bytes, void* stream);

/* Book spreads (DESIGN.md section 7b, "Book spreads"): the spine of an open book, searched on the page component and corners
 * that mn_find_page_quads_u8 left in its work, on the same stream, before that work is freed.  spines[i].page points to the
 * mn_quad_page record of the spread's image.  mn_find_page_spines_u8 issues 2 launches for every spread of a call:
 *   1. per 32 x 32 tile, each column's extent of the page component: cols[x] = max(h - y), cols[w + x] = max(y + 1) over the
 *      component's pixels of column x (0: none), so cols[x] = h - t(x) and cols[w + x] = b(x);
 *   2. one CTA per spread: over the columns with 4 (x - tl.x) >= tr.x - tl.x and 4 (tr.x - x) >= tr.x - tl.x, the top point
 *      T_x = (x, t(x)) of the largest D_x = cross(tr - tl, T_x - tl), ties to the smallest x; over bl.x .. br.x likewise the
 *      bottom point B_x = (x, b(x)) of the largest E_x = cross(B_x - bl, br - bl); found when D, E > 0, D^2 >= 4 |tr - tl|^2,
 *      100 D >= |tr - tl|^2 and the same for E against |br - bl|.  All in int64.
 * cols holds 2 w int32 in zeroed memory (mn_find_page_quads_u8's work); res is written whole.  spines: DEVICE array. */
typedef struct {
    int32_t found;              /* 1 when both notches are deep enough */
    int32_t st[2];              /* the top spine point (x, t(x)); (-1, -1) when no column lies in the range */
    int32_t sb[2];              /* the bottom spine point (x, b(x)); (-1, -1) likewise */
    int32_t pad;
    int64_t D, E;               /* the largest top and bottom depths, doubled-area units (INT64_MIN: no column) */
} mn_page_spine;
typedef struct {
    const mn_quad_page* page;
    int32_t* cols;
    mn_page_spine* res;
} mn_spine_page;
int mn_find_page_spines_u8(const mn_spine_page* spines, int n, long long max_tiles, void* stream);

/* Seals (DESIGN.md section 7b, "Seals"): round and oval stamps found by colour and shape on a level page crop b (w x h, 3
 * channels), kept out of its layout and described for restoration.  A pixel is seal-coloured when max(c) - min(c) >=
 * MN_SEAL_CHROMA over its three channels (any channel order).  The crop is cut into MN_SEAL_CELL x MN_SEAL_CELL cells (cell
 * (cx, cy) = pixels [4 cx, 4 cx + 4) x [4 cy, 4 cy + 4) of the crop, index cy cw + cx, cw = ceil(w / 4), ch = ceil(h / 4)); a
 * cell is on when it holds at least MN_SEAL_CELL_MIN seal-coloured pixels.  A candidate is an 8-connected component of on cells
 * whose seal-coloured pixels' box (x0, y0, x1, y1) (crop pixels, end exclusive) has sides A = x1 - x0, B = y1 - y0 in
 * [seal_size, MN_SEAL_MAX_SIDE] and 2 max(A, B) <= 3 min(A, B).  For a pixel (x, y), X = 2 x + 1 - (x0 + x1),
 * Y = 2 y + 1 - (y0 + y1); its radial bin is k = floor(32 rho), rho^2 = (X / A)^2 + (Y / B)^2, the largest k with
 * k^2 A^2 B^2 <= 1024 (X^2 B^2 + Y^2 A^2) in int64, and only k < MN_SEAL_BINS counts (rho < 33 / 32); its sector s in
 * [0, 72) is the 5-degree sector of (X B, -Y A) between the directions d_s and d_s+1 of MN_SEAL_DIRS (d_s+36 = -d_s): for p in
 * the upper half plane (p.y > 0, or p.y = 0 < p.x) the largest s < 36 with cross(d_s, p) >= 0, else 36 + that of -p; p = 0 is
 * sector 0.  Per candidate, ink[k][s] counts the seal-coloured pixels and area[k] all pixels of the box in each bin:
 *   ring = the sectors with ink at k in [MN_SEAL_RING_K, 32]; a seal when ring >= MN_SEAL_RING_SECTORS.
 *   band: from k = 32 inward, the first run of bins with 4 ink_k >= area_k (the ring), then the bins with 32 ink_k >= area_k
 *   (its edge), then at least one bin with 32 ink_k < area_k (the gap), then the run of bins with 32 ink_k >= area_k down to
 *   k = MN_SEAL_BAND_MIN_K at most: k_top its first bin and k_bottom its last; no gap or no such run is MN_SEAL_NO_BAND.
 *   arc: per sector the ink of the band's bins; a sector is empty when 720 ink < max(720, band_ink); the gap [g0, g0 + n) is the
 *   longest circular run of empty sectors, ties to the smallest g0 (n = 72, g0 = 0 when all are empty); MN_SEAL_NO_GAP when
 *   n < MN_SEAL_MIN_GAP, MN_SEAL_SHORT when 72 - n < MN_SEAL_MIN_TEXT.
 * mn_find_seals_u8 issues 6 launches for every page of a call, whatever the number of pages and candidates:
 *   1. per cell, its seal-coloured count and their box: label[c] = c for an on cell, else -1; box[4 c ..] the on cell's box;
 *   2. per on cell, union with its on neighbours W, NW, N and NE (uf_union: a root is the smallest index of its set);
 *   3. per on cell, path compression and its box folded into its root's by atomicMin / atomicMax;
 *   4. per root, the size test, and the candidate (box, root) appended to cand (out->n_cand counts them all);
 *   5. one CTA per candidate slot (MN_PAGE_MAX_SEALS per page): the histograms in shared memory and the ring, band and arc
 *      into out->seal[r], r the candidate's rank by (y0, x0, root); out->n_seals counts the seals.  A page with more than
 *      MN_PAGE_MAX_SEALS candidates gets out->error = MN_SEAL_ERR_SEALS and no seal;
 *   6. the layout copy (mn_seal_layout_u8's launch).
 * mn_seal_layout_u8 issues that one launch: copy (h x 3 w bytes, pitch 3 w) = the crop, with every seal-coloured pixel at
 * rho < 33 / 32 of a seal of out (the out->n_cand entries with found != 0, boxes in crop pixels) set to (255, 255, 255).
 * label and box hold cw ch and 4 cw ch int32, cand MN_PAGE_MAX_SEALS 8 int32; out tables lie in work (work_bytes, zeroed by
 * mn_find_seals_u8); the copy is written whole.  pages: DEVICE array, every crop at most 32767 on a side. */
#define MN_PAGE_SEALS 16
#define MN_PAGE_MAX_SEALS 64
#define MN_SEAL_CHROMA 64
#define MN_SEAL_CELL 4
#define MN_SEAL_CELL_MIN 2
#define MN_SEAL_MAX_SIDE 4096
#define MN_SEAL_BINS 33
#define MN_SEAL_SECTORS 72
#define MN_SEAL_RING_K 26
#define MN_SEAL_RING_SECTORS 54
#define MN_SEAL_RING_DENSITY 4
#define MN_SEAL_BAND_DENSITY 32
#define MN_SEAL_BAND_MIN_K 10
#define MN_SEAL_EMPTY_DIV 720
#define MN_SEAL_MIN_GAP 2
#define MN_SEAL_MIN_TEXT 9
#define MN_SEAL_NO_BAND 1
#define MN_SEAL_NO_GAP 2
#define MN_SEAL_SHORT 3
#define MN_SEAL_ERR_SEALS 1
/* d_s = (round(2^20 cos 5s), round(2^20 sin 5s)) for s < 36 */
#define MN_SEAL_DIRS {{1048576, 0}, {1044586, 91389}, {1032646, 182083}, {1012847, 271391}, {985339, 358634}, {950333, 443147}, \
    {908093, 524288}, {858943, 601438}, {803256, 674012}, {741455, 741455}, {674012, 803256}, {601438, 858943}, {524288, 908093}, \
    {443147, 950333}, {358634, 985339}, {271391, 1012847}, {182083, 1032646}, {91389, 1044586}, {0, 1048576}, {-91389, 1044586}, \
    {-182083, 1032646}, {-271391, 1012847}, {-358634, 985339}, {-443147, 950333}, {-524288, 908093}, {-601438, 858943}, \
    {-674012, 803256}, {-741455, 741455}, {-803256, 674012}, {-858943, 601438}, {-908093, 524288}, {-950333, 443147}, \
    {-985339, 358634}, {-1012847, 271391}, {-1032646, 182083}, {-1044586, 91389}}
typedef struct {
    int32_t x0, y0, x1, y1;     /* the box, in crop pixels */
    int32_t root;               /* the component's smallest cell index */
    int32_t ring;               /* sectors hit at k >= MN_SEAL_RING_K */
    int32_t found;              /* 1: a seal */
    int32_t k_bottom, k_top;    /* the band, or -1 */
    int32_t g0, n_gap;          /* the arc's gap, or -1 */
    int32_t why;                /* 0, MN_SEAL_NO_BAND, MN_SEAL_NO_GAP or MN_SEAL_SHORT; 0 for a candidate that is no seal */
    int32_t band_ink;           /* the band's seal-coloured pixels */
    int32_t pad[3];
} mn_seal;
typedef struct {
    int32_t error, n_cand, n_seals, pad;
    mn_seal seal[MN_PAGE_MAX_SEALS];   /* the candidates by (y0, x0, root) */
} mn_seal_table;
typedef struct {
    mn_text_block b;            /* the crop record (img, pitch, x0, y0, w, h) */
    uint8_t* copy;              /* the layout copy */
    int32_t* label;
    int32_t* box;
    int32_t* cand;
    mn_seal_table* out;
    int32_t seal_size, pad;
} mn_seal_page;
int mn_find_seals_u8(const mn_seal_page* pages, int n, long long max_tiles, long long max_cell_tiles, void* work,
                     long long work_bytes, void* stream);
int mn_seal_layout_u8(const mn_seal_page* pages, int n, long long max_tiles, void* stream);

/* Seal centre lines (DESIGN.md section 7b, "Seal centre lines"): the horizontal text across a found seal's centre, and the
 * seal's turn.  Per found seal j of a page's mn_seal_table, with its box, A x B, and histograms as mn_find_seals_u8 defines them:
 *   head: with a band whose k_top >= MN_SEAL_HEAD_MIN_K, sec[s] = the ink of bins [k_top - MN_SEAL_HEAD_BINS + 1, k_top] in sector s, and (g0, n)
 *   its gap by the arc rule; why = MN_SEAL_NO_GAP / MN_SEAL_SHORT / 0 as for the arc.  The turn t = 2 g0 + n - 108 in
 *   2.5-degree steps, normalised to (-72, 72], counter-clockwise on screen; t = 0 when why != 0.  A seal without such a
 *   band gets why = MN_SEAL_NO_BAND, t = 0, no gap and no band (-1).
 *   arc band: the arc sectors are all but [g0, g0 + n); ink'_k their ink in bin k.  From k = k_top inward, k_bottom is the last
 *   bin of the run with 32 * 72 * ink'_k >= area_k (72 - n), down to MN_SEAL_BAND_MIN_K; k_top is always in it.
 *   interior: the seal-coloured pixels at k < k_in, k_in = k_bottom, and those at k < k_gap = max(k_bottom, k_top -
 *   MN_SEAL_HEAD_BINS + 1) in the gap's sectors less MN_SEAL_GAP_MARGIN at each end, (s - g0 - margin) mod 72 < n - 2 margin.
 *   Without a band, k_in = k_gap = the first bin inside the ring's edge of the band walk (gap_top; 0 when negative).
 *   rows: a pixel's (X, Y) turned by -t with (c, s) = MN_SEAL_TURNS[t mod 36] turned by (t mod 144) / 36 quarter turns
 *   ((c, s) -> (-s, c)): u = (X c - Y s) >> 21, v = (X s + Y c) >> 21 (floor).  Per row v, the min and max u of its ink.
 *   lines: runs of ink rows whose gaps are under MN_SEAL_LINE_GAP rows; a run h rows high and w = u_max - u_min + 1 wide is a
 *   line when h >= max(MN_SEAL_LINE_MIN_H, (A + B) / MN_SEAL_LINE_H_DIV) and w >= MN_SEAL_LINE_RATIO h.  Its box (u0, v0, u1,
 *   v1), end exclusive, is padded by p = max(MN_SEAL_LINE_PAD, h / MN_SEAL_LINE_PAD_DIV) and clipped to [-R - 1, R + 1],
 *   R = k_gap max(A, B) / 64.  n_found counts the lines, the first MN_SEAL_MAX_LINES from the top are kept.
 * mn_find_seal_lines_u8 issues 1 launch: one CTA per seal slot (MN_PAGE_MAX_SEALS per page) writes the slot's record of
 * page->lines.  It rebuilds the seal's histograms and the row extents (at most MN_SEAL_MAX_SIDE + 4 rows) in shared memory.  A
 * slot that is no found seal, and every slot of a table with an error, gets a zero record.  It reads the tables
 * mn_find_seals_u8 wrote before it on the same stream.  pages: DEVICE array. */
#define MN_SEAL_HEAD_BINS 4
#define MN_SEAL_HEAD_MIN_K 16
#define MN_SEAL_GAP_MARGIN 2
#define MN_SEAL_LINE_GAP 3
#define MN_SEAL_LINE_MIN_H 4
#define MN_SEAL_LINE_H_DIV 64
#define MN_SEAL_LINE_RATIO 2
#define MN_SEAL_LINE_PAD 2
#define MN_SEAL_LINE_PAD_DIV 8
#define MN_SEAL_MAX_LINES 4
#define MN_SEAL_TURN_STEPS 144
/* (round(2^20 cos 2.5 j), round(2^20 sin 2.5 j)) for j < 36 */
#define MN_SEAL_TURNS {{1048576, 0}, {1047578, 45738}, {1044586, 91389}, {1039605, 136867}, {1032646, 182083}, {1023721, 226953}, \
    {1012847, 271391}, {1000045, 315313}, {985339, 358634}, {968758, 401273}, {950333, 443147}, {930098, 484179}, \
    {908093, 524288}, {884360, 563399}, {858943, 601438}, {831891, 638333}, {803256, 674012}, {773091, 708408}, \
    {741455, 741455}, {708408, 773091}, {674012, 803256}, {638333, 831891}, {601438, 858943}, {563399, 884360}, \
    {524288, 908093}, {484179, 930098}, {443147, 950333}, {401273, 968758}, {358634, 985339}, {315313, 1000045}, \
    {271391, 1012847}, {226953, 1023721}, {182083, 1032646}, {136867, 1039605}, {91389, 1044586}, {45738, 1047578}}
typedef struct {
    int32_t turn;               /* t, 2.5-degree steps */
    int32_t g0, n_gap;          /* the head gap, or -1 */
    int32_t k_bottom, k_top;    /* the arc band, or -1 */
    int32_t why;                /* 0, MN_SEAL_NO_BAND, MN_SEAL_NO_GAP or MN_SEAL_SHORT */
    int32_t k_in, k_gap;        /* the interior's bins, and in the head gap */
    int32_t n_found, n_lines;   /* the lines found, and kept */
    int32_t pad[2];
    int32_t box[MN_SEAL_MAX_LINES][4];  /* (u0, v0, u1, v1) in the stamp frame, pixels from the box centre */
} mn_seal_lines;
typedef struct {
    mn_seal_lines seal[MN_PAGE_MAX_SEALS];   /* slot j describes the table's seal[j] */
} mn_seal_line_table;
typedef struct {
    mn_text_block b;            /* the crop record, as in the page's mn_seal_page */
    const mn_seal_table* seals;
    mn_seal_line_table* lines;
} mn_centre_page;
int mn_find_seal_lines_u8(const mn_centre_page* pages, int n, void* stream);

/* Flat pages (DESIGN.md section 7b, "Flat pages"): the dewarp field of a curled page, built from its traced lines, composed with
 * the page's frame and sampled from the photo.  A page's line table (built on the host, pipeline.flat_line_table) holds
 * MN_FLAT_LINE_DOUBLES fp64 values per line, sorted by anchor Y (ties in reading order): xs, xe, mu_0 .. mu_3, Y, bx0, bx1.
 * mn_flat_columns_batched: blockIdx.y = page, one thread per frame column x (centre xc = x + 0.5).  For every line k whose
 * block holds x (bx0 <= x < bx1), in table order, it writes (Y_k, m_k(x)) to field[(x * stride + n) * 2 ..], n counting up,
 * with m_k(x) the de Casteljau value of mu at t = clamp(fl(fl(xc - xs) / fl(xe - xs)), 0, 1); then cols[x] = n,
 * cols[dw + x] = the nearest column left of x that some line's block holds (-1: none) and cols[2 dw + x] the nearest one right
 * of it (-1: none).  The host sizes stride as the most lines any column meets (at most MN_FLAT_MAX_COLUMN_LINES).
 * mn_flat_remap_u8_batched: blockIdx.y = page, one thread per pixel (x, y) of the [dh][dw][cn] flat page, yc = y + 0.5.  In a
 * column with n > 0 lines, k = the last line with Y_k <= yc (a binary search): src = fl(yc + fl(M_0 - Y_0)) above the first line,
 * fl(yc + fl(M_last - Y_last)) below the last, else fl(M_k + fl(fl(fl(yc - Y_k) fl(M_k+1 - M_k)) / fl(Y_k+1 - Y_k))).  A column
 * without lines takes d = src - yc of its neighbours l < x < r at the same yc, fl(dl + fl(fl(fl(x - l) fl(dr - dl)) / fl(r - l)))
 * (the one side's d when only one exists, 0 when none does), and src = fl(yc + d).  The frame point (xc, src) maps to the photo:
 * MN_FLAT_RECT (m = x0, y0): (fl(x0 + xc), fl(y0 + src)); MN_FLAT_QUAD (m = H's a .. h): u = xc / dw, v = src / dh, w =
 * fl(fl(fl(g u) + fl(h v)) + 1), X = fl(fl(fl(fl(a u) + fl(b v)) + c) / w), Y likewise with d, e, f.  Then mapx = fl(X - 0.5),
 * mapy = fl(Y - 0.5), and remap's cubic sampler exactly as mn_remap_curved_u8_batched uses it.  Byte offsets are 64-bit.
 * pages: DEVICE array of records whose tables point into device memory (validated by the caller). */
#define MN_FLAT_LINE_DOUBLES 9
#define MN_FLAT_MAX_COLUMN_LINES 256
#define MN_FLAT_RECT 0
#define MN_FLAT_QUAD 1
typedef struct {
    const uint8_t* src;         /* row 0 of the photo */
    int64_t src_pitch;
    int32_t h, w;
    uint8_t* dst;               /* row 0 of the flat page */
    int64_t dst_pitch;
    int32_t dh, dw;
    const double* lines;        /* the line table */
    int32_t* cols;              /* [3][dw]: line counts, left and right neighbours */
    double* field;              /* [dw][stride][2]: (Y, M) per column */
    int32_t n_lines, stride;
    int32_t kind, pad;          /* MN_FLAT_RECT or MN_FLAT_QUAD */
    double m[8];
} mn_flat_page;
int mn_flat_columns_batched(const mn_flat_page* pages, int n, int max_width, void* stream);
int mn_flat_remap_u8_batched(const mn_flat_page* pages, int n, int cn, long long max_pixels, void* stream);

/* Even lighting (DESIGN.md section 7b, "Even lighting"): page i (h x w, three channels, odd window k) is evened as
 * E = rint(255 F / B) per channel (half to even, 0 where B = 0, at most 255), B the grey closing of F (the min over the k x k
 * window cut to the page of the max over the k x k window cut to the page), computed as rintf(__fdiv_rn(255.f F, (float)B)).
 * For light ink every byte is complemented on read and on write (v ^ 255), so E = 255 - E_dark(255 - F) on one code path.
 * mn_even_light_u8 issues 6 launches for every page of a call (4 when `threshold` is 0), whatever their number:
 *   1, 2. (threshold != 0) mn_find_lines_u8's histogram and threshold over blocks[] (blocks[i] and pages[i].b the same
 *         record: the frame whose ink decides the polarity, b.polarity; MN_INK_AUTO: the minority side of Otsu's threshold),
 *         the ink into b.out->ink;
 *   3-6. a row max, a column max, a row min and a column min pass, the divide fused into the last; blockIdx.y = page.  Each pass
 *        gives thread (line, s) the outputs i in [s k, s k + k) of its line and costs O(1) comparisons per pixel whatever k:
 *        the van Herk / Gil-Werman suffix extrema of segment s and prefix extrema of segment s + 1 of the line padded by k / 2
 *        identities (0 for max, 255 for min) at each end, the padding never read.
 * ink is read from b.out->ink on the device: written by launch 2, or left there by an earlier call when `threshold` is 0.
 * src and dst may be the same pixels (evened in place).  s1, s2: dense scratch planes of h w 3 bytes.  b.out needs only its
 * first 16 bytes (threshold and ink), b.hist 256 int32 in work (work_bytes, zeroed by the call when `threshold` is set).
 * max_tiles >= every frame's tile count, max_lines >= every page's h ceil(w / k) and w ceil(h / k).  Byte offsets are 64-bit.
 * blocks, pages: DEVICE arrays (validated by the caller: 1 <= h, w <= 32767, k odd in [3, 32767]; blocks may be NULL when
 * `threshold` is 0). */
typedef struct {
    mn_text_block b;            /* the frame whose ink is used */
    const uint8_t* src;         /* row 0 of the page F */
    int64_t src_pitch;
    uint8_t* dst;               /* row 0 of the evened page */
    int64_t dst_pitch;
    int32_t h, w;
    int32_t k, pad;             /* the window */
    uint8_t* s1;                /* scratch planes */
    uint8_t* s2;
} mn_light_page;
int mn_even_light_u8(const mn_text_block* blocks, const mn_light_page* pages, int n, int threshold, long long max_tiles,
                     long long max_lines, void* work, long long work_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MARCONET_B200_H */
