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
 *      rounded on its own), D = #{g <= t}; ink = polarity, or for MN_INK_AUTO dark (g <= t) iff 2 D <= h w, else light (g > t);
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

#ifdef __cplusplus
}
#endif
#endif /* MARCONET_B200_H */
