/* fsb200.h -- C ABI of libfsb200.so: H100 (sm_90a) kernels for the FasterSeg conv hot path.
 *
 * The reference (VITA-Group/FasterSeg) has no FFI of its own: its hot path bottoms out in
 * torch.nn.functional calls (SURVEY.md section 8b).  Each entry point below therefore cites the
 * reference call site(s) whose arithmetic it replaces; the Python operator classes in
 * fasterseg_b200/{operations,slimmable_ops,seg_oprs,model_seg}.py (same names / signatures /
 * state_dict keys as the reference) bind these symbols through ctypes (INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless stated otherwise;
 *   - activations are NHWC fp16 ("channels-last"), addressed as base + pixel * cstride + channel,
 *     so a channel slice of a wider concat buffer is just (base + offset, cstride) -- this is how
 *     torch.cat(dim=1) call sites become zero-copy;
 *   - master weights stay fp32 OIHW in the caller's module (checkpoint format); kernels consume a
 *     packed fp16 copy produced by fsb_pack_conv_weight;
 *   - all work is enqueued on `stream` (a cudaStream_t passed as void*); no call synchronises;
 *   - return value: 0 on success, negative fsb_status otherwise; fsb_last_error_string() gives the
 *     text of the last failure on the calling thread.  The library owns no buffers.
 */
#ifndef FSB200_H_
#define FSB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FSB_ABI_VERSION 2

typedef enum fsb_status {
  FSB_OK = 0,
  FSB_ERR_INVALID = -1,     /* bad argument / unsupported shape */
  FSB_ERR_CUDA = -2,        /* CUDA runtime or driver error (text in fsb_last_error_string) */
  FSB_ERR_UNSUPPORTED = -3, /* valid request this build has no kernel for */
  FSB_ERR_NO_DEVICE = -4
} fsb_status;

/* epilogue / layout flags for fsb_conv_desc.flags */
#define FSB_CONV_RELU 1u        /* y = max(y, 0) */
#define FSB_CONV_AFFINE 2u      /* y = y * scale[c] + shift[c]  (BN eval folded, or conv bias in shift) */
#define FSB_CONV_FORCE_DIRECT 4u /* use the CUDA-core direct kernel (validation / odd shapes) */
#define FSB_CONV_OUT_F32 16u    /* y is fp32 NHWC (y_cstride in fp32 elements): the training path keeps the raw conv output in
                                   fp32 so that BatchNorm normalises un-rounded values, like the fp32 reference */
#define FSB_ACT_IN_F32 32u      /* fsb_affine_act: x is fp32 NHWC */
#define FSB_CONV_STATS 8u       /* also produce per-channel sum / sum-of-squares of the fp32 conv output as PARTIAL ROWS, one
                                   per CTA (BN train, K2) -- see "Deterministic statistics" below.  Only with FSB_CONV_OUT_F32
                                   and without FSB_CONV_AFFINE / FSB_CONV_RELU (the raw output is what is summed, on every
                                   kernel); any other combination is FSB_ERR_INVALID before anything is written */
/* Nearest-neighbour resizes folded into the tensor maps of the wgmma conv (latency/ deployment network,
 * latency/operations.py:265,269,427,434, latency/model_seg.py:305,309,315).  Addresses change, nothing else: the result is
 * bit for bit the conv of the resized input / the resized conv output. */
#define FSB_CONV_X_DOWN2 64u    /* x is a 2H x 2W map (pixel stride x_cstride); the conv reads its even rows and columns, i.e.
                                   F.interpolate(x, (H, W), mode='nearest'); H, W in the desc are the HALF size. Stride 1 only */
#define FSB_CONV_Y_UP2 128u     /* y is a 2Ho x 2Wo map (pixel stride y_cstride); every output pixel is stored to its 2x2 block,
                                   i.e. F.interpolate(conv, (2Ho, 2Wo), mode='nearest').  Needs the TMA-store epilogue: fp16
                                   output, Cout and y_cstride multiples of 8, 16-byte aligned y, Cin >= 16; not with
                                   FSB_CONV_STATS / FSB_CONV_OUT_F32 / FSB_CONV_FORCE_DIRECT (FSB_ERR_UNSUPPORTED) */

/* One convolution launch.  Replaces F.conv2d at search/slimmable_ops.py:47 and every nn.Conv2d in
 * search/operations.py:42-534 / search/seg_oprs.py:17-39,228-274, fused with the BatchNorm (eval) +
 * ReLU that follow it there. */
typedef struct fsb_conv_desc {
  int32_t N, H, W;       /* input batch / height / width                      */
  int32_t Cin, Cout;     /* ACTIVE channels (slimmable slice), not max widths */
  int32_t ksize;         /* 1 or 3                                            */
  int32_t stride;        /* 1 or 2                                            */
  int32_t pad;           /* 0 or 1 (ksize 3 uses dil*1)                       */
  int32_t dil;           /* 1 (kept for API parity with the reference ctor)   */
  int32_t off_h, off_w;  /* input origin shift: conv runs on x[:, off_h:, off_w:, :]
                            (FactorizedReduce's x[:,:,1:,1:], operations.py:523) */
  int32_t Ho, Wo;        /* output height / width                             */
  int32_t x_cstride;     /* elements between consecutive pixels of x (>= Cin) */
  int32_t y_cstride;     /* elements between consecutive pixels of y (>= Cout)*/
  uint32_t flags;
  int32_t stats_C;       /* FSB_CONV_STATS: half-width SC of a statistics row (0 -> Cout); row stride = 2*SC floats     */
  int32_t stats_off;     /* FSB_CONV_STATS: this conv's channel c lands at row[stats_off + c] / row[SC + stats_off + c]
                            (FactorizedReduce: two convs fill the two halves of one BatchNorm's statistics)             */
} fsb_conv_desc;

/* Deterministic statistics.  BatchNorm statistics (forward: sum x, sum x^2; backward: sum dz, sum dz*xhat) and the scalar
 * gradients of fsb_wsum_bwd are never accumulated with floating-point atomics: a chain of BatchNorm layers amplifies the
 * run-to-run last-bit differences of atomics into percent-level gradient differences.  Every producer CTA writes one
 * PARTIAL ROW [sum(0..SC) | sumsq(0..SC)] and the consumer adds the rows in index order in double precision
 * (fsb_bn_finalize folds this in; fsb_rowsum is the stand-alone form).  The same inputs therefore give bit-identical
 * activations and activation gradients on every run.  Weight gradients use split-K fp32 atomics by default (their
 * rounding noise is not amplified); fsb_set_option("FSB_DETERMINISTIC", 1) removes those too. */

/* BatchNorm parameter set selected ON THE DEVICE (captured training graphs: a slimmable unit runs at its maximum width,
 * the width index of the pass lives in device memory, and channels >= C of the selected set are forced to zero --
 * USBatchNorm2d's per-width nn.BatchNorm2d list, search/slimmable_ops.py:51-70). */
typedef struct fsb_bn_sel {
  float* gamma;
  float* beta;
  float* running_mean;
  float* running_var;
  long long* num_batches_tracked;
  float* dgamma; /* gradient destinations, accumulated into (may be NULL) */
  float* dbeta;
  int32_t C;     /* channels of this parameter set */
  int32_t reserved;
} fsb_bn_sel;

int fsb_abi_version(void);
const char* fsb_last_error_string(void);
/* number of SMs / compute capability of the current device (host ints, may be NULL) */
int fsb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* Programmatic dependent launch between consecutive kernels of this library (default on; env FSB_PDL=0 disables).
 * With it a kernel's prologue (barrier init, descriptor prefetch) overlaps its predecessor's tail. */
int fsb_set_pdl(int enabled);
/* Tuning / validation switches, named like their environment variables (FSB_CONV_TC2: mode of the conv kernel for 3x3
 * stride-1 convs, 0 = per-tap, 1 = window, unset = chosen per problem; FSB_DGRAD_S2_DIRECT, FSB_WGRAD_TC, FSB_UPSAMPLE_V2,
 * FSB_DETERMINISTIC).  The environment is read once at first use; value -1 = unset.  FSB_ERR_INVALID for any other name. */
int fsb_set_option(const char* name, int value);
int fsb_get_option(const char* name);

/* Developer aid: registers a device buffer (128 uint64) for in-kernel timelines of experimental kernels.  No kernel of this
 * build writes it.  NULL disables (default). */
int fsb_debug_set_buffer(void* dev_u64x128);

/* --- weights -------------------------------------------------------------------------------- */
/* bytes of the packed fp16 weight buffer for `d` */
size_t fsb_conv_packed_bytes(const fsb_conv_desc* d);
/* w: fp32 OIHW master weight, possibly a max-width tensor: element (o,i,r,s) at
 * w[o*w_stride_o + i*w_stride_i + r*ksize + s]; only [0,Cout) x [0,Cin) is read
 * (USConv2d's weight[:out, :in] slice, search/slimmable_ops.py:42). */
int fsb_pack_conv_weight(const fsb_conv_desc* d, const float* w, int64_t w_stride_o, int64_t w_stride_i,
                         void* packed, void* stream);
/* scale = gamma / sqrt(var + eps), shift = beta - mean * scale (+ scale*conv_bias if conv_bias != NULL).
 * nn.BatchNorm2d eval forward as used at operations.py:79-83,149,221,... gamma/beta may be NULL (1/0). */
int fsb_bn_fold(int C, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                const float* conv_bias, float* scale, float* shift, void* stream);

/* --- convolution ---------------------------------------------------------------------------- */
/* y[n,ho,wo,co] = act( (sum_{r,s,ci} x[n, ho*stride + r*dil - pad + off_h, wo*stride + s*dil - pad + off_w, ci]
 *                      * w[co,ci,r,s]) * scale[co] + shift[co] )
 * x, y: fp16 NHWC with the strides in `d`; wpacked from fsb_pack_conv_weight; scale/shift fp32[Cout] or NULL;
 * stats: fp32[fsb_conv_stats_rows(d) * 2 * SC] partial rows (only with FSB_CONV_STATS; no zeroing needed).
 * Dense 3x3 / 1x1 contractions run as an im2col-free implicit GEMM on the wgmma tensor cores with TMA-staged
 * NHWC tiles; Cin < 16 (the RGB stem), x_cstride % 8 != 0, a stride-2 conv one of whose taps reads no input row or column
 * (H or W of 1) and FSB_CONV_FORCE_DIRECT use the CUDA-core direct kernel.  The choice is made from the descriptor alone
 * (fsb_conv_kernel_id, fsb_conv_stats_rows): a descriptor the wgmma kernel takes whose x or wpacked is not 16-byte aligned
 * (TMA) is FSB_ERR_INVALID, before anything is written -- it does not fall back to the direct kernel, whose statistics rows
 * would not be the fsb_conv_stats_rows(d) the caller sized the buffer for. */
int fsb_conv_fwd(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                 void* y, float* stats, void* stream);
/* which kernel fsb_conv_fwd dispatches for `d`: 0 = CUDA-core direct, 1 = the wgmma kernel conv_tc on 16x8 / 8x16 pixel tiles
 * (per-tap mode, or window mode: one halo window of the input per 64-channel chunk, taps as descriptor offsets); negative =
 * invalid descriptor.  y and with_stats are accepted for compatibility and do not change the choice. */
int fsb_conv_kernel_id(const fsb_conv_desc* d, const void* y, int with_stats);
/* number of partial statistic rows fsb_conv_fwd writes for `d` with FSB_CONV_STATS (depends on the kernel it dispatches):
 * stats must hold rows * 2 * SC floats; every row's entries of this conv's channels are written (no zeroing needed). */
int fsb_conv_stats_rows(const fsb_conv_desc* d);
/* CTAs per SM of the conv_tc launch fsb_conv_fwd makes for `d` (with stats iff d->flags has FSB_CONV_STATS): the CUDA occupancy
 * calculator's answer for the kernel instance and the dynamic shared memory the launcher picks.  Launches nothing.
 * FSB_ERR_UNSUPPORTED when `d` runs on the CUDA-core direct kernel; other negative values are errors. */
int fsb_conv_residency(const fsb_conv_desc* d);
/* fsb_conv_fwd that also writes y_half = bilinear(y, (Ho / 2, Wo / 2), align_corners=True): NHWC fp16 with pixel stride
 * y_half_cstride (a channel slice of a wider buffer is fine), bit for bit fsb_conv_fwd followed by fsb_bilinear_fwd, in one
 * launch (the conv tiles start on even pixels and each /2 pixel reads only its own 2x2 block).  FSB_ERR_UNSUPPORTED, before
 * anything is written, unless the wgmma kernel runs `d` with its TMA-store epilogue (fp16 output, Cout and y_cstride multiples
 * of 8, y 16-byte aligned), Ho and Wo are even and at most 4096, and d->flags has none of FSB_CONV_STATS, FSB_CONV_OUT_F32,
 * FSB_CONV_Y_UP2, FSB_CONV_X_DOWN2, FSB_CONV_FORCE_DIRECT: the caller then runs the two calls. */
int fsb_conv_fwd_half(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                      void* y, void* y_half, int y_half_cstride, void* stream);

/* Stem conv reading the caller's NCHW tensor directly (fp32 if x_is_f32 else fp16), 3x3 stride 2 pad 1,
 * Cin = 3, fused BN(eval)+ReLU, fp16 NHWC out.  ConvNorm at train/model_seg.py:193, search/model_search.py:148.
 * w: fp32 OIHW (read directly, no packing). */
int fsb_stem_conv_nchw(int N, int H, int W, int Cout, const void* x_nchw, int x_is_f32, const float* w,
                       const float* scale, const float* shift, void* y, int y_cstride, uint32_t flags, void* stream);

/* Same stem conv fed with the image itself: uint8 HWC frame [N, H, W, 3] (what the dataset / camera delivers) + a 3 x 256
 * fp16 lookup table of the normalised value of every byte per channel ((v / 255 - mean[c]) / std[c],
 * tools/utils/img_utils.py:179-185, applied at tools/engine/evaluator.py:329).  Zero padding applies to the NORMALISED image.
 * Bit-identical to fsb_stem_conv_nchw on the normalised fp32 frame; the host->device copy is 4x smaller. */
int fsb_stem_conv_u8hwc(int N, int H, int W, int Cout, const uint8_t* x_hwc, const void* lut_f16, const float* w,
                        const float* scale, const float* shift, void* y, int y_cstride, uint32_t flags, void* stream);
/* The stem's first two convs as one kernel: stem.0 (the RGB ConvNorm above, C0 output channels) followed by conv1 of the stride-2
 * BasicResidual2x stem.1 (3x3 stride 2 pad 1, C0 -> C1) with its BN(eval) + ReLU, without writing the 1/2-resolution map
 * (ConvNorm at train/model_seg.py:193, BasicResidual2x at search/operations.py:280-359).  in_kind: 0 = fp32 NCHW, 1 = fp16 NCHW,
 * 2 = uint8 HWC with lut_f16 as in fsb_stem_conv_u8hwc.  w0: fp32 OIHW [C0][3][3][3]; w1_packed: fsb_pack_conv_weight's layout of
 * the C0 -> C1 weight; scale / shift: folded BN of each conv.  y: fp16 NHWC 1/4-resolution map with channel stride y_cstride.
 * Bit-identical to fsb_stem_conv_nchw / fsb_stem_conv_u8hwc (AFFINE | RELU) followed by fsb_conv_fwd (AFFINE | RELU).
 * FSB_ERR_UNSUPPORTED unless 16 <= C0 <= 32, C1 == 64, y_cstride % 8 == 0 and w1_packed, y 16-byte aligned (the student's stem);
 * the caller then runs the two kernels. */
int fsb_stem_fused(int N, int H, int W, int in_kind, const void* x, const void* lut_f16, int C0, const float* w0, const float* scale0,
                   const float* shift0, int C1, const void* w1_packed, const float* scale1, const float* shift1, void* y, int y_cstride,
                   void* stream);
/* Evaluator's confusion matrix on the device (tools/seg_opr/metric.py:7-15 hist_info): for the n pixels with 0 <= gt < n_cl:
 * out[n_cl * gt + pred] += 1, out[n_cl^2] += 1 (labeled), out[n_cl^2 + 1] += (pred == gt) (correct).  out: int64
 * [n_cl * n_cl + 2], accumulated into (caller zeroes once per evaluation); gt: uint8 / int32 / int64 (gt_bytes = 1 / 4 / 8). */
int fsb_confusion_matrix(int64_t n, const uint8_t* pred, const void* gt, int gt_bytes, int n_cl, long long* out, void* stream);

/* --- resize / layout ------------------------------------------------------------------------ */
/* F.interpolate(mode='bilinear', align_corners=True) on fp16 NHWC; call sites operations.py:271,275,437,444,
 * model_search.py:339-343, model_seg.py:305,310,317.  flags: FSB_CONV_RELU applies ReLU after the resize
 * (BasicResidual_downup_*: upsample then ReLU, operations.py:275-276). */
int fsb_bilinear_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, void* y,
                     int y_cstride, uint32_t flags, void* stream);
/* Exact x2 upsample of fsb_bilinear_fwd (y: 2Hi x 2Wi, same flags) that also writes y_half = bilinear(y, (Hi, Wi)) (no ReLU),
 * bit for bit the two fsb_bilinear_fwd calls, in one launch.  FSB_ERR_UNSUPPORTED when 2Hi or 2Wi exceeds 4096. */
int fsb_bilinear_fwd_half(int N, int C, int Hi, int Wi, const void* x, int x_cstride, void* y, int y_cstride, void* y_half,
                          int y_half_cstride, uint32_t flags, void* stream);
/* Final logits upsample (model_seg.py:365, model_search.py:353-357): fp16 NHWC (C classes, cstride) low-res
 * logits -> NCHW output at (Ho, Wo), bilinear align_corners=True.  out_dtype: 0 = fp16, 1 = fp32. */
int fsb_upsample_logits_nchw(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, void* y,
                             int out_dtype, void* stream);
/* Same interpolation fused with argmax over classes -> uint8 label map [N, Ho, Wo] (first max wins, like
 * torch.argmax / np.argmax at tools/engine/evaluator.py:315-318). */
int fsb_upsample_argmax(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, uint8_t* labels,
                        void* stream);
/* The two above fused for validation (tools/engine/evaluator.py:297-318 + tools/seg_opr/metric.py:7-15): fsb_upsample_argmax of
 * the n_cl-class logits x, then fsb_confusion_matrix of those labels against gt [N, Ho, Wo] (uint8 / int32 / int64, gt_bytes =
 * 1 / 4 / 8; values outside [0, n_cl) are ignored), accumulated into out (int64 [n_cl * n_cl + 2], same layout).  The label
 * map is never written.  Bit-identical counters to the two calls; 1 <= n_cl <= 64. */
int fsb_upsample_argmax_confusion(int N, int n_cl, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, const void* gt,
                                  int gt_bytes, long long* out, void* stream);
/* fsb_upsample_argmax fused with the test-set writer's per-pixel maps (train/test.py:49-69 after
 * tools/engine/tester.py:179-204,270-291; colour map of tools/utils/visualize.py:6-21): with label = the fsb_upsample_argmax label,
 *   ids[p] = lut[label]                         (lut: C entries, NULL = identity; ids [N, Ho, Wo], or NULL)
 *   viz[p] = palette[label].use_image ? image[p] reversed to BGR : palette[label].bgr
 * palette: C x 4 bytes (B, G, R, use_image), required with viz; image: [N, Ho, Wo, 3] RGB uint8, read only where use_image is set
 * (the caller guarantees it is given then); viz: [N, Ho, Wo, 3] BGR, or NULL.  These are the bytes cv2.imwrite receives.
 * 1 <= C <= 255, at least one of ids / viz. */
int fsb_upsample_argmax_map(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, const uint8_t* lut,
                            uint8_t* ids, const uint8_t* palette, const uint8_t* image, uint8_t* viz, void* stream);
/* F.interpolate(mode='nearest') (torch's legacy rule, not 'nearest-exact') on fp16 NHWC channel slices (latency/ network,
 * latency/operations.py:265,269,427,434, latency/model_seg.py:305,309,315).  Per axis
 *   src = min((int)floorf((float)dst * ((float)in / (float)out)), in - 1)   in fp32, exactly as torch computes it.
 * C, strides multiples of 8, pointers 16-byte aligned.  No ReLU flag: a copy commutes with ReLU, apply it in the producer. */
int fsb_nearest_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, void* y, int y_cstride,
                    void* stream);
/* Final x8 logits upsample of the latency/ network (latency/model_seg.py:362) with the same index rule: NHWC fp16 -> NCHW
 * (out_dtype 0 = fp16, 1 = fp32), 16-byte stores along W. */
int fsb_upsample_logits_nearest_nchw(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, void* y,
                                     int out_dtype, void* stream);
/* argmax over classes of fsb_upsample_logits_nearest_nchw's output -> uint8 labels [N, Ho, Wo], first maximum wins; the argmax
 * is taken once per source pixel and replicated. */
int fsb_upsample_argmax_nearest(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int x_cstride, uint8_t* labels,
                                void* stream);
/* NCHW (fp32 or fp16) -> NHWC fp16 and back; plumbing for callers that hand us reference-layout tensors. */
int fsb_nchw_to_nhwc_f16(int N, int C, int H, int W, const void* x, int x_is_f32, void* y, int y_cstride,
                         void* stream);
int fsb_nhwc_f16_to_nchw(int N, int C, int H, int W, const void* x, int x_cstride, void* y, int y_is_f32,
                         void* stream);
/* strided channel-slice copy (torch.cat(dim=1) call sites that cannot be made zero-copy) */
int fsb_copy_channels(int64_t pixels, int C, const void* x, int x_cstride, void* y, int y_cstride, void* stream);

/* --- BatchNorm training path (K2/K3) -------------------------------------------------------- */
/* rows that fsb_bn_stats / fsb_bn_bwd_reduce produce for `pixels` (their buffers hold 1 + rows rows) */
int fsb_stat_rows(int64_t pixels);
/* out[c] = sum over r in [0, rows) of src[r * stride + c], c < L, added in index order in double precision */
int fsb_rowsum(int L, const float* src, int rows, int stride, float* out, void* stream);
/* per-channel sum and sum of squares over `pixels` of an fp16 NHWC tensor.  buf: (1 + fsb_stat_rows(pixels)) rows of 2*C
 * floats; rows 1.. receive the per-CTA partials, row 0 their total: buf[0..C) = sum, buf[C..2C) = sumsq. */
int fsb_bn_stats(int64_t pixels, int C, const void* x, int x_cstride, float* buf, void* stream);
/* from `rows` partial rows of statistics (row stride 2*SC floats, sums at [c], sums of squares at [SC + c]; rows = 1 for
 * totals, e.g. after an all-reduce across ranks), summed over `count` elements per channel:
 * mean, biased var -> scale/shift for the apply pass; running stats updated with momentum and UNBIASED var
 * (nn.BatchNorm2d training semantics; sequential per invocation, model_search.py:326-329). Also writes
 * save_mean / save_invstd (fp32[C]) for the backward pass when non-NULL. */
int fsb_bn_finalize(int C, const float* stats, int rows, int SC, double count, const float* gamma, const float* beta, float eps,
                    float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                    float* save_mean, float* save_invstd, void* stream);
/* y = act(x * scale[c] + shift[c]) elementwise on fp16 NHWC (in place allowed) */
int fsb_affine_act(int64_t pixels, int C, const void* x, int x_cstride, const float* scale, const float* shift,
                   void* y, int y_cstride, uint32_t flags, void* stream);

/* --- backward / training kernels (K5, K7, K8 + resize backward) ------------------------------ */
/* All gradient tensors are fp16 NHWC like activations unless stated; `gscale` is the static loss scale the caller
 * applied to the incoming gradients: parameter / scalar gradients written in fp32 are divided by it. */

/* BatchNorm(+ReLU) backward, pass 1: per-channel sums over `pixels` of dz and dz * xhat, with
 *   dz = dy * (relu ? y > 0 : 1),  xhat = (raw - mean[c]) * invstd[c]   (raw = conv output saved by the forward)
 * sums: (1 + fsb_stat_rows(pixels)) rows of 2*C floats; row 0 = totals: sums[0..C) = sum dz, sums[C..2C) = sum dz*xhat
 * (no zeroing needed; all-reduce row 0 across ranks for SyncBN). */
int fsb_bn_bwd_reduce(int64_t pixels, int C, const void* dy, int dy_cstride, const void* y, int y_cstride, const void* raw,
                      int raw_cstride, int raw_is_f32, const float* mean, const float* invstd, int relu, float* sums,
                      void* stream);
/* pass 2: draw = gamma*invstd * (dz - sum_dz/count - xhat * sum_dzxhat/count); also dgamma = sum_dzxhat/gscale,
 * dbeta = sum_dz/gscale written (accumulate = 0) or added (accumulate != 0) to fp32 dgamma/dbeta when non-NULL. */
int fsb_bn_bwd_apply(int64_t pixels, int C, const void* dy, int dy_cstride, const void* y, int y_cstride, const void* raw,
                     int raw_cstride, int raw_is_f32, const float* mean, const float* invstd, const float* gamma, const float* sums,
                     double count, int relu, void* draw, int draw_cstride, float* dgamma, float* dbeta, float gscale,
                     int accumulate, void* stream);
/* Device-selected variants (captured training graphs).  The BatchNorm parameter set is sel[*width_idx]; channels at or
 * beyond its width C get scale = shift = mean = invstd = 0 (forward) and draw = 0 (backward); gamma / beta gradients are
 * ACCUMULATED into sel[...].dgamma / dbeta.  hmax > 0 (FactorizedReduce at maximum width, C == 2*hmax): the conv outputs
 * (raw, statistics columns, draw) are in "raw" channel order [conv1 0..hmax | conv2 0..hmax) while y / dy / the parameter
 * set use the compact order [conv1 0..h | conv2 0..h | inactive], h = sel[...].C / 2; the kernels apply the bijection. */
int fsb_bn_finalize_sel(int C, const float* stats, int rows, int SC, double count, float eps, float momentum, float* scale,
                        float* shift, float* save_mean, float* save_invstd, const fsb_bn_sel* sel, const int* width_idx, int hmax,
                        void* stream);
int fsb_affine_act_sel(int64_t pixels, int C, const void* x, int x_cstride, const float* scale, const float* shift, void* y,
                       int y_cstride, uint32_t flags, const fsb_bn_sel* sel, const int* width_idx, int hmax, void* stream);
int fsb_bn_bwd_reduce_sel(int64_t pixels, int C, const void* dy, int dy_cstride, const void* y, int y_cstride, const void* raw,
                          int raw_cstride, int raw_is_f32, const float* mean, const float* invstd, int relu, float* sums,
                          const fsb_bn_sel* sel, const int* width_idx, int hmax, void* stream);
/* local_sums (may be NULL): under data parallelism `sums` are the all-reduced sums (they shape draw) while gamma / beta
 * gradients must come from this rank's own sums -- the gradient average over ranks divides by the world size afterwards. */
int fsb_bn_bwd_apply_sel(int64_t pixels, int C, const void* dy, int dy_cstride, const void* y, int y_cstride, const void* raw,
                         int raw_cstride, int raw_is_f32, const float* mean, const float* invstd, const float* sums,
                         const float* local_sums, double count, int relu, void* draw, int draw_cstride, float gscale,
                         const fsb_bn_sel* sel, const int* width_idx, int hmax, void* stream);
/* dy_in = dy * (y > 0)  (ReLU backward for affine-free paths) */
int fsb_relu_bwd(int64_t pixels, int C, const void* dy, int dy_cstride, const void* y, int y_cstride, void* dx, int dx_cstride,
                 void* stream);

/* conv data gradient (autograd of F.conv2d wrt input): dx[n,hi,wi,ci] = sum_{r,s,co} dy[n,ho,wo,co] * w[co,ci,r,s] over the
 * (ho,wo,r,s) with ho*stride + r - pad + off_h == hi (same for w).  `d` describes the FORWARD conv (x: N,H,W,Cin ...);
 * dy has d->Ho x d->Wo x Cout with pixel stride dy_cstride; dx has H x W x Cin with pixel stride dx_cstride.
 * w: fp32 OIHW master weight with strides like fsb_pack_conv_weight.  Paths, given wpacked_t (the transposed / rotated pack of
 * fsb_pack_conv_weight_dgrad), a 16-byte aligned dy and wpacked_t, and no FSB_CONV_FORCE_DIRECT:
 *   - stride 1 without an input offset: the tensor-core conv kernel (Cout >= 16, dy_cstride % 8 == 0), per-tap or window mode;
 *   - stride 2: one stride-1 tensor-core GEMM per (row, column) parity plane of dx (Cout >= 16; Cin, dx_cstride and dy_cstride
 *     multiples of 8; dx 16-byte aligned; FSB_DGRAD_S2_DIRECT=1 turns it off).  A plane that no filter tap reaches (1x1
 *     stride 2) is zeroed: only its Cin channels, so dx may be a channel slice of a wider buffer;
 *   - everything else, misaligned dy included: the direct CUDA-core kernel, which needs w (FSB_ERR_INVALID before any write
 *     without it).
 * Every dx element of the Cin channels is written; the channels beyond Cin in the pixel stride are never touched.  Argument
 * and descriptor errors return before any write; only a failure to encode a TMA tensor map or to launch (a CUDA error) can
 * follow the stride-2 zeroing. */
size_t fsb_conv_packed_dgrad_bytes(const fsb_conv_desc* d);
int fsb_pack_conv_weight_dgrad(const fsb_conv_desc* d, const float* w, int64_t w_stride_o, int64_t w_stride_i, void* packed_t,
                               void* stream);
int fsb_conv_dgrad(const fsb_conv_desc* d, const void* dy, int dy_cstride, const void* wpacked_t, const float* w,
                   int64_t w_stride_o, int64_t w_stride_i, void* dx, int dx_cstride, void* stream);
/* conv weight gradient: dw[co,ci,r,s] (+)= (1/gscale) * sum_{n,ho,wo} dy[n,ho,wo,co] * x[n, ho*stride+r-pad+off_h, ..., ci]
 * written into the fp32 OIHW gradient tensor with the master weight's strides (only the [0,Cout) x [0,Cin) corner).
 * accumulate != 0 adds to the existing contents (a cell invoked twice, model_search.py:326-329); accumulate == 0 zeroes the
 * corner first.  Elements outside the corner are never touched.  1x1 / 3x3, stride 1 or 2, dilation 1, Cin, Cout >= 16,
 * x_cstride and dy_cstride multiples of 8, 16-byte aligned x and dy, no stride-2 parity plane of x left empty (H or W of 1),
 * no FSB_CONV_FORCE_DIRECT and FSB_WGRAD_TC != 0: the tensor-core kernel; everything else (misaligned x or dy included) the
 * direct CUDA-core kernel.  Every rejection (FSB_ERR_INVALID, or a TMA tensor map that cannot be encoded) returns before dw is
 * zeroed or written.  Both kernels split the pixels over CTAs that add with fp32 atomics, except under FSB_DETERMINISTIC=1,
 * where each element has one writer and the result is bit-reproducible. */
int fsb_conv_wgrad(const fsb_conv_desc* d, const void* x, const void* dy, int dy_cstride, float* dw, int64_t w_stride_o,
                   int64_t w_stride_i, int accumulate, float gscale, void* stream);

/* bilinear (align_corners=True) backward: dx (Hi x Wi) = transpose of the forward interpolation applied to dy (Ho x Wo);
 * relu_mask_y != NULL fuses the ReLU-after-upsample backward (dy * (y > 0)). */
int fsb_bilinear_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy, int dy_cstride, const void* relu_mask_y,
                     int y_cstride, void* dx, int dx_cstride, void* stream);
/* backward of fsb_upsample_logits_nchw: dlogits NCHW (fp32 if dy_is_f32 else fp16) at (Ho, Wo) -> NHWC fp16 (Hi, Wi),
 * multiplied by gscale. */
int fsb_upsample_logits_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy_nchw, int dy_is_f32, void* dx,
                            int dx_cstride, float gscale, void* stream);
/* NCHW (fp32/fp16) gradient -> NHWC fp16 scaled by gscale (backward of fsb_nhwc_f16_to_nchw) */
int fsb_nchw_grad_to_nhwc(int N, int C, int H, int W, const void* dy, int dy_is_f32, void* dx, int dx_cstride, float gscale,
                          void* stream);

/* K5: weighted multi-tensor sum (MixedOp / beta aggregation, model_search.py:75-78,326-333):
 *   out = sum_k wts[k] * xs[k]   (K <= 8 tensors of identical shape; wts fp32[K] on the device)
 * backward: dxs[k] = wts[k] * dout (fp16), dwts[k] = <dout, xs[k]> / gscale (fp32).  dwts: (1 + fsb_wsum_rows(pixels, C))
 * rows of 8 floats (row 0 = totals, rows 1.. = per-CTA partials; no zeroing needed) or NULL. */
int fsb_wsum_rows(int64_t pixels, int C);
int fsb_wsum_fwd(int K, int64_t pixels, int C, const void* const* xs, const int* x_cstrides, const float* wts, void* out,
                 int out_cstride, void* stream);
int fsb_wsum_bwd(int K, int64_t pixels, int C, const void* dout, int dout_cstride, const void* const* xs,
                 const int* x_cstrides, const float* wts, void* const* dxs, const int* dx_cstrides, float* dwts, float gscale,
                 void* stream);
/* One training unit per call (host-overhead reduction; same kernels as the separate entry points):
 * forward  = conv (fp32 raw output + per-CTA statistic rows) -> fsb_bn_finalize (+ running stats, num_batches_tracked)
 *            -> fsb_affine_act.   vec: fp32[(6 + 2*R) * Cout], R = fsb_conv_stats_rows(d) =
 *            [sum | sumsq (totals; written under data parallelism only) | scale | shift | mean | invstd | R partial rows].
 * backward = fsb_bn_bwd_reduce -> fsb_bn_bwd_apply -> fsb_conv_dgrad (if dx) -> fsb_conv_wgrad accumulate (if dw).
 *            vec_bwd: fp32[(4 + 2*Rb) * Cout], Rb = fsb_stat_rows(N*Ho*Wo) =
 *            [sum dz | sum dz*xhat | Rb partial rows | dgamma | dbeta]; draw: fp16 NHWC scratch.  Nothing needs zeroing.
 * Both calls need Cout, raw_cstride and y_cstride (backward also dy_cstride, draw_cstride; Cout <= 2048) multiples of 8 and
 *            raw / y / vec (backward dy / y / raw / draw) 16-byte aligned; the backward also needs x when dw is given, and w
 *            and dx_cstride >= Cin when dx is given.  These arguments are checked before the first launch: a call rejected
 *            for them returns FSB_ERR_INVALID with the running statistics, num_batches_tracked and the selected set's
 *            gradients untouched.
 * sel / width_idx (may be NULL): the BatchNorm parameter set is chosen on the device, sel[*width_idx] (see fsb_bn_sel);
 *            gamma / beta / running stats arguments are then ignored and dgamma / dbeta accumulate into the selected set.
 * Data parallel: once fsb_dp_init() has created a communicator, both calls all-reduce their 2*Cout statistics over the ranks
 * on `stream` between the stages (SyncBN: global count, gamma/beta gradients from the rank-local sums); without it they are
 * single-process and SyncBN callers use the separate entry points with their own exchange. */
int fsb_conv_bn_act_train_fwd(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* gamma, const float* beta,
                              float eps, float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                              void* raw_f32, int raw_cstride, void* y, int y_cstride, float* vec, int relu,
                              const fsb_bn_sel* sel, const int* width_idx, void* stream);
int fsb_conv_bn_act_train_bwd(const fsb_conv_desc* d, const void* x, const void* dy, int dy_cstride, const void* y, int y_cstride,
                              const void* raw_f32, int raw_cstride, const float* vec_fwd, const float* gamma, int relu,
                              const void* wpacked_t, const float* w, int64_t w_stride_o, int64_t w_stride_i, void* draw,
                              int draw_cstride, float* vec_bwd, void* dx, int dx_cstride, float* dw, float gscale,
                              const fsb_bn_sel* sel, const int* width_idx, void* stream);

/* y (+)= x elementwise over a channel-slice view (gradient accumulation when a tensor feeds several consumers) */
int fsb_add_inplace(int64_t pixels, int C, const void* x, int x_cstride, void* y, int y_cstride, void* stream);

/* ---- data-parallel exchange (SURVEY section 8e; replaces the SyncBN / gradient all-reduce a DDP port of
 * search/train_search.py:215-256 and train/train.py:219-271 would issue through torch.distributed) --------------------------
 * One process per GPU.  Rank 0 obtains a 128-byte NCCL id (fsb_dp_unique_id), the launcher broadcasts it by any means,
 * every rank calls fsb_dp_init(id, rank, world) with its device current (collective).  From then on the fused training
 * units exchange their BatchNorm statistics themselves and fsb_dp_allreduce_f32 sums fp32 buffers (gradient buckets) in
 * place on the given stream.  NCCL is loaded with dlopen at first use; fsb_dp_world() is 1 until fsb_dp_init succeeded. */
int fsb_dp_unique_id(void* out128);
int fsb_dp_init(const void* id128, int rank, int world);
int fsb_dp_world(void);
int fsb_dp_enable(int on); /* 0: keep the communicator but behave single-process (fsb_dp_world() == 1) until re-enabled */
int fsb_dp_allreduce_f32(void* buf, int64_t n, void* stream);
int fsb_dp_shutdown(void);

/* Peer-memory exchange for the latency-bound part of data parallelism: the per-unit SyncBN statistics (<= 4096 floats each,
 * ~7 000 per supernet step), summed over the ranks IN RANK ORDER by a single-block kernel through buffers the ranks map into
 * each other with CUDA IPC (NVLink / NVSwitch peer access) -- no host involvement, capturable in CUDA graphs, bit-identical
 * results on every rank.  Launcher: every rank calls fsb_peer_alloc (64-byte IPC handle out), all-gathers the handles by any
 * means, calls fsb_peer_open(all handles, rank, world) and barriers.  From then on fsb_dp_world() == world, the fused training
 * units exchange through peer memory, and fsb_dp_allreduce_f32 still serves large buffers (NCCL, if fsb_dp_init was called).
 * Exchanges are issued inside REGIONS (fsb_peer_begin(region, stream): one per captured graph / eager pass); every rank must
 * issue the same regions with the same sequence of exchanges. */
int fsb_peer_alloc(void* handle_out64);
int fsb_peer_open(const void* handles, int rank, int world);
int fsb_peer_world(void);
int fsb_peer_enable(int on);
int fsb_peer_begin(int region, void* stream);
int fsb_peer_allreduce_f32(void* buf, int64_t n, void* stream);
int fsb_peer_shutdown(void);

/* N1 (SURVEY 8f): the drivers' training criteria evaluated from the LOW-RESOLUTION logits -- no label-resolution class tensor exists.
 * Replaces, for the fused path, tools/seg_opr/loss_opr.py:63-93 (ProbOhemCrossEntropy2d on F.interpolate'd logits,
 * train/model_seg.py:357-362) and train/train.py:254-260 (KLDivLoss(log_softmax(student), softmax(teacher))).
 * logits: NHWC fp16 (N, Hi, Wi, C <= 32) with channel stride a multiple of 8 >= round8(C); labels int64 (N, Ho, Wo);
 * the upsample is bilinear with align_corners=True to (Ho, Wo).
 *   fsb_loss_logp_fwd : per label pixel, logp_t = log softmax(up(logits))[target] (0 for ignored / out-of-range labels, i.e.
 *                       probability 1 like loss_opr.py:73) and lse = log-sum-exp of the interpolated logits.
 *   fsb_kth_smallest_f32 : exact k-th smallest (1-based) of n floats into *out (device), three radix-histogram passes, no sort;
 *                       workspace of fsb_kth_workspace_bytes() bytes.
 *   fsb_ohem_reduce   : out2 = {sum(-logp_t * kept), count(kept)}, kept = valid label & logp_t <= *thr (thr NULL: every valid
 *                       pixel); partial needs 2 * fsb_loss_rows() floats; fixed-order reduction.
 *   fsb_loss_ce_bwd   : dlogits (NHWC fp16, stride dcs) (+)= gscale * *coef * sum over kept label pixels of
 *                       bilinear weight * (softmax - onehot); gather form, no atomics.
 *   fsb_loss_kl_fwd   : out2[0] = sum over label pixels and classes of q (log q - log p), p = softmax(up(student)),
 *                       q = softmax(up(teacher)); stores both log-sum-exps.   fsb_loss_kl_bwd: dstudent (+)= gscale * *coef * (p - q)^T. */
int fsb_loss_logp_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* logits, int cstride, const int64_t* target,
                      int ignore_label, float* logp_t, float* lse, void* stream);
size_t fsb_kth_workspace_bytes(void);
int fsb_kth_smallest_f32(const float* x, int64_t n, int64_t k, float* out, void* workspace, void* stream);
int fsb_loss_rows(void);
int fsb_ohem_reduce(const float* logp_t, const int64_t* target, int64_t n, int ignore_label, int C, const float* thr, float* partial,
                    float* out2, void* stream);
int fsb_loss_ce_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* logits, int cstride, const int64_t* target,
                    int ignore_label, const float* lse, const float* logp_t, const float* thr, const float* coef, void* dlogits,
                    int dcs, float gscale, int accumulate, void* stream);
int fsb_loss_kl_fwd(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* student, int scs, const void* teacher,
                    int tcs, float* lse_s, float* lse_t, float* partial, float* out2, void* stream);
int fsb_loss_kl_bwd(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* student, int scs, const void* teacher,
                    int tcs, const float* lse_s, const float* lse_t, const float* coef, void* dstudent, int dcs, float gscale,
                    int accumulate, void* stream);

/* Step tail on the flat gradient buffer of the captured passes: nn.utils.clip_grad_norm_ + torch.optim.SGD(momentum, weight_decay)
 * (search/train_search.py:249-250, train/train.py:269) as table-driven kernels instead of a Python walk over ~5 000 tensors.
 * segs: array of {float* param, uint32 offset into G / M, uint32 numel} (16 bytes each); map: int32 pairs {segment, chunk} for every
 * fsb_flat_chunk()-element chunk of every segment; live: one byte per segment (parameters without a gradient this step are skipped,
 * like torch skips `grad is None`).  fsb_flat_grad_norm: out2 = {total 2-norm of the live gradients (+ sqrt-folded *extra_sq),
 * min(1, max_norm / (norm + 1e-6))}, fixed summation order; partial: nblocks floats.  fsb_flat_scale: G *= *coef on the live segments.
 * fsb_flat_sgd: d = g + wd * p; m = momentum * m + d; p -= lr * m. */
int fsb_flat_chunk(void);
int fsb_flat_grad_norm(const void* map, int nblocks, const void* segs, const uint8_t* live, const float* G, float* partial,
                       const float* extra_sq, float max_norm, float* out2, void* stream);
int fsb_flat_scale(const void* map, int nblocks, const void* segs, const uint8_t* live, float* G, const float* coef, void* stream);
int fsb_flat_sgd(const void* map, int nblocks, const void* segs, const uint8_t* live, const float* G, float* M, float lr, float momentum,
                 float weight_decay, void* stream);

/* K14: the supernet's expected latency, search/model_search.py:361-475 (Network_Multi_Path.forward_latency, called three times per
 * architect step by search/architect.py:60-74, then loss_latency.backward()), as one launch forward and one backward with no host
 * synchronisation.  `plan` is the int32 walk description built by fasterseg_b200/supernet_latency.py (header, constants, MixedOp
 * terms with their [5][n_w][n_w] latency slices, the settle recurrence as ADD / MUL instructions, CSR use lists); the kernels read
 * the device copy `plan`, the host copy `plan_host` sizes the launch.  Arch parameters are one architecture's fp32 logits
 * (alphas [L|L-1|L-2][5], betas [L-2|L-3][2], ratios [L-1|L-1|L-2][n_w]); a tensor the plan's flags do not use may be NULL.
 *   noise : gumbel uniforms [ratio rows][n_w] (arch_ratio sampling), else the forced width index of every ratio row (as float).
 *   fsb_supernet_latency_fwd : *out = expected latency (ms); saves what the backward needs in `workspace`
 *                              (fsb_supernet_latency_workspace_bytes(plan_host) bytes, caller-owned, kept until the backward).
 *   fsb_supernet_latency_bwd : d/d(logits) of *gout * latency, written (not accumulated) in full for every tensor the plan
 *                              differentiates: alphas / betas through their softmax, ratios through the straight-through gumbel
 *                              sample (model_search.py:13-43).  Deterministic (fixed summation order, no atomics). */
size_t fsb_supernet_latency_workspace_bytes(const int32_t* plan_host);
int fsb_supernet_latency_fwd(const int32_t* plan_host, const int32_t* plan, const float* alpha0, const float* alpha1, const float* alpha2,
                             const float* beta1, const float* beta2, const float* ratio0, const float* ratio1, const float* ratio2,
                             const float* noise, float* workspace, float* out, void* stream);
int fsb_supernet_latency_bwd(const int32_t* plan_host, const int32_t* plan, const float* gout, const float* workspace, float* dalpha0,
                             float* dalpha1, float* dalpha2, float* dbeta1, float* dbeta2, float* dratio0, float* dratio1, float* dratio2,
                             void* stream);

/* --- training augmentation ------------------------------------------------------------------ */
/* Batch geometry of fsb_train_pre: the crop (config.image_height x image_width) and the label map it is resized to
 * (image_height / gt_down_sampling x image_width / gt_down_sampling, train/dataloader.py:25). */
typedef struct fsb_train_pre_desc {
  int32_t n;        /* images */
  int32_t crop_h, crop_w;
  int32_t label_h, label_w; /* 1 <= label_h <= crop_h, 1 <= label_w <= crop_w */
} fsb_train_pre_desc;

/* TrainPre.__call__ (train/dataloader.py:14-31, same in search/dataloader.py) for a batch, after the host drew its random numbers.
 * img: uint8 HWC RGB sources (the dataset's img[:, :, ::-1]) and gt: uint8 HW labels, packed back to back; geom: int32 [n][8]
 * = {H, W, mirror, sh, sw, pos_h, pos_w, pixel offset of image i in img (x3 bytes) and gt}, with 0 <= pos_h < sh,
 * 0 <= pos_w < sw; lut: float [3][256] normalisation table.  Writes
 *   out_img float [n][3][crop_h][crop_w]: random_mirror (tools/utils/img_utils.py:125-130), the cv2.resize INTER_LINEAR of
 *     random_scale (:105-112), normalize (:179-184) as lut[c][v], random_crop_pad_to_shape (:24-39, pad_image_to_shape :60-74)
 *     with 0 in the padding;
 *   out_gt int64 [n][label_h][label_w]: the label mirrored, INTER_NEAREST resized to (sh, sw), cropped and padded with 255, then
 *     INTER_NEAREST resized to (label_h, label_w) (train/dataloader.py:25).
 * The resizes reproduce OpenCV's 8-bit integer arithmetic (fasterseg_b200/csrc/trainpre.cu), so with lut built from the same
 * float64 expression as normalize, both outputs are bit-identical to the reference's tensors. */
int fsb_train_pre(const fsb_train_pre_desc* desc, const uint8_t* img, const uint8_t* gt, const int32_t* geom, const float* lut,
                  float* out_img, int64_t* out_gt, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FSB200_H_ */
