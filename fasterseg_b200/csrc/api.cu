// api.cu -- the extern "C" surface of libfsb200.so (declared in include/fsb200.h).
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "fsb_internal.h"

namespace fsb {

static thread_local char g_err[512] = "";
thread_local cudaError_t g_launch_err = cudaSuccess;

int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
int set_cuda_error(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorString(e), cudaGetErrorName(e));
  return FSB_ERR_CUDA;
}

static int g_pdl = -1;
bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("FSB_PDL");
    g_pdl = (e && e[0] == '0') ? 0 : 1;
  }
  return g_pdl != 0;
}
int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

static const char* const kOptNames[OPT_COUNT] = {"FSB_CONV_TC2", "FSB_DGRAD_S2_DIRECT", "FSB_WGRAD_TC", "FSB_UPSAMPLE_V2",
                                                 "FSB_DETERMINISTIC"};
static int g_opts[OPT_COUNT];
static std::once_flag g_opts_once;
static void load_opts() {
  for (int i = 0; i < OPT_COUNT; ++i) {
    const char* e = getenv(kOptNames[i]);
    g_opts[i] = (e && e[0]) ? atoi(e) : -1;
  }
}
int opt(Opt o) {
  std::call_once(g_opts_once, load_opts);
  return g_opts[o];
}

int ensure_dyn_smem(const void* kernel, int bytes, const char* what) {
  struct Entry { const void* k; unsigned long long mask; };
  static Entry table[64];
  static int n = 0;
  static std::mutex mu;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_cuda_error(e, "cudaGetDevice");
  const unsigned long long bit = 1ull << (dev & 63);
  std::lock_guard<std::mutex> lock(mu);
  Entry* hit = nullptr;
  for (int i = 0; i < n; ++i)
    if (table[i].k == kernel) hit = &table[i];
  if (hit && (hit->mask & bit)) return FSB_OK;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_cuda_error(e, what);
  if (!hit && n < 64) {
    table[n].k = kernel;
    table[n].mask = 0;
    hit = &table[n++];
  }
  if (hit) hit->mask |= bit;
  return FSB_OK;
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// defined in the other translation units
int pack_conv_weight(const fsb_conv_desc*, const float*, int64_t, int64_t, void*, cudaStream_t);
int stem_conv_nchw_launch(int, int, int, int, const void*, int, const float*, const float*, const float*, void*, int, uint32_t,
                          cudaStream_t);
int stem_conv_u8hwc_launch(int, int, int, int, const uint8_t*, const void*, const float*, const float*, const float*, void*, int, uint32_t,
                           cudaStream_t);
int stem_fused_launch(int, int, int, int, const void*, const void*, int, const float*, const float*, const float*, int, const void*,
                      const float*, const float*, void*, int, cudaStream_t);
int confusion_launch(int64_t, const uint8_t*, const void*, int, int, long long*, cudaStream_t);
int bilinear_launch(int, int, int, int, int, int, const void*, int, void*, int, uint32_t, cudaStream_t);
int bilinear_up2_half_launch(int, int, int, int, const void*, int, void*, int, void*, int, uint32_t, cudaStream_t);
int upsample_logits_launch(int, int, int, int, int, int, const void*, int, void*, int, cudaStream_t);
int upsample_argmax_launch(int, int, int, int, int, int, const void*, int, uint8_t*, cudaStream_t);
int upsample_argmax_confusion_launch(int, int, int, int, int, int, const void*, int, const void*, int, long long*, cudaStream_t);
int upsample_argmax_map_launch(int, int, int, int, int, int, const void*, int, const uint8_t*, uint8_t*, const uint8_t*, const uint8_t*,
                               uint8_t*, cudaStream_t);
int train_pre_launch(const fsb_train_pre_desc&, const uint8_t*, const uint8_t*, const int32_t*, const float*, float*, long long*,
                     cudaStream_t);
int nearest_launch(int, int, int, int, int, int, const void*, int, void*, int, cudaStream_t);
int upsample_logits_nearest_launch(int, int, int, int, int, int, const void*, int, void*, int, cudaStream_t);
int upsample_argmax_nearest_launch(int, int, int, int, int, int, const void*, int, uint8_t*, cudaStream_t);
int nchw_to_nhwc_launch(int, int, int, int, const void*, int, void*, int, cudaStream_t);
int nhwc_to_nchw_launch(int, int, int, int, const void*, int, void*, int, cudaStream_t);
int copy_channels_launch(int64_t, int, const void*, int, void*, int, cudaStream_t);
int bn_fold_launch(int, const float*, const float*, const float*, const float*, float, const float*, float*, float*, cudaStream_t);
int bn_stats_launch(int64_t, int, const void*, int, int, float*, cudaStream_t);
int wsum_rows(int64_t, int);
int rowsum_launch(int, const float*, int, int, float*, cudaStream_t);
int bn_finalize_launch(int, const float*, int, int, double, const float*, const float*, float, float, float*, float*, float*, float*,
                       float*, float*, cudaStream_t, long long* = nullptr, const fsb_bn_sel* = nullptr, const int* = nullptr, int = 0);
int affine_act_launch(int64_t, int, const void*, int, const float*, const float*, void*, int, uint32_t, cudaStream_t,
                      const fsb_bn_sel* = nullptr, const int* = nullptr, int = 0);

int bn_bwd_reduce_launch(int64_t, int, const void*, int, const void*, int, const void*, int, int, const float*, const float*, int,
                         float*, cudaStream_t, const fsb_bn_sel* = nullptr, const int* = nullptr, int = 0);
int bn_bwd_apply_launch(int64_t, int, const void*, int, const void*, int, const void*, int, int, const float*, const float*,
                        const float*, const float*, double, int, void*, int, float*, float*, float, cudaStream_t, int = 1,
                        const fsb_bn_sel* = nullptr, const int* = nullptr, int = 0, const float* = nullptr);
int relu_bwd_launch(int64_t, int, const void*, int, const void*, int, void*, int, cudaStream_t);
fsb_conv_desc dgrad_as_fwd_desc(const fsb_conv_desc*, int, int);
int pack_dgrad_launch(const fsb_conv_desc*, const float*, int64_t, int64_t, void*, cudaStream_t);
int conv_dgrad_launch(const fsb_conv_desc*, const void*, int, const void*, const float*, int64_t, int64_t, void*, int, cudaStream_t);
int conv_wgrad_launch(const fsb_conv_desc*, const void*, const void*, int, float*, int64_t, int64_t, int, float, cudaStream_t);
int bilinear_bwd_launch(int, int, int, int, int, int, const void*, int, const void*, int, void*, int, cudaStream_t);
int upsample_logits_bwd_launch(int, int, int, int, int, int, const void*, int, void*, int, float, cudaStream_t);
int loss_logp_fwd_launch(int, int, int, int, int, int, const void*, int, const long long*, int, float*, float*, cudaStream_t);
size_t kth_workspace_bytes();
int kth_smallest_launch(const float*, int64_t, int64_t, float*, void*, cudaStream_t);
int loss_rows();
int ohem_reduce_launch(const float*, const long long*, int64_t, int, int, const float*, float*, float*, cudaStream_t);
int loss_ce_bwd_launch(int, int, int, int, int, int, const void*, int, const long long*, int, const float*, const float*, const float*,
                       const float*, void*, int, float, int, cudaStream_t);
int loss_kl_fwd_launch(int, int, int, int, int, int, int, int, const void*, int, const void*, int, float*, float*, float*, float*, cudaStream_t);
int loss_kl_bwd_launch(int, int, int, int, int, int, int, int, const void*, int, const void*, int, const float*, const float*, const float*,
                       void*, int, float, int, cudaStream_t);
int nchw_grad_to_nhwc_launch(int, int, int, int, const void*, int, void*, int, float, cudaStream_t);
int wsum_fwd_launch(int, int64_t, int, const void* const*, const int*, const float*, void*, int, cudaStream_t);
int wsum_bwd_launch(int, int64_t, int, const void*, int, const void* const*, const int*, const float*, void* const*, const int*,
                    float*, float, cudaStream_t);
int add_inplace_launch(int64_t, int, const void*, int, void*, int, cudaStream_t);

// device buffer for in-kernel timelines of experimental kernels (fsb_debug_set_buffer); no kernel of this build writes it
unsigned long long* g_dbg_buffer = nullptr;

static int check_desc(const fsb_conv_desc* d) {
  if (!d) return set_error(FSB_ERR_INVALID, "null conv desc");
  if (d->N <= 0 || d->H <= 0 || d->W <= 0 || d->Cin <= 0 || d->Cout <= 0)
    return set_error(FSB_ERR_INVALID, "conv desc: non-positive dimension");
  if (!(d->ksize == 1 || d->ksize == 3)) return set_error(FSB_ERR_INVALID, "conv desc: ksize must be 1 or 3");
  if (!(d->stride == 1 || d->stride == 2)) return set_error(FSB_ERR_INVALID, "conv desc: stride must be 1 or 2");
  if (d->dil < 1) return set_error(FSB_ERR_INVALID, "conv desc: dil must be >= 1");
  if (d->x_cstride < d->Cin || d->y_cstride < d->Cout) return set_error(FSB_ERR_INVALID, "conv desc: channel stride < channels");
  const int He = d->H - d->off_h, We = d->W - d->off_w;
  const int ext = d->dil * (d->ksize - 1) + 1;
  const int Ho = (He + 2 * d->pad - ext) / d->stride + 1, Wo = (We + 2 * d->pad - ext) / d->stride + 1;
  if (Ho != d->Ho || Wo != d->Wo) {
    char buf[160];
    snprintf(buf, sizeof(buf), "conv desc: Ho/Wo (%d,%d) inconsistent with geometry (expected %d,%d)", d->Ho, d->Wo, Ho, Wo);
    return set_error(FSB_ERR_INVALID, buf);
  }
  return FSB_OK;
}

}  // namespace fsb

using namespace fsb;

extern "C" {

int fsb_abi_version(void) { return FSB_ABI_VERSION; }
const char* fsb_last_error_string(void) { return g_err; }

int fsb_set_pdl(int enabled) {
  g_pdl = enabled ? 1 : 0;
  return FSB_OK;
}

static int find_opt(const char* name) {
  if (!name) return -1;
  for (int i = 0; i < OPT_COUNT; ++i)
    if (strcmp(name, kOptNames[i]) == 0) return i;
  return -1;
}
int fsb_set_option(const char* name, int value) {
  const int i = find_opt(name);
  if (i < 0) return set_error(FSB_ERR_INVALID, "fsb_set_option: unknown option");
  opt(static_cast<Opt>(i));  // make sure the environment has been read, then override
  g_opts[i] = value;
  return FSB_OK;
}
int fsb_get_option(const char* name) {
  const int i = find_opt(name);
  return i < 0 ? -1 : opt(static_cast<Opt>(i));
}

int fsb_conv_stats_rows(const fsb_conv_desc* d) {
  if (check_desc(d)) return 0;
  return conv_plan(d).stat_rows;
}
int fsb_conv_kernel_id(const fsb_conv_desc* d, const void* y, int with_stats) {
  if (check_desc(d)) return -1;
  (void)y;
  (void)with_stats;
  return conv_plan(d).direct ? 0 : 1;
}
int fsb_conv_residency(const fsb_conv_desc* d) {
  int rc = check_desc(d);
  if (rc) return rc;
  const ConvPlan plan = conv_plan(d);
  if (plan.direct) return set_error(FSB_ERR_UNSUPPORTED, "conv_residency: the descriptor runs on the direct kernel");
  return plan.rc ? plan.rc : conv_tc_occupancy(plan);
}
int fsb_stat_rows(int64_t pixels) { return stat_rows(pixels); }
int fsb_wsum_rows(int64_t pixels, int C) { return wsum_rows(pixels, C); }
int fsb_rowsum(int L, const float* src, int rows, int stride, float* out, void* stream) {
  if (L <= 0 || rows <= 0 || !src || !out || stride < L) return set_error(FSB_ERR_INVALID, "rowsum: bad argument");
  return rowsum_launch(L, src, rows, stride, out, static_cast<cudaStream_t>(stream));
}

int fsb_debug_set_buffer(void* dev_u64x128) {
  g_dbg_buffer = static_cast<unsigned long long*>(dev_u64x128);
  return FSB_OK;
}

int fsb_loss_logp_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* logits, int cstride, const int64_t* target,
                      int ignore_label, float* logp_t, float* lse, void* stream) {
  return loss_logp_fwd_launch(N, C, Hi, Wi, Ho, Wo, logits, cstride, reinterpret_cast<const long long*>(target), ignore_label, logp_t, lse,
                              static_cast<cudaStream_t>(stream));
}
size_t fsb_kth_workspace_bytes(void) { return kth_workspace_bytes(); }
int fsb_kth_smallest_f32(const float* x, int64_t n, int64_t k, float* out, void* workspace, void* stream) {
  return kth_smallest_launch(x, n, k, out, workspace, static_cast<cudaStream_t>(stream));
}
int fsb_loss_rows(void) { return loss_rows(); }
int fsb_ohem_reduce(const float* logp_t, const int64_t* target, int64_t n, int ignore_label, int C, const float* thr, float* partial,
                    float* out2, void* stream) {
  return ohem_reduce_launch(logp_t, reinterpret_cast<const long long*>(target), n, ignore_label, C, thr, partial, out2,
                            static_cast<cudaStream_t>(stream));
}
int fsb_loss_ce_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* logits, int cstride, const int64_t* target,
                    int ignore_label, const float* lse, const float* logp_t, const float* thr, const float* coef, void* dlogits,
                    int dcs, float gscale, int accumulate, void* stream) {
  return loss_ce_bwd_launch(N, C, Hi, Wi, Ho, Wo, logits, cstride, reinterpret_cast<const long long*>(target), ignore_label, lse, logp_t, thr,
                            coef, dlogits, dcs, gscale, accumulate, static_cast<cudaStream_t>(stream));
}
int fsb_loss_kl_fwd(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* student, int scs, const void* teacher,
                    int tcs, float* lse_s, float* lse_t, float* partial, float* out2, void* stream) {
  return loss_kl_fwd_launch(N, C, Hs, Ws, Ht, Wt, Ho, Wo, student, scs, teacher, tcs, lse_s, lse_t, partial, out2,
                            static_cast<cudaStream_t>(stream));
}
int fsb_loss_kl_bwd(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* student, int scs, const void* teacher,
                    int tcs, const float* lse_s, const float* lse_t, const float* coef, void* dstudent, int dcs, float gscale,
                    int accumulate, void* stream) {
  return loss_kl_bwd_launch(N, C, Hs, Ws, Ht, Wt, Ho, Wo, student, scs, teacher, tcs, lse_s, lse_t, coef, dstudent, dcs, gscale, accumulate,
                            static_cast<cudaStream_t>(stream));
}

int fsb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error(FSB_ERR_NO_DEVICE, "no CUDA device");
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return set_cuda_error(e, "cudaGetDeviceProperties");
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return FSB_OK;
}

size_t fsb_conv_packed_bytes(const fsb_conv_desc* d) {
  if (!d || d->Cin <= 0 || d->Cout <= 0) return 0;
  const ConvGeom g = conv_geom(d);
  return static_cast<size_t>(g.taps) * g.npad * g.kpad * 2;
}

int fsb_pack_conv_weight(const fsb_conv_desc* d, const float* w, int64_t so, int64_t si, void* packed, void* stream) {
  if (!d || !w || !packed) return set_error(FSB_ERR_INVALID, "pack_conv_weight: null argument");
  return pack_conv_weight(d, w, so, si, packed, static_cast<cudaStream_t>(stream));
}

int fsb_bn_fold(int C, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                const float* conv_bias, float* scale, float* shift, void* stream) {
  if (C <= 0 || !mean || !var || !scale || !shift) return set_error(FSB_ERR_INVALID, "bn_fold: bad argument");
  return bn_fold_launch(C, gamma, beta, mean, var, eps, conv_bias, scale, shift, static_cast<cudaStream_t>(stream));
}

int fsb_conv_fwd(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift, void* y,
                 float* stats, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  if (!x || !wpacked || !y) return set_error(FSB_ERR_INVALID, "conv_fwd: null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const ConvPlan plan = conv_plan(d);
  if (plan.rc) return plan.rc;
  if (plan.direct) return conv_direct_launch(d, x, wpacked, scale, shift, y, stats, st);
  return conv_tc_launch(plan, d, x, wpacked, scale, shift, y, stats, st);
}

int fsb_conv_fwd_half(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift, void* y,
                      void* y_half, int y_half_cstride, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  if (!x || !wpacked || !y || !y_half) return set_error(FSB_ERR_INVALID, "conv_fwd_half: null pointer");
  if (y_half_cstride < d->Cout || (y_half_cstride % 8) || (reinterpret_cast<uintptr_t>(y_half) & 15))
    return set_error(FSB_ERR_INVALID, "conv_fwd_half: y_half_cstride must be >= Cout and a multiple of 8, y_half 16-byte aligned");
  if (d->flags & (FSB_CONV_STATS | FSB_CONV_OUT_F32 | FSB_CONV_Y_UP2 | FSB_CONV_X_DOWN2 | FSB_CONV_FORCE_DIRECT))
    return set_error(FSB_ERR_UNSUPPORTED, "conv_fwd_half: no FSB_CONV_STATS / OUT_F32 / Y_UP2 / X_DOWN2 / FORCE_DIRECT");
  if ((d->Ho % 2) || (d->Wo % 2) || d->Ho > kBilinearLocalMax || d->Wo > kBilinearLocalMax)
    return set_error(FSB_ERR_UNSUPPORTED, "conv_fwd_half: Ho and Wo must be even and at most kBilinearLocalMax");
  const ConvPlan plan = conv_plan(d);
  if (plan.rc) return plan.rc;
  if (plan.direct) return set_error(FSB_ERR_UNSUPPORTED, "conv_fwd_half: this problem runs on the direct kernel");
  const ConvHalfOut half = {y_half, y_half_cstride};
  return conv_tc_launch(plan, d, x, wpacked, scale, shift, y, nullptr, static_cast<cudaStream_t>(stream), nullptr, &half);
}

int fsb_stem_conv_nchw(int N, int H, int W, int Cout, const void* x, int x_is_f32, const float* w, const float* scale,
                       const float* shift, void* y, int y_cstride, uint32_t flags, void* stream) {
  if (N <= 0 || H <= 0 || W <= 0 || Cout <= 0 || !x || !w || !y || y_cstride < Cout)
    return set_error(FSB_ERR_INVALID, "stem_conv_nchw: bad argument");
  return stem_conv_nchw_launch(N, H, W, Cout, x, x_is_f32, w, scale, shift, y, y_cstride, flags, static_cast<cudaStream_t>(stream));
}

int fsb_stem_conv_u8hwc(int N, int H, int W, int Cout, const uint8_t* x, const void* lut_f16, const float* w, const float* scale,
                        const float* shift, void* y, int y_cstride, uint32_t flags, void* stream) {
  if (N <= 0 || H <= 0 || W <= 0 || Cout <= 0 || !x || !lut_f16 || !w || !y || y_cstride < Cout)
    return set_error(FSB_ERR_INVALID, "stem_conv_u8hwc: bad argument");
  return stem_conv_u8hwc_launch(N, H, W, Cout, x, lut_f16, w, scale, shift, y, y_cstride, flags, static_cast<cudaStream_t>(stream));
}
int fsb_stem_fused(int N, int H, int W, int in_kind, const void* x, const void* lut_f16, int C0, const float* w0, const float* scale0,
                   const float* shift0, int C1, const void* w1_packed, const float* scale1, const float* shift1, void* y, int y_cstride,
                   void* stream) {
  if (N <= 0 || H <= 0 || W <= 0 || in_kind < 0 || in_kind > 2 || !x || (in_kind == 2 && !lut_f16) || !w0 || !scale0 || !shift0 ||
      !w1_packed || !scale1 || !shift1 || !y || C1 <= 0 || y_cstride < C1)
    return set_error(FSB_ERR_INVALID, "stem_fused: bad argument");
  return stem_fused_launch(N, H, W, in_kind, x, lut_f16, C0, w0, scale0, shift0, C1, w1_packed, scale1, shift1, y, y_cstride,
                           static_cast<cudaStream_t>(stream));
}
int fsb_confusion_matrix(int64_t n, const uint8_t* pred, const void* gt, int gt_bytes, int n_cl, long long* out, void* stream) {
  if (n <= 0 || !pred || !gt || !out) return set_error(FSB_ERR_INVALID, "confusion_matrix: bad argument");
  return confusion_launch(n, pred, gt, gt_bytes, n_cl, out, static_cast<cudaStream_t>(stream));
}

int fsb_bilinear_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int ycs, uint32_t flags,
                     void* stream) {
  if (N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || !y) return set_error(FSB_ERR_INVALID, "bilinear: bad argument");
  return bilinear_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, y, ycs, flags, static_cast<cudaStream_t>(stream));
}

int fsb_bilinear_fwd_half(int N, int C, int Hi, int Wi, const void* x, int xcs, void* y, int ycs, void* y_half, int yhcs,
                          uint32_t flags, void* stream) {
  if (N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || !x || !y || !y_half) return set_error(FSB_ERR_INVALID, "bilinear_fwd_half: bad argument");
  return bilinear_up2_half_launch(N, C, Hi, Wi, x, xcs, y, ycs, y_half, yhcs, flags, static_cast<cudaStream_t>(stream));
}

int fsb_upsample_logits_nchw(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int out_dtype,
                             void* stream) {
  if (N <= 0 || C <= 0 || !x || !y || xcs < C) return set_error(FSB_ERR_INVALID, "upsample_logits: bad argument");
  return upsample_logits_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, y, out_dtype, static_cast<cudaStream_t>(stream));
}

int fsb_upsample_argmax(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, uint8_t* labels, void* stream) {
  if (N <= 0 || C <= 0 || C > 255 || !x || !labels || xcs < C) return set_error(FSB_ERR_INVALID, "upsample_argmax: bad argument");
  return upsample_argmax_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, labels, static_cast<cudaStream_t>(stream));
}
int fsb_upsample_argmax_confusion(int N, int n_cl, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const void* gt, int gt_bytes,
                                  long long* out, void* stream) {
  if (N <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || !gt || !out || xcs < n_cl)
    return set_error(FSB_ERR_INVALID, "upsample_argmax_confusion: bad argument");
  return upsample_argmax_confusion_launch(N, n_cl, Hi, Wi, Ho, Wo, x, xcs, gt, gt_bytes, out, static_cast<cudaStream_t>(stream));
}
int fsb_upsample_argmax_map(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const uint8_t* lut, uint8_t* ids,
                            const uint8_t* palette, const uint8_t* image, uint8_t* viz, void* stream) {
  if (N <= 0 || C < 1 || C > 255 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || xcs < C || (!ids && !viz) || (viz && !palette))
    return set_error(FSB_ERR_INVALID, "upsample_argmax_map: bad argument");
  return upsample_argmax_map_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, lut, ids, palette, image, viz, static_cast<cudaStream_t>(stream));
}
int fsb_train_pre(const fsb_train_pre_desc* d, const uint8_t* img, const uint8_t* gt, const int32_t* geom, const float* lut,
                  float* out_img, int64_t* out_gt, void* stream) {
  if (!d || d->n <= 0 || d->n > 65535 || d->crop_h <= 0 || d->crop_h > 65535 || d->crop_w <= 0 || d->label_h <= 0 ||
      d->label_h > d->crop_h || d->label_w <= 0 || d->label_w > d->crop_w || !img || !gt || !geom || !lut || !out_img || !out_gt)
    return set_error(FSB_ERR_INVALID, "train_pre: bad argument");
  return train_pre_launch(*d, img, gt, geom, lut, out_img, reinterpret_cast<long long*>(out_gt), static_cast<cudaStream_t>(stream));
}

int fsb_nearest_fwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int ycs, void* stream) {
  if (N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || !y || xcs < C || ycs < C)
    return set_error(FSB_ERR_INVALID, "nearest: bad argument");
  return nearest_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, y, ycs, static_cast<cudaStream_t>(stream));
}
int fsb_upsample_logits_nearest_nchw(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int out_dtype,
                                     void* stream) {
  if (N <= 0 || C <= 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || !y || xcs < C || (out_dtype != 0 && out_dtype != 1))
    return set_error(FSB_ERR_INVALID, "upsample_logits_nearest: bad argument");
  return upsample_logits_nearest_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, y, out_dtype, static_cast<cudaStream_t>(stream));
}
int fsb_upsample_argmax_nearest(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, uint8_t* labels, void* stream) {
  if (N <= 0 || C <= 0 || C > 255 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x || !labels || xcs < C)
    return set_error(FSB_ERR_INVALID, "upsample_argmax_nearest: bad argument");
  return upsample_argmax_nearest_launch(N, C, Hi, Wi, Ho, Wo, x, xcs, labels, static_cast<cudaStream_t>(stream));
}

int fsb_nchw_to_nhwc_f16(int N, int C, int H, int W, const void* x, int x_is_f32, void* y, int ycs, void* stream) {
  if (N <= 0 || C <= 0 || !x || !y || ycs < C) return set_error(FSB_ERR_INVALID, "nchw_to_nhwc: bad argument");
  return nchw_to_nhwc_launch(N, C, H, W, x, x_is_f32, y, ycs, static_cast<cudaStream_t>(stream));
}
int fsb_nhwc_f16_to_nchw(int N, int C, int H, int W, const void* x, int xcs, void* y, int y_is_f32, void* stream) {
  if (N <= 0 || C <= 0 || !x || !y || xcs < C) return set_error(FSB_ERR_INVALID, "nhwc_to_nchw: bad argument");
  return nhwc_to_nchw_launch(N, C, H, W, x, xcs, y, y_is_f32, static_cast<cudaStream_t>(stream));
}
int fsb_copy_channels(int64_t pixels, int C, const void* x, int xcs, void* y, int ycs, void* stream) {
  if (pixels <= 0 || C <= 0 || !x || !y) return set_error(FSB_ERR_INVALID, "copy_channels: bad argument");
  return copy_channels_launch(pixels, C, x, xcs, y, ycs, static_cast<cudaStream_t>(stream));
}

int fsb_bn_stats(int64_t pixels, int C, const void* x, int xcs, float* stats, void* stream) {
  if (pixels <= 0 || C <= 0 || !x || !stats) return set_error(FSB_ERR_INVALID, "bn_stats: bad argument");
  return bn_stats_launch(pixels, C, x, xcs, 0, stats, static_cast<cudaStream_t>(stream));
}
int fsb_bn_finalize(int C, const float* stats, int rows, int SC, double count, const float* gamma, const float* beta, float eps,
                    float momentum, float* running_mean, float* running_var, float* scale, float* shift, float* save_mean,
                    float* save_invstd, void* stream) {
  if (C <= 0 || !stats || count <= 0 || rows <= 0 || SC < C) return set_error(FSB_ERR_INVALID, "bn_finalize: bad argument");
  return bn_finalize_launch(C, stats, rows, SC, count, gamma, beta, eps, momentum, running_mean, running_var, scale, shift, save_mean,
                            save_invstd, static_cast<cudaStream_t>(stream));
}
int fsb_affine_act(int64_t pixels, int C, const void* x, int xcs, const float* scale, const float* shift, void* y, int ycs,
                   uint32_t flags, void* stream) {
  if (pixels <= 0 || C <= 0 || !x || !y || !scale || !shift) return set_error(FSB_ERR_INVALID, "affine_act: bad argument");
  return affine_act_launch(pixels, C, x, xcs, scale, shift, y, ycs, flags, static_cast<cudaStream_t>(stream));
}


int fsb_bn_bwd_reduce(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                      int raw_is_f32, const float* mean, const float* invstd, int relu, float* sums, void* stream) {
  if (pixels <= 0 || C <= 0 || !dy || !raw || !mean || !invstd || !sums || (relu && !y))
    return set_error(FSB_ERR_INVALID, "bn_bwd_reduce: bad argument");
  return bn_bwd_reduce_launch(pixels, C, dy, dcs, y, ycs, raw, rcs, raw_is_f32, mean, invstd, relu, sums,
                              static_cast<cudaStream_t>(stream));
}
int fsb_bn_bwd_apply(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                     int raw_is_f32, const float* mean, const float* invstd, const float* gamma, const float* sums, double count, int relu,
                     void* draw, int ocs, float* dgamma, float* dbeta, float gscale, int accumulate, void* stream) {
  if (pixels <= 0 || C <= 0 || !dy || !raw || !mean || !invstd || !sums || !draw || count <= 0 || gscale <= 0 || (relu && !y))
    return set_error(FSB_ERR_INVALID, "bn_bwd_apply: bad argument");
  return bn_bwd_apply_launch(pixels, C, dy, dcs, y, ycs, raw, rcs, raw_is_f32, mean, invstd, gamma, sums, count, relu, draw, ocs,
                             dgamma, dbeta, gscale, static_cast<cudaStream_t>(stream), accumulate);
}
/* ---- device-selected BatchNorm sets (captured training graphs) ---- */
int fsb_bn_finalize_sel(int C, const float* stats, int rows, int SC, double count, float eps, float momentum, float* scale,
                        float* shift, float* save_mean, float* save_invstd, const fsb_bn_sel* sel, const int* width_idx, int hmax,
                        void* stream) {
  if (C <= 0 || !stats || count <= 0 || rows <= 0 || SC < C || !sel || !width_idx || hmax < 0 || (hmax > 0 && C != 2 * hmax))
    return set_error(FSB_ERR_INVALID, "bn_finalize_sel: bad argument");
  return bn_finalize_launch(C, stats, rows, SC, count, nullptr, nullptr, eps, momentum, nullptr, nullptr, scale, shift, save_mean,
                            save_invstd, static_cast<cudaStream_t>(stream), nullptr, sel, width_idx, hmax);
}
int fsb_affine_act_sel(int64_t pixels, int C, const void* x, int xcs, const float* scale, const float* shift, void* y, int ycs,
                       uint32_t flags, const fsb_bn_sel* sel, const int* width_idx, int hmax, void* stream) {
  if (pixels <= 0 || C <= 0 || !x || !y || !scale || !shift) return set_error(FSB_ERR_INVALID, "affine_act_sel: bad argument");
  return affine_act_launch(pixels, C, x, xcs, scale, shift, y, ycs, flags, static_cast<cudaStream_t>(stream), sel, width_idx, hmax);
}
int fsb_bn_bwd_reduce_sel(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                          int raw_is_f32, const float* mean, const float* invstd, int relu, float* sums, const fsb_bn_sel* sel,
                          const int* width_idx, int hmax, void* stream) {
  if (pixels <= 0 || C <= 0 || !dy || !raw || !mean || !invstd || !sums || (relu && !y))
    return set_error(FSB_ERR_INVALID, "bn_bwd_reduce_sel: bad argument");
  return bn_bwd_reduce_launch(pixels, C, dy, dcs, y, ycs, raw, rcs, raw_is_f32, mean, invstd, relu, sums,
                              static_cast<cudaStream_t>(stream), sel, width_idx, hmax);
}
int fsb_bn_bwd_apply_sel(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                         int raw_is_f32, const float* mean, const float* invstd, const float* sums, const float* local_sums,
                         double count, int relu, void* draw, int ocs, float gscale, const fsb_bn_sel* sel, const int* width_idx,
                         int hmax, void* stream) {
  if (pixels <= 0 || C <= 0 || !dy || !raw || !mean || !invstd || !sums || !draw || count <= 0 || gscale <= 0 || (relu && !y) || !sel ||
      !width_idx)
    return set_error(FSB_ERR_INVALID, "bn_bwd_apply_sel: bad argument");
  return bn_bwd_apply_launch(pixels, C, dy, dcs, y, ycs, raw, rcs, raw_is_f32, mean, invstd, nullptr, sums, count, relu, draw, ocs,
                             nullptr, nullptr, gscale, static_cast<cudaStream_t>(stream), 1, sel, width_idx, hmax, local_sums);
}

int fsb_relu_bwd(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, void* dx, int xcs, void* stream) {
  if (pixels <= 0 || C <= 0 || !dy || !y || !dx) return set_error(FSB_ERR_INVALID, "relu_bwd: bad argument");
  return relu_bwd_launch(pixels, C, dy, dcs, y, ycs, dx, xcs, static_cast<cudaStream_t>(stream));
}
size_t fsb_conv_packed_dgrad_bytes(const fsb_conv_desc* d) {
  if (!d || d->Cin <= 0 || d->Cout <= 0) return 0;
  const fsb_conv_desc t = dgrad_as_fwd_desc(d, d->Cout, d->Cin);
  const ConvGeom g = conv_geom(&t);
  return static_cast<size_t>(g.taps) * g.npad * g.kpad * 2;
}
int fsb_pack_conv_weight_dgrad(const fsb_conv_desc* d, const float* w, int64_t so, int64_t si, void* packed_t, void* stream) {
  if (!d || !w || !packed_t) return set_error(FSB_ERR_INVALID, "pack_conv_weight_dgrad: null argument");
  return pack_dgrad_launch(d, w, so, si, packed_t, static_cast<cudaStream_t>(stream));
}
int fsb_conv_dgrad(const fsb_conv_desc* d, const void* dy, int dcs, const void* wpacked_t, const float* w, int64_t so, int64_t si,
                   void* dx, int xcs, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  if (!dy || !dx || dcs < d->Cout || xcs < d->Cin) return set_error(FSB_ERR_INVALID, "conv_dgrad: bad argument");
  return conv_dgrad_launch(d, dy, dcs, wpacked_t, w, so, si, dx, xcs, static_cast<cudaStream_t>(stream));
}
int fsb_conv_wgrad(const fsb_conv_desc* d, const void* x, const void* dy, int dcs, float* dw, int64_t so, int64_t si,
                   int accumulate, float gscale, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  if (!x || !dy || !dw || dcs < d->Cout || gscale <= 0) return set_error(FSB_ERR_INVALID, "conv_wgrad: bad argument");
  return conv_wgrad_launch(d, x, dy, dcs, dw, so, si, accumulate, gscale, static_cast<cudaStream_t>(stream));
}
int fsb_bilinear_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy, int dcs, const void* ymask, int ycs, void* dx,
                     int xcs, void* stream) {
  if (N <= 0 || C <= 0 || !dy || !dx) return set_error(FSB_ERR_INVALID, "bilinear_bwd: bad argument");
  return bilinear_bwd_launch(N, C, Hi, Wi, Ho, Wo, dy, dcs, ymask, ycs, dx, xcs, static_cast<cudaStream_t>(stream));
}
int fsb_upsample_logits_bwd(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy, int dy_is_f32, void* dx, int xcs,
                            float gscale, void* stream) {
  if (N <= 0 || C <= 0 || !dy || !dx || xcs < C) return set_error(FSB_ERR_INVALID, "upsample_logits_bwd: bad argument");
  return upsample_logits_bwd_launch(N, C, Hi, Wi, Ho, Wo, dy, dy_is_f32, dx, xcs, gscale, static_cast<cudaStream_t>(stream));
}
int fsb_nchw_grad_to_nhwc(int N, int C, int H, int W, const void* dy, int dy_is_f32, void* dx, int xcs, float gscale, void* stream) {
  if (N <= 0 || C <= 0 || !dy || !dx || xcs < C) return set_error(FSB_ERR_INVALID, "nchw_grad_to_nhwc: bad argument");
  return nchw_grad_to_nhwc_launch(N, C, H, W, dy, dy_is_f32, dx, xcs, gscale, static_cast<cudaStream_t>(stream));
}
int fsb_wsum_fwd(int K, int64_t pixels, int C, const void* const* xs, const int* xcs, const float* wts, void* out, int ocs,
                 void* stream) {
  if (pixels <= 0 || C <= 0 || !xs || !xcs || !wts || !out) return set_error(FSB_ERR_INVALID, "wsum_fwd: bad argument");
  return wsum_fwd_launch(K, pixels, C, xs, xcs, wts, out, ocs, static_cast<cudaStream_t>(stream));
}
int fsb_wsum_bwd(int K, int64_t pixels, int C, const void* dout, int docs, const void* const* xs, const int* xcs, const float* wts,
                 void* const* dxs, const int* dxcs, float* dwts, float gscale, void* stream) {
  if (pixels <= 0 || C <= 0 || !dout || !wts || gscale <= 0) return set_error(FSB_ERR_INVALID, "wsum_bwd: bad argument");
  return wsum_bwd_launch(K, pixels, C, dout, docs, xs, xcs, wts, dxs, dxcs, dwts, gscale, static_cast<cudaStream_t>(stream));
}
int fsb_add_inplace(int64_t pixels, int C, const void* x, int xcs, void* y, int ycs, void* stream) {
  if (pixels <= 0 || C <= 0 || !x || !y) return set_error(FSB_ERR_INVALID, "add_inplace: bad argument");
  return add_inplace_launch(pixels, C, x, xcs, y, ycs, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
