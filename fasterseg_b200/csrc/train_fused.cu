// train_fused.cu -- native orchestration of one training "unit" (conv -> BatchNorm(train) -> activation) so that the host
// pays for ONE C-ABI call per unit and direction instead of a dozen Python-level calls.  The supernet step launches
// ~3 400 such units per forward pass set (search/model_search.py:487-500) and is host-bound otherwise.
#include "fsb_internal.h"

namespace fsb {

int bn_finalize_launch(int, const float*, int, int, double, const float*, const float*, float, float, float*, float*, float*, float*,
                       float*, float*, cudaStream_t, long long*, const fsb_bn_sel*, const int*, int);
int affine_act_launch(int64_t, int, const void*, int, const float*, const float*, void*, int, uint32_t, cudaStream_t,
                      const fsb_bn_sel*, const int*, int);
int bn_bwd_reduce_launch(int64_t, int, const void*, int, const void*, int, const void*, int, int, const float*, const float*, int,
                         float*, cudaStream_t, const fsb_bn_sel*, const int*, int);
int bn_bwd_apply_launch(int64_t, int, const void*, int, const void*, int, const void*, int, int, const float*, const float*,
                        const float*, const float*, double, int, void*, int, float*, float*, float, cudaStream_t, int,
                        const fsb_bn_sel*, const int*, int, const float*);
int rowsum_launch(int, const float*, int, int, float*, cudaStream_t);
int conv_dgrad_launch(const fsb_conv_desc*, const void*, int, const void*, const float*, int64_t, int64_t, void*, int, cudaStream_t);
int conv_wgrad_launch(const fsb_conv_desc*, const void*, const void*, int, float*, int64_t, int64_t, int, float, cudaStream_t);
int dp_world();                                        // dp.cu: 1 unless fsb_dp_init created a communicator
int dp_allreduce_f32(float*, int64_t, cudaStream_t);   // in-place sum over ranks on the stream

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
// what the vectorised BatchNorm kernels of the unit need: whole 8-channel vectors, 16-byte aligned pixels.  Checked before the
// first launch so that a rejected call has changed nothing (the forward updates the running statistics half way through).
static inline bool vec_view_ok(int C, int cstride, const void* p) { return C % 8 == 0 && cstride % 8 == 0 && aligned16(p); }

// dgamma = sum(dz * xhat) / gscale, dbeta = sum(dz) / gscale from the rank-LOCAL sums (the data-parallel gradient average
// divides by the world size afterwards, so these must not come from the all-reduced buffer)
__global__ void local_param_grads_kernel(int C, const float* __restrict__ sums, float inv_gscale, float* __restrict__ dgamma,
                                         float* __restrict__ dbeta, const fsb_bn_sel* sel, const int* width_idx) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (sel) {  // device-selected parameter set: accumulate into its gradient slots
    const fsb_bn_sel s = sel[*width_idx];
    if (c < s.C) {
      if (s.dbeta) s.dbeta[c] += sums[c] * inv_gscale;
      if (s.dgamma) s.dgamma[c] += sums[C + c] * inv_gscale;
    }
    return;
  }
  if (c < C) {
    dbeta[c] = sums[c] * inv_gscale;
    dgamma[c] = sums[C + c] * inv_gscale;
  }
}

}  // namespace fsb

using namespace fsb;

extern "C" {

/* vec: fp32[(6 + 2R)*Cout] = [sum | sumsq | scale | shift | mean | invstd | R partial rows]; mean/invstd are what backward needs. */
int fsb_conv_bn_act_train_fwd(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* gamma, const float* beta,
                              float eps, float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                              void* raw_f32, int raw_cstride, void* y, int y_cstride, float* vec, int relu,
                              const fsb_bn_sel* sel, const int* width_idx, void* stream) {
  if (!d || !x || !wpacked || !raw_f32 || !y || !vec) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_fwd: null argument");
  if ((sel == nullptr) != (width_idx == nullptr)) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_fwd: sel and width_idx go together");
  const int C = d->Cout;
  if (!vec_view_ok(C, raw_cstride, raw_f32) || !vec_view_ok(C, y_cstride, y) || !aligned16(vec))
    return set_error(FSB_ERR_INVALID, "conv_bn_act_train_fwd: Cout and strides multiples of 8, raw / y / vec 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  fsb_conv_desc c = *d;
  c.y_cstride = raw_cstride;
  c.flags = (d->flags & FSB_CONV_FORCE_DIRECT) | FSB_CONV_OUT_F32 | FSB_CONV_STATS;
  c.stats_C = 0;
  c.stats_off = 0;
  float* rows = vec + 6 * C;
  const ConvPlan plan = conv_plan(&c);
  const int64_t pixels = static_cast<int64_t>(d->N) * d->Ho * d->Wo;
  int R = plan.stat_rows;
  int rc = plan.direct ? conv_direct_launch(&c, x, wpacked, nullptr, nullptr, raw_f32, rows, st)
                       : conv_tc_launch(plan, &c, x, wpacked, nullptr, nullptr, raw_f32, rows, st);
  if (rc) return rc;
  const int world = dp_world();
  const float* stats = rows;
  if (world > 1) {  // SyncBN: the statistics of all ranks, exchanged on the stream between the two kernels
    rc = rowsum_launch(2 * C, rows, R, 2 * C, vec, st);
    if (rc) return rc;
    rc = dp_allreduce_f32(vec, 2 * C, st);
    if (rc) return rc;
    stats = vec;
    R = 1;
  }
  rc = bn_finalize_launch(C, stats, R, C, static_cast<double>(pixels) * world, gamma, beta, eps, momentum, running_mean, running_var,
                          vec + 2 * C, vec + 3 * C, vec + 4 * C, vec + 5 * C, st, num_batches_tracked, sel, width_idx, 0);
  if (rc) return rc;
  return affine_act_launch(pixels, C, raw_f32, raw_cstride, vec + 2 * C, vec + 3 * C, y, y_cstride,
                           (relu ? FSB_CONV_RELU : 0u) | FSB_ACT_IN_F32, st, nullptr, nullptr, 0);
}

/* Backward of the unit.  vec_fwd: the forward's vec (mean at 4C, invstd at 5C).  vec_bwd: fp32[(4 + 2Rb)*Cout] = [sum dz |
 * sum dz*xhat | Rb partial rows | dgamma | dbeta].  draw: scratch NHWC fp16 (Cout channels).  dx / dw may be NULL; dw is
 * ACCUMULATED into. */
int fsb_conv_bn_act_train_bwd(const fsb_conv_desc* d, const void* x, const void* dy, int dy_cstride, const void* y, int y_cstride,
                              const void* raw_f32, int raw_cstride, const float* vec_fwd, const float* gamma, int relu,
                              const void* wpacked_t, const float* w, int64_t so, int64_t si, void* draw, int draw_cstride,
                              float* vec_bwd, void* dx, int dx_cstride, float* dw, float gscale, const fsb_bn_sel* sel,
                              const int* width_idx, void* stream) {
  if (!d || !dy || !raw_f32 || !vec_fwd || !vec_bwd || !draw) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_bwd: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int C = d->Cout;
  const int64_t pixels = static_cast<int64_t>(d->N) * d->Ho * d->Wo;
  cudaError_t e;
  if ((sel == nullptr) != (width_idx == nullptr)) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_bwd: sel and width_idx go together");
  if (!vec_view_ok(C, dy_cstride, dy) || !vec_view_ok(C, raw_cstride, raw_f32) || !vec_view_ok(C, draw_cstride, draw) ||
      (relu && (!y || !vec_view_ok(C, y_cstride, y))) || C > 2048)
    return set_error(FSB_ERR_INVALID, "conv_bn_act_train_bwd: Cout <= 2048 and strides multiples of 8, dy / y / raw / draw 16-byte aligned");
  if (dw && !x) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_bwd: wgrad needs x");
  // the dgrad's direct fallback reads the fp32 master weight; which path runs is decided inside conv_dgrad_launch
  if (dx && (!w || dx_cstride < d->Cin)) return set_error(FSB_ERR_INVALID, "conv_bn_act_train_bwd: dx needs w and dx_cstride >= Cin");
  const int Rb = stat_rows(pixels);
  float* dgamma = vec_bwd + static_cast<size_t>(2 + 2 * Rb) * C;  // [totals (2C) | Rb partial rows | dgamma | dbeta]
  float* dbeta = dgamma + C;
  int rc = bn_bwd_reduce_launch(pixels, C, dy, dy_cstride, y, y_cstride, raw_f32, raw_cstride, 1, vec_fwd + 4 * C, vec_fwd + 5 * C, relu,
                                vec_bwd, st, nullptr, nullptr, 0);
  if (rc) return rc;
  const int world = dp_world();
  if (world > 1) {
    // SyncBN backward: gamma / beta gradients from the LOCAL sums, dx from the GLOBAL sums and the global pixel count
    local_param_grads_kernel<<<(C + 127) / 128, 128, 0, st>>>(C, vec_bwd, 1.0f / gscale, dgamma, dbeta, sel, width_idx);
    e = cudaGetLastError();
    if (e != cudaSuccess) return set_cuda_error(e, "conv_bn_act_train_bwd: local_param_grads launch");
    rc = dp_allreduce_f32(vec_bwd, 2 * C, st);
    if (rc) return rc;
    rc = bn_bwd_apply_launch(pixels, C, dy, dy_cstride, y, y_cstride, raw_f32, raw_cstride, 1, vec_fwd + 4 * C, vec_fwd + 5 * C, gamma, vec_bwd,
                             static_cast<double>(pixels) * world, relu, draw, draw_cstride, nullptr, nullptr, gscale, st, -1, sel, width_idx, 0,
                             nullptr);
  } else {
    rc = bn_bwd_apply_launch(pixels, C, dy, dy_cstride, y, y_cstride, raw_f32, raw_cstride, 1, vec_fwd + 4 * C, vec_fwd + 5 * C, gamma, vec_bwd,
                             static_cast<double>(pixels), relu, draw, draw_cstride, dgamma, dbeta, gscale, st, sel ? 1 : 0, sel, width_idx, 0, nullptr);
  }
  if (rc) return rc;
  if (dx) {
    rc = conv_dgrad_launch(d, draw, draw_cstride, wpacked_t, w, so, si, dx, dx_cstride, st);
    if (rc) return rc;
  }
  if (dw) {
    rc = conv_wgrad_launch(d, x, draw, draw_cstride, dw, so, si, 1, gscale, st);
    if (rc) return rc;
  }
  return FSB_OK;
}

}  // extern "C"
