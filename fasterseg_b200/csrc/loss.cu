// loss.cu -- N1 (SURVEY 8f): the training criteria of the reference drivers evaluated straight from the LOW-RESOLUTION logits.
//
// Reference path (train/model_seg.py:357-362 + tools/seg_opr/loss_opr.py:63-93 + train/train.py:254-260): every head's logits
// are bilinearly upsampled (align_corners=True, x8 / x16 / x32) to the label resolution as fp32 NCHW tensors (478 MB each at
// 12 x 19 x 512 x 1024), then softmax / log_softmax / gather / argsort / KLDivLoss run over those tensors, and autograd walks the
// same tensors backwards.  Here nothing of label resolution with a class axis ever exists:
//   logp_fwd   : one thread per label pixel interpolates its 19 logits from the 4 low-resolution neighbours (NHWC fp16, L1/L2
//                resident), keeps the log-sum-exp and the log-probability of the true class       -> 8 B per pixel instead of 76+
//   kth_select : exact k-th smallest of the true-class log-probabilities (the OHEM threshold the reference reads off a full
//                argsort) by three histogram passes over the monotone integer image of the floats -> no sort, no host sync
//   ohem_reduce: sum(-logp * kept), count(kept) with kept = valid & (logp <= threshold), fixed-order two-stage reduction
//   ce_bwd     : gather form of (upsample o softmax-CE)^T: one thread per LOW-RESOLUTION pixel walks the label pixels whose
//                bilinear footprint contains it, re-derives softmax from the stored log-sum-exp and accumulates
//                weight * kept * (p - onehot)                                                       -> fp16 NHWC gradient, no atomics
//   kl_fwd/bwd : the same two steps for KLDivLoss(log_softmax(student), softmax(teacher)) with both logit maps low-resolution.
// Arithmetic is fp32 throughout; gradients leave in the fp16 NHWC gradient domain of train.cu (x gscale).
#include <algorithm>

#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

namespace {

__device__ __forceinline__ void lz_src(int dst, float scale, int n_in, int& i0, int& i1, float& l1) {
  const float src = scale * static_cast<float>(dst);   // ATen's align_corners=True rule (area_pixel_compute_source_index)
  i0 = static_cast<int>(src);
  if (i0 > n_in - 1) i0 = n_in - 1;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
}
__host__ __device__ inline float lz_scale(int n_in, int n_out) {
  return n_out > 1 ? static_cast<float>(n_in - 1) / static_cast<float>(n_out - 1) : 0.f;
}
__device__ __forceinline__ float lz_tapw(int o, int i, float scale, int n_in) {
  int i0, i1;
  float l1;
  lz_src(o, scale, n_in, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}
__device__ __forceinline__ void lz_range(int i, float scale, int n_out, int& lo, int& hi) {
  if (scale <= 0.f) {
    lo = 0;
    hi = n_out - 1;
    return;
  }
  lo = static_cast<int>(floorf((static_cast<float>(i) - 1.f) / scale)) - 1;
  hi = static_cast<int>(ceilf((static_cast<float>(i) + 1.f) / scale)) + 1;
  if (lo < 0) lo = 0;
  if (hi > n_out - 1) hi = n_out - 1;
}

// the CP (= classes rounded up to 8) logits of one label pixel, interpolated from the low-resolution NHWC fp16 map
template <int CP>
__device__ __forceinline__ void lz_logits(const __half* __restrict__ x, int xcs, int n, int Hi, int Wi, int ho, int wo, float sh, float sw,
                                          float (&l)[CP]) {
  int h0, h1, w0, w1;
  float lh, lw;
  lz_src(ho, sh, Hi, h0, h1, lh);
  lz_src(wo, sw, Wi, w0, w1, lw);
  const __half* base = x + static_cast<size_t>(n) * Hi * Wi * xcs;
  const __half* p00 = base + (static_cast<size_t>(h0) * Wi + w0) * xcs;
  const __half* p01 = base + (static_cast<size_t>(h0) * Wi + w1) * xcs;
  const __half* p10 = base + (static_cast<size_t>(h1) * Wi + w0) * xcs;
  const __half* p11 = base + (static_cast<size_t>(h1) * Wi + w1) * xcs;
  const float w00 = (1.f - lh) * (1.f - lw), w01 = (1.f - lh) * lw, w10 = lh * (1.f - lw), w11 = lh * lw;
#pragma unroll
  for (int v = 0; v < CP / 8; ++v) {
    const uint4 a = *reinterpret_cast<const uint4*>(p00 + v * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(p01 + v * 8);
    const uint4 c = *reinterpret_cast<const uint4*>(p10 + v * 8);
    const uint4 d = *reinterpret_cast<const uint4*>(p11 + v * 8);
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
    const __half2* hc = reinterpret_cast<const __half2*>(&c);
    const __half2* hd = reinterpret_cast<const __half2*>(&d);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]), fc = __half22float2(hc[j]), fd = __half22float2(hd[j]);
      // same operation order as ATen's upsample_bilinear2d: w00*a + w01*b + w10*c + w11*d grouped by rows
      l[v * 8 + 2 * j] = (1.f - lh) * ((1.f - lw) * fa.x + lw * fb.x) + lh * ((1.f - lw) * fc.x + lw * fd.x);
      l[v * 8 + 2 * j + 1] = (1.f - lh) * ((1.f - lw) * fa.y + lw * fb.y) + lh * ((1.f - lw) * fc.y + lw * fd.y);
    }
  }
  (void)w00; (void)w01; (void)w10; (void)w11;
}

template <int CP>
__device__ __forceinline__ float lz_lse(const float (&l)[CP], int C) {
  float m = -INFINITY;
#pragma unroll
  for (int c = 0; c < CP; ++c)
    if (c < C) m = fmaxf(m, l[c]);
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < CP; ++c)
    if (c < C) s += expf(l[c] - m);
  return m + logf(s);
}

// ---- forward: true-class log-probability and log-sum-exp per label pixel ----------------------------------------------------
template <int CP>
__global__ void __launch_bounds__(256)
loss_logp_fwd_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs, const long long* __restrict__ target,
                     int ignore_label, float* __restrict__ logp_t, float* __restrict__ lse_out, float sh, float sw) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wo = static_cast<int>(gid % Wo);
  const int ho = static_cast<int>((gid / Wo) % Ho);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(Wo) * Ho));
  float l[CP];
  lz_logits<CP>(x, xcs, n, Hi, Wi, ho, wo, sh, sw, l);
  const float lse = lz_lse<CP>(l, C);
  const long long t = target[gid];
  const bool valid = t != ignore_label && t >= 0 && t < C;
  float lt = 0.f;
#pragma unroll
  for (int c = 0; c < CP; ++c)
    if (c == static_cast<int>(t)) lt = l[c];
  logp_t[gid] = valid ? lt - lse : 0.f;   // ignored pixels carry probability 1 (loss_opr.py:73 masked_fill_(~valid_mask, 1))
  lse_out[gid] = lse;
}

// ---- exact k-th smallest by radix histograms -----------------------------------------------------------------------------------
// state[0] = key prefix found so far, state[1] = remaining rank (1-based) inside the current prefix class
__device__ __forceinline__ uint32_t lz_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // monotone: a < b  <=>  key(a) < key(b)
}
__device__ __forceinline__ float lz_unkey(uint32_t k) {
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  return __uint_as_float(u);
}
// pass 0: bits [31:20] (4096 bins), pass 1: bits [19:8] among keys whose bits [31:20] match, pass 2: bits [7:0]
__global__ void __launch_bounds__(256)
kth_hist_kernel(const float* __restrict__ x, int64_t n, int pass, const unsigned long long* __restrict__ state, unsigned int* __restrict__ hist) {
  __shared__ unsigned int sh[4096];
  const int bins = pass == 2 ? 256 : 4096;
  for (int i = threadIdx.x; i < bins; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  const uint32_t prefix = pass == 0 ? 0u : static_cast<uint32_t>(state[0]);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const uint32_t k = lz_key(x[i]);
    if (pass == 0) {
      atomicAdd(&sh[k >> 20], 1u);
    } else if (pass == 1) {
      if ((k >> 20) == (prefix >> 20)) atomicAdd(&sh[(k >> 8) & 0xFFFu], 1u);
    } else {
      if ((k >> 8) == (prefix >> 8)) atomicAdd(&sh[k & 0xFFu], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < bins; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);   // integer atomics: the histogram does not depend on arrival order
}
// one block of 256 threads: thread t sums bins [16 t, 16 t + 16) (pass 2: one bin), thread 0 walks the 256 group sums and then the
// 16 bins of the group that contains the rank
__global__ void __launch_bounds__(256)
kth_scan_kernel(const unsigned int* __restrict__ hist, int pass, int64_t k_in, unsigned long long* __restrict__ state, float* __restrict__ out) {
  __shared__ unsigned int grp[256];
  const int per = pass == 2 ? 1 : 16;
  unsigned int g = 0;
  for (int i = 0; i < per; ++i) g += hist[threadIdx.x * per + i];
  grp[threadIdx.x] = g;
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned long long rank = pass == 0 ? static_cast<unsigned long long>(k_in) : state[1];
  uint32_t prefix = pass == 0 ? 0u : static_cast<uint32_t>(state[0]);
  unsigned long long acc = 0;
  int gi = 0;
  for (; gi < 255; ++gi) {
    if (acc + grp[gi] >= rank) break;
    acc += grp[gi];
  }
  int b = gi * per;
  for (; b < gi * per + per - 1; ++b) {
    if (acc + hist[b] >= rank) break;
    acc += hist[b];
  }
  rank -= acc;
  if (pass == 0) prefix = static_cast<uint32_t>(b) << 20;
  else if (pass == 1) prefix |= static_cast<uint32_t>(b) << 8;
  else prefix |= static_cast<uint32_t>(b);
  state[0] = prefix;
  state[1] = rank;
  if (pass == 2) *out = lz_unkey(prefix);
}

// ---- OHEM reduction -----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ohem_partial_kernel(const float* __restrict__ logp_t, const long long* __restrict__ target, int64_t n, int ignore_label, int C,
                    const float* __restrict__ thr, float* __restrict__ partial) {
  pdl_launch_dependents();
  pdl_wait();
  const float th = thr ? *thr : INFINITY;
  float s = 0.f, cnt = 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const long long t = target[i];
    const bool valid = t != ignore_label && t >= 0 && t < C;
    const float lp = logp_t[i];
    if (valid && lp <= th) {
      s -= lp;
      cnt += 1.f;
    }
  }
  __shared__ float ss[8], sc[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0) {
    ss[threadIdx.x >> 5] = s;
    sc[threadIdx.x >> 5] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < 8; ++w) {
      a += ss[w];
      b += sc[w];
    }
    partial[2 * blockIdx.x] = a;
    partial[2 * blockIdx.x + 1] = b;
  }
}
__global__ void pair_rowsum_kernel(const float* __restrict__ partial, int rows, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0, b = 0.0;
  for (int r = 0; r < rows; ++r) {   // fixed order: bit-reproducible
    a += partial[2 * r];
    b += partial[2 * r + 1];
  }
  out[0] = static_cast<float>(a);
  out[1] = static_cast<float>(b);
}

// ---- cross-entropy backward, gather form ------------------------------------------------------------------------------------------
template <int CP>
__global__ void __launch_bounds__(128)
loss_ce_bwd_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs, const long long* __restrict__ target,
                   int ignore_label, const float* __restrict__ lse, const float* __restrict__ logp_t, const float* __restrict__ thr,
                   const float* __restrict__ coef, __half* __restrict__ dx, int dcs, float gscale, float sh, float sw, int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wi = static_cast<int>(gid % Wi);
  const int hi = static_cast<int>((gid / Wi) % Hi);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(Wi) * Hi));
  const float th = thr ? *thr : INFINITY;
  int hlo, hhi, wlo, whi;
  lz_range(hi, sh, Ho, hlo, hhi);
  lz_range(wi, sw, Wo, wlo, whi);
  float acc[CP];
#pragma unroll
  for (int c = 0; c < CP; ++c) acc[c] = 0.f;
  for (int ho = hlo; ho <= hhi; ++ho) {
    const float wh = lz_tapw(ho, hi, sh, Hi);
    if (wh == 0.f) continue;
    for (int wo = wlo; wo <= whi; ++wo) {
      const float ww = lz_tapw(wo, wi, sw, Wi);
      if (ww == 0.f) continue;
      const size_t op = (static_cast<size_t>(n) * Ho + ho) * Wo + wo;
      const long long t = target[op];
      const bool valid = t != ignore_label && t >= 0 && t < C;
      if (!valid || !(logp_t[op] <= th)) continue;   // not among the kept pixels: no gradient
      float l[CP];
      lz_logits<CP>(x, xcs, n, Hi, Wi, ho, wo, sh, sw, l);
      const float ls = lse[op];
      const float wgt = wh * ww;
#pragma unroll
      for (int c = 0; c < CP; ++c) {
        if (c < C) {
          const float p = expf(l[c] - ls);
          acc[c] = fmaf(wgt, p - (c == static_cast<int>(t) ? 1.f : 0.f), acc[c]);
        }
      }
    }
  }
  const float k = (*coef) * gscale;
  __half* out = dx + static_cast<size_t>(gid) * dcs;
#pragma unroll
  for (int v = 0; v < CP / 8; ++v) {
    float prev[8];
    if (accumulate) {
      const uint4 pv = *reinterpret_cast<const uint4*>(out + v * 8);
      const __half2* hp = reinterpret_cast<const __half2*>(&pv);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(hp[j]);
        prev[2 * j] = f.x;
        prev[2 * j + 1] = f.y;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) prev[j] = 0.f;
    }
    uint4 o;
    o.x = pack_half2(fmaf(acc[v * 8 + 0], k, prev[0]), fmaf(acc[v * 8 + 1], k, prev[1]));
    o.y = pack_half2(fmaf(acc[v * 8 + 2], k, prev[2]), fmaf(acc[v * 8 + 3], k, prev[3]));
    o.z = pack_half2(fmaf(acc[v * 8 + 4], k, prev[4]), fmaf(acc[v * 8 + 5], k, prev[5]));
    o.w = pack_half2(fmaf(acc[v * 8 + 6], k, prev[6]), fmaf(acc[v * 8 + 7], k, prev[7]));
    *reinterpret_cast<uint4*>(out + v * 8) = o;
  }
}

// ---- KL distillation --------------------------------------------------------------------------------------------------------------
template <int CP>
__global__ void __launch_bounds__(256)
loss_kl_fwd_kernel(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const __half* __restrict__ xs, int scs,
                   const __half* __restrict__ xt, int tcs, float* __restrict__ lse_s, float* __restrict__ lse_t, float* __restrict__ partial,
                   float shs, float sws, float sht, float swt) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo;
  float s = 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; gid < total; gid += stride) {
    const int wo = static_cast<int>(gid % Wo);
    const int ho = static_cast<int>((gid / Wo) % Ho);
    const int n = static_cast<int>(gid / (static_cast<int64_t>(Wo) * Ho));
    float ls[CP], lt[CP];
    lz_logits<CP>(xs, scs, n, Hs, Ws, ho, wo, shs, sws, ls);
    lz_logits<CP>(xt, tcs, n, Ht, Wt, ho, wo, sht, swt, lt);
    const float es = lz_lse<CP>(ls, C), et = lz_lse<CP>(lt, C);
    float kl = 0.f;
#pragma unroll
    for (int c = 0; c < CP; ++c)
      if (c < C) {
        const float logq = lt[c] - et;
        kl = fmaf(expf(logq), logq - (ls[c] - es), kl);   // q * (log q - log p): KLDivLoss pointwise term (xlogy form)
      }
    s += kl;
    lse_s[gid] = es;
    lse_t[gid] = et;
  }
  __shared__ float ss[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) ss[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    for (int w = 0; w < 8; ++w) a += ss[w];
    partial[2 * blockIdx.x] = a;
    partial[2 * blockIdx.x + 1] = 0.f;
  }
}

template <int CP>
__global__ void __launch_bounds__(128)
loss_kl_bwd_kernel(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const __half* __restrict__ xs, int scs,
                   const __half* __restrict__ xt, int tcs, const float* __restrict__ lse_s, const float* __restrict__ lse_t,
                   const float* __restrict__ coef, __half* __restrict__ dx, int dcs, float gscale, float shs, float sws, float sht, float swt,
                   int accumulate) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(N) * Hs * Ws;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wi = static_cast<int>(gid % Ws);
  const int hi = static_cast<int>((gid / Ws) % Hs);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(Ws) * Hs));
  int hlo, hhi, wlo, whi;
  lz_range(hi, shs, Ho, hlo, hhi);
  lz_range(wi, sws, Wo, wlo, whi);
  float acc[CP];
#pragma unroll
  for (int c = 0; c < CP; ++c) acc[c] = 0.f;
  for (int ho = hlo; ho <= hhi; ++ho) {
    const float wh = lz_tapw(ho, hi, shs, Hs);
    if (wh == 0.f) continue;
    for (int wo = wlo; wo <= whi; ++wo) {
      const float ww = lz_tapw(wo, wi, sws, Ws);
      if (ww == 0.f) continue;
      const size_t op = (static_cast<size_t>(n) * Ho + ho) * Wo + wo;
      float ls[CP], lt[CP];
      lz_logits<CP>(xs, scs, n, Hs, Ws, ho, wo, shs, sws, ls);
      lz_logits<CP>(xt, tcs, n, Ht, Wt, ho, wo, sht, swt, lt);
      const float es = lse_s[op], et = lse_t[op];
      const float wgt = wh * ww;
#pragma unroll
      for (int c = 0; c < CP; ++c)
        if (c < C) acc[c] = fmaf(wgt, expf(ls[c] - es) - expf(lt[c] - et), acc[c]);   // d/dl_s of sum_c q_c (log q_c - log p_c) = p - q
    }
  }
  const float k = (*coef) * gscale;
  __half* out = dx + static_cast<size_t>(gid) * dcs;
#pragma unroll
  for (int v = 0; v < CP / 8; ++v) {
    float prev[8];
    if (accumulate) {
      const uint4 pv = *reinterpret_cast<const uint4*>(out + v * 8);
      const __half2* hp = reinterpret_cast<const __half2*>(&pv);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(hp[j]);
        prev[2 * j] = f.x;
        prev[2 * j + 1] = f.y;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) prev[j] = 0.f;
    }
    uint4 o;
    o.x = pack_half2(fmaf(acc[v * 8 + 0], k, prev[0]), fmaf(acc[v * 8 + 1], k, prev[1]));
    o.y = pack_half2(fmaf(acc[v * 8 + 2], k, prev[2]), fmaf(acc[v * 8 + 3], k, prev[3]));
    o.z = pack_half2(fmaf(acc[v * 8 + 4], k, prev[4]), fmaf(acc[v * 8 + 5], k, prev[5]));
    o.w = pack_half2(fmaf(acc[v * 8 + 6], k, prev[6]), fmaf(acc[v * 8 + 7], k, prev[7]));
    *reinterpret_cast<uint4*>(out + v * 8) = o;
  }
}

int loss_check(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs) {
  if (N <= 0 || C <= 0 || C > 32 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || !x) return set_error(FSB_ERR_INVALID, "loss: bad shape");
  const int cp = (C + 7) / 8 * 8;
  if (xcs < cp || (xcs % 8) != 0 || (reinterpret_cast<uintptr_t>(x) & 15))
    return set_error(FSB_ERR_INVALID, "loss: logits need a channel stride >= round8(C), multiple of 8, 16-byte aligned");
  return FSB_OK;
}

constexpr int kLossRows = 1056;   // 8 x 132 partial rows

}  // namespace

#define LZ_DISPATCH(C, CALL)              \
  switch (((C) + 7) / 8) {                \
    case 1: { constexpr int CP = 8; CALL; } break;  \
    case 2: { constexpr int CP = 16; CALL; } break; \
    case 3: { constexpr int CP = 24; CALL; } break; \
    default: { constexpr int CP = 32; CALL; } break; \
  }

int loss_logp_fwd_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const long long* target, int ignore_label,
                         float* logp_t, float* lse, cudaStream_t stream) {
  if (int rc = loss_check(N, C, Hi, Wi, Ho, Wo, x, xcs)) return rc;
  if (!target || !logp_t || !lse) return set_error(FSB_ERR_INVALID, "loss_logp_fwd: null pointer");
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  LZ_DISPATCH(C, FSB_LAUNCH(loss_logp_fwd_kernel<CP>, dim3(blocks), dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs,
                            target, ignore_label, logp_t, lse, lz_scale(Hi, Ho), lz_scale(Wi, Wo)));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "loss_logp_fwd launch");
  return FSB_OK;
}

size_t kth_workspace_bytes() { return (4096 + 4096 + 256) * sizeof(unsigned int) + 2 * sizeof(unsigned long long) + 16; }

int kth_smallest_launch(const float* x, int64_t n, int64_t k, float* out, void* workspace, cudaStream_t stream) {
  if (!x || !out || !workspace || n <= 0 || k < 1 || k > n) return set_error(FSB_ERR_INVALID, "kth_smallest: need 1 <= k <= n");
  unsigned int* hist = static_cast<unsigned int*>(workspace);
  unsigned long long* state = reinterpret_cast<unsigned long long*>(hist + 4096 + 4096 + 256 + 2);   // 8-byte aligned: 8450 words in
  if (cudaMemsetAsync(workspace, 0, kth_workspace_bytes(), stream) != cudaSuccess) return set_error(FSB_ERR_CUDA, "kth_smallest: memset");
  const int sms = sm_count();
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((n + 255) / 256, static_cast<int64_t>(sms) * 8));
  unsigned int* h[3] = {hist, hist + 4096, hist + 8192};
  for (int pass = 0; pass < 3; ++pass) {
    kth_hist_kernel<<<blocks, 256, 0, stream>>>(x, n, pass, state, h[pass]);
    kth_scan_kernel<<<1, 256, 0, stream>>>(h[pass], pass, k, state, out);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, "kth_smallest launch");
  return FSB_OK;
}

int ohem_reduce_launch(const float* logp_t, const long long* target, int64_t n, int ignore_label, int C, const float* thr, float* partial,
                       float* out2, cudaStream_t stream) {
  if (!logp_t || !target || !partial || !out2 || n <= 0) return set_error(FSB_ERR_INVALID, "ohem_reduce: bad argument");
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((n + 255) / 256, kLossRows));
  FSB_LAUNCH(ohem_partial_kernel, dim3(blocks), dim3(256), 0, stream, logp_t, target, n, ignore_label, C, thr, partial);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "ohem_reduce launch");
  pair_rowsum_kernel<<<1, 32, 0, stream>>>(partial, static_cast<int>(blocks), out2);
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, "ohem_reduce final launch");
  return FSB_OK;
}

int loss_rows() { return kLossRows; }

int loss_ce_bwd_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const long long* target, int ignore_label,
                       const float* lse, const float* logp_t, const float* thr, const float* coef, void* dx, int dcs, float gscale, int accumulate,
                       cudaStream_t stream) {
  if (int rc = loss_check(N, C, Hi, Wi, Ho, Wo, x, xcs)) return rc;
  if (int rc = loss_check(N, C, Hi, Wi, Ho, Wo, dx, dcs)) return rc;
  if (!target || !lse || !logp_t || !coef) return set_error(FSB_ERR_INVALID, "loss_ce_bwd: null pointer");
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi;
  const unsigned blocks = static_cast<unsigned>((total + 127) / 128);
  LZ_DISPATCH(C, FSB_LAUNCH(loss_ce_bwd_kernel<CP>, dim3(blocks), dim3(128), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs,
                            target, ignore_label, lse, logp_t, thr, coef, static_cast<__half*>(dx), dcs, gscale, lz_scale(Hi, Ho),
                            lz_scale(Wi, Wo), accumulate));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "loss_ce_bwd launch");
  return FSB_OK;
}

int loss_kl_fwd_launch(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* xs, int scs, const void* xt, int tcs,
                       float* lse_s, float* lse_t, float* partial, float* out2, cudaStream_t stream) {
  if (int rc = loss_check(N, C, Hs, Ws, Ho, Wo, xs, scs)) return rc;
  if (int rc = loss_check(N, C, Ht, Wt, Ho, Wo, xt, tcs)) return rc;
  if (!lse_s || !lse_t || !partial || !out2) return set_error(FSB_ERR_INVALID, "loss_kl_fwd: null pointer");
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, kLossRows));
  LZ_DISPATCH(C, FSB_LAUNCH(loss_kl_fwd_kernel<CP>, dim3(blocks), dim3(256), 0, stream, N, C, Hs, Ws, Ht, Wt, Ho, Wo,
                            static_cast<const __half*>(xs), scs, static_cast<const __half*>(xt), tcs, lse_s, lse_t, partial, lz_scale(Hs, Ho),
                            lz_scale(Ws, Wo), lz_scale(Ht, Ho), lz_scale(Wt, Wo)));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "loss_kl_fwd launch");
  pair_rowsum_kernel<<<1, 32, 0, stream>>>(partial, static_cast<int>(blocks), out2);
  e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, "loss_kl_fwd final launch");
  return FSB_OK;
}

int loss_kl_bwd_launch(int N, int C, int Hs, int Ws, int Ht, int Wt, int Ho, int Wo, const void* xs, int scs, const void* xt, int tcs,
                       const float* lse_s, const float* lse_t, const float* coef, void* dx, int dcs, float gscale, int accumulate,
                       cudaStream_t stream) {
  if (int rc = loss_check(N, C, Hs, Ws, Ho, Wo, xs, scs)) return rc;
  if (int rc = loss_check(N, C, Ht, Wt, Ho, Wo, xt, tcs)) return rc;
  if (int rc = loss_check(N, C, Hs, Ws, Ho, Wo, dx, dcs)) return rc;
  if (!lse_s || !lse_t || !coef) return set_error(FSB_ERR_INVALID, "loss_kl_bwd: null pointer");
  const int64_t total = static_cast<int64_t>(N) * Hs * Ws;
  const unsigned blocks = static_cast<unsigned>((total + 127) / 128);
  LZ_DISPATCH(C, FSB_LAUNCH(loss_kl_bwd_kernel<CP>, dim3(blocks), dim3(128), 0, stream, N, C, Hs, Ws, Ht, Wt, Ho, Wo,
                            static_cast<const __half*>(xs), scs, static_cast<const __half*>(xt), tcs, lse_s, lse_t, coef, static_cast<__half*>(dx), dcs,
                            gscale, lz_scale(Hs, Ho), lz_scale(Ws, Wo), lz_scale(Ht, Ho), lz_scale(Wt, Wo), accumulate));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "loss_kl_bwd launch");
  return FSB_OK;
}

}  // namespace fsb
