// train.cu -- backward / training kernels: BatchNorm(+ReLU) backward (K8), conv dgrad / wgrad (K7), bilinear and logits
// upsample backward (K4/K9 transposes), weighted multi-tensor sum (K5).  These replace what autograd derives for the
// reference's F.conv2d / nn.BatchNorm2d / nn.ReLU / F.interpolate / `result + op(x) * w` call sites
// (search/operations.py, search/model_search.py:75-78,326-333).  Activation gradients are fp16 NHWC carrying a static
// loss scale `gscale`; everything written in fp32 (parameter and scalar gradients) is divided by it.
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

__device__ __forceinline__ void src_index_t(int dst, float scale, int n_in, int& i0, int& i1, float& l1) {
  const float src = scale * static_cast<float>(dst);
  i0 = static_cast<int>(src);
  if (i0 > n_in - 1) i0 = n_in - 1;
  i1 = i0 + (i0 < n_in - 1 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
}
__host__ __device__ inline float ac_scale_t(int n_in, int n_out) {
  return n_out > 1 ? static_cast<float>(n_in - 1) / static_cast<float>(n_out - 1) : 0.f;
}
// weight with which output index `o` reads input index `i` along one axis (0 if it does not)
__device__ __forceinline__ float tap_weight(int o, int i, float scale, int n_in) {
  int i0, i1;
  float l1;
  src_index_t(o, scale, n_in, i0, i1, l1);
  return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}
// candidate output range [lo, hi] that may read input index i
__device__ __forceinline__ void cand_range(int i, float scale, int n_out, int& lo, int& hi) {
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

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __half22float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
template <typename T>
__device__ __forceinline__ void load8t(const T* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load8t<__half>(const __half* p, float (&f)[8]) { unpack8(*reinterpret_cast<const uint4*>(p), f); }
template <>
__device__ __forceinline__ void load8t<float>(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_half2(f[0], f[1]);
  o.y = pack_half2(f[2], f[3]);
  o.z = pack_half2(f[4], f[5]);
  o.w = pack_half2(f[6], f[7]);
  return o;
}

// ------------------------------------------------------------------------------------------
// BatchNorm (+ReLU) backward
// ------------------------------------------------------------------------------------------
// compact -> raw channel bijection of a FactorizedReduce running at maximum width (see bn.cu split_remap)
__device__ __forceinline__ int split_remap_t(int c, int h, int hmax) {
  if (hmax <= 0) return c;
  if (c < h) return c;
  if (c < 2 * h) return hmax + (c - h);
  const int k = c - 2 * h;
  return k < hmax - h ? h + k : hmax + h + (k - (hmax - h));
}
template <typename TR>
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(int64_t pixels, int C, const __half* __restrict__ dy, int dcs, const __half* __restrict__ y, int ycs,
                     const TR* __restrict__ raw, int rcs, const float* __restrict__ mean, const float* __restrict__ invstd,
                     int relu, float* __restrict__ rows_out, const fsb_bn_sel* sel, const int* width_idx, int hmax) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float red[];
  const int cvec = C >> 3;
  const int rows = blockDim.x / cvec;
  const int cv = threadIdx.x % cvec;
  const int row = threadIdx.x / cvec;
  const int rcv = split_remap_t(cv, (sel && hmax > 0) ? sel[*width_idx].C / 16 : 0, hmax >> 3);  // raw is in raw channel order
  float s[8], q[8], mu[8], is[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = 0.f;
    mu[j] = mean[cv * 8 + j];
    is[j] = invstd[cv * 8 + j];
  }
  if (row < rows) {
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * rows + row; p < pixels; p += static_cast<int64_t>(gridDim.x) * rows) {
      float d[8], r[8], yy[8];
      unpack8(*reinterpret_cast<const uint4*>(dy + p * dcs + cv * 8), d);
      load8t<TR>(raw + p * rcs + rcv * 8, r);
      if (relu) unpack8(*reinterpret_cast<const uint4*>(y + p * ycs + cv * 8), yy);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dz = (relu && !(yy[j] > 0.f)) ? 0.f : d[j];
        s[j] += dz;
        q[j] += dz * (r[j] - mu[j]) * is[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      red[(row * C + cv * 8 + j) * 2 + 0] = s[j];
      red[(row * C + cv * 8 + j) * 2 + 1] = q[j];
    }
  }
  __syncthreads();
  // this block's partial row (fixed intra-block order; the rows are added in index order by rowsum_kernel)
  float* out = rows_out + static_cast<size_t>(blockIdx.x) * 2 * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < rows; ++r) {
      a += red[(r * C + c) * 2 + 0];
      b += red[(r * C + c) * 2 + 1];
    }
    out[c] = a;
    out[C + c] = b;
  }
}

template <typename TR>
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(int64_t pixels, int C, const __half* __restrict__ dy, int dcs, const __half* __restrict__ y, int ycs,
                    const TR* __restrict__ raw, int rcs, const float* __restrict__ mean, const float* __restrict__ invstd,
                    const float* __restrict__ gamma, const float* __restrict__ sums, float inv_count, int relu,
                    __half* __restrict__ draw, int ocs, float* __restrict__ dgamma, float* __restrict__ dbeta, float inv_gscale,
                    int accumulate, const fsb_bn_sel* sel, const int* width_idx, int hmax, const float* __restrict__ psums) {
  pdl_launch_dependents();
  pdl_wait();
  const int cvec = C >> 3;
  int active = C;
  if (sel) {  // parameter set chosen on the device (see bn_finalize_kernel); channels >= its width have invstd = 0 -> draw = 0
    const fsb_bn_sel sl = sel[*width_idx];
    gamma = sl.gamma;
    dgamma = sl.dgamma;
    dbeta = sl.dbeta;
    active = sl.C;
  }
  // gamma / beta gradients: accumulate = 1 add, 0 assign, -1 none.  psums: the rank-LOCAL sums under data parallelism (the
  // gradient average over ranks divides by the world size afterwards), `sums` then being the all-reduced ones.
  if (blockIdx.x == 0 && accumulate >= 0) {
    const float* ps = psums ? psums : sums;
    for (int c = threadIdx.x; c < active; c += blockDim.x) {
      if (dbeta) dbeta[c] = (accumulate ? dbeta[c] : 0.f) + ps[c] * inv_gscale;
      if (dgamma) dgamma[c] = (accumulate ? dgamma[c] : 0.f) + ps[C + c] * inv_gscale;
    }
  }
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t p = i / cvec;
    const int rcv = split_remap_t(cv, hmax > 0 ? active >> 4 : 0, hmax >> 3);  // raw and draw are in raw channel order
    float d[8], r[8], yy[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(dy + p * dcs + cv * 8), d);
    load8t<TR>(raw + p * rcs + rcv * 8, r);
    if (relu) unpack8(*reinterpret_cast<const uint4*>(y + p * ycs + cv * 8), yy);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = cv * 8 + j;
      const float dz = (relu && !(yy[j] > 0.f)) ? 0.f : d[j];
      const float xh = (r[j] - mean[c]) * invstd[c];
      const float g = (gamma && c < active) ? gamma[c] : (c < active ? 1.f : 0.f);
      o[j] = g * invstd[c] * (dz - sums[c] * inv_count - xh * sums[C + c] * inv_count);
    }
    *reinterpret_cast<uint4*>(draw + p * ocs + rcv * 8) = pack8(o);
  }
}

__global__ void __launch_bounds__(256)
relu_bwd_kernel(int64_t pixels, int cvec, const __half* __restrict__ dy, int dcs, const __half* __restrict__ y, int ycs,
                __half* __restrict__ dx, int xcs) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t p = i / cvec;
    float d[8], yy[8];
    unpack8(*reinterpret_cast<const uint4*>(dy + p * dcs + cv * 8), d);
    unpack8(*reinterpret_cast<const uint4*>(y + p * ycs + cv * 8), yy);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = yy[j] > 0.f ? d[j] : 0.f;
    *reinterpret_cast<uint4*>(dx + p * xcs + cv * 8) = pack8(d);
  }
}

static inline bool vec_ok(int C, int cs, const void* p) { return C % 8 == 0 && cs % 8 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
static inline unsigned grid_for(int64_t total, int threads) {
  int64_t b = (total + threads - 1) / threads;
  if (b < 1) b = 1;
  if (b > 132 * 16) b = 132 * 16;
  return static_cast<unsigned>(b);
}

int rowsum_launch(int L, const float* rows, int P, int stride, float* out, cudaStream_t stream);

// sums: (1 + stat_rows(pixels)) rows of 2*C floats; the partial rows land in rows 1.., their fixed-order total in row 0
int bn_bwd_reduce_launch(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                         int raw_f32, const float* mean, const float* invstd, int relu, float* sums, cudaStream_t stream,
                         const fsb_bn_sel* sel, const int* width_idx, int hmax) {
  if (hmax > 0 && (!sel || !width_idx || hmax % 8 || C != 2 * hmax)) return set_error(FSB_ERR_INVALID, "bn_bwd_reduce: bad split arguments");
  if (!vec_ok(C, dcs, dy) || !vec_ok(C, rcs, raw) || (relu && !vec_ok(C, ycs, y)) || C > 2048)
    return set_error(FSB_ERR_INVALID, "bn_bwd_reduce: C/strides multiples of 8, pointers 16B aligned");
  const int cvec = C / 8, threads = 256;
  const int rows = threads / cvec;
  if (rows < 1) return set_error(FSB_ERR_INVALID, "bn_bwd_reduce: C too large");
  const int blocks = stat_rows(pixels);
  float* part = sums + 2 * C;
  const size_t smem = static_cast<size_t>(rows) * C * 2 * sizeof(float);
  if (raw_f32)
    FSB_LAUNCH(bn_bwd_reduce_kernel<float>, dim3(static_cast<unsigned>(blocks)), dim3(threads), smem, stream, pixels, C,
               static_cast<const __half*>(dy), dcs, static_cast<const __half*>(y), ycs, static_cast<const float*>(raw), rcs, mean,
               invstd, relu, part, sel, width_idx, hmax);
  else
    FSB_LAUNCH(bn_bwd_reduce_kernel<__half>, dim3(static_cast<unsigned>(blocks)), dim3(threads), smem, stream, pixels, C,
               static_cast<const __half*>(dy), dcs, static_cast<const __half*>(y), ycs, static_cast<const __half*>(raw), rcs, mean,
               invstd, relu, part, sel, width_idx, hmax);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bn_bwd_reduce launch");
  return rowsum_launch(2 * C, part, blocks, 2 * C, sums, stream);
}
int bn_bwd_apply_launch(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, const void* raw, int rcs,
                        int raw_f32, const float* mean, const float* invstd, const float* gamma, const float* sums, double count, int relu,
                        void* draw, int ocs, float* dgamma, float* dbeta, float gscale, cudaStream_t stream, int accumulate,
                        const fsb_bn_sel* sel, const int* width_idx, int hmax, const float* psums) {
  if (hmax > 0 && (!sel || !width_idx || hmax % 8 || C != 2 * hmax)) return set_error(FSB_ERR_INVALID, "bn_bwd_apply: bad split arguments");
  if (!vec_ok(C, dcs, dy) || !vec_ok(C, rcs, raw) || !vec_ok(C, ocs, draw) || (relu && !vec_ok(C, ycs, y)))
    return set_error(FSB_ERR_INVALID, "bn_bwd_apply: C/strides multiples of 8, pointers 16B aligned");
  if (raw_f32)
    FSB_LAUNCH(bn_bwd_apply_kernel<float>, dim3(grid_for(pixels * (C / 8), 256)), dim3(256), 0, stream, pixels, C,
               static_cast<const __half*>(dy), dcs, static_cast<const __half*>(y), ycs, static_cast<const float*>(raw), rcs, mean,
               invstd, gamma, sums, static_cast<float>(1.0 / count), relu, static_cast<__half*>(draw), ocs, dgamma, dbeta,
               1.0f / gscale, accumulate, sel, width_idx, hmax, psums);
  else
    FSB_LAUNCH(bn_bwd_apply_kernel<__half>, dim3(grid_for(pixels * (C / 8), 256)), dim3(256), 0, stream, pixels, C,
               static_cast<const __half*>(dy), dcs, static_cast<const __half*>(y), ycs, static_cast<const __half*>(raw), rcs, mean,
               invstd, gamma, sums, static_cast<float>(1.0 / count), relu, static_cast<__half*>(draw), ocs, dgamma, dbeta,
               1.0f / gscale, accumulate, sel, width_idx, hmax, psums);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bn_bwd_apply launch");
  return FSB_OK;
}
int relu_bwd_launch(int64_t pixels, int C, const void* dy, int dcs, const void* y, int ycs, void* dx, int xcs, cudaStream_t stream) {
  if (!vec_ok(C, dcs, dy) || !vec_ok(C, ycs, y) || !vec_ok(C, xcs, dx))
    return set_error(FSB_ERR_INVALID, "relu_bwd: C/strides multiples of 8, pointers 16B aligned");
  FSB_LAUNCH(relu_bwd_kernel, dim3(grid_for(pixels * (C / 8), 256)), dim3(256), 0, stream, pixels, C / 8,
             static_cast<const __half*>(dy), dcs, static_cast<const __half*>(y), ycs, static_cast<__half*>(dx), xcs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "relu_bwd launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// conv dgrad
// ------------------------------------------------------------------------------------------
// weights for the tensor-core path: the data gradient of a stride-1 conv is itself a stride-1 conv of dy with the
// spatially flipped, channel-transposed filter: packed_t[tap'][n = ci][k = co] = w[co][ci][K-1-r'][K-1-s']
__global__ void pack_dgrad_kernel(const float* __restrict__ w, int64_t so, int64_t si, int ks, int Cout, int Cin, int npad,
                                  int kpad, __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int taps = ks * ks;
  const int64_t total = static_cast<int64_t>(taps) * npad * kpad;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % kpad);          // co
    const int n = static_cast<int>((i / kpad) % npad);  // ci
    const int tap = static_cast<int>(i / (static_cast<int64_t>(kpad) * npad));
    const int r = ks - 1 - tap / ks, s = ks - 1 - tap % ks;
    float v = 0.f;
    if (n < Cin && k < Cout) v = w[k * so + n * si + r * ks + s];
    out[i] = __float2half_rn(v);
  }
}

fsb_conv_desc dgrad_as_fwd_desc(const fsb_conv_desc* d, int dy_cstride, int dx_cstride) {
  fsb_conv_desc t;
  memset(&t, 0, sizeof(t));
  t.N = d->N;
  t.H = d->Ho;
  t.W = d->Wo;
  t.Cin = d->Cout;
  t.Cout = d->Cin;
  t.ksize = d->ksize;
  t.stride = 1;
  t.pad = d->dil * (d->ksize - 1) - d->pad;
  t.dil = d->dil;
  t.Ho = d->H;
  t.Wo = d->W;
  t.x_cstride = dy_cstride;
  t.y_cstride = dx_cstride;
  t.flags = 0;
  return t;
}

int pack_dgrad_launch(const fsb_conv_desc* d, const float* w, int64_t so, int64_t si, void* packed, cudaStream_t stream) {
  const fsb_conv_desc t = dgrad_as_fwd_desc(d, d->Cout, d->Cin);
  const ConvGeom g = conv_geom(&t);
  const int64_t total = static_cast<int64_t>(g.taps) * g.npad * g.kpad;
  FSB_LAUNCH(pack_dgrad_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, w, so, si, d->ksize, d->Cout, d->Cin, g.npad,
             g.kpad, static_cast<__half*>(packed));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "pack_dgrad launch");
  return FSB_OK;
}

// generic gather-form dgrad on CUDA cores: one thread = one input pixel x 8 input channels
struct DgradParams {
  fsb_conv_desc d;
  const __half* dy;
  int dcs;
  const float* w;
  int64_t so, si;
  __half* dx;
  int xcs;
};
__global__ void __launch_bounds__(128) conv_dgrad_direct_kernel(const DgradParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const fsb_conv_desc& d = p.d;
  const int cgroups = (d.Cin + 7) / 8;
  const int64_t npix = static_cast<int64_t>(d.N) * d.H * d.W;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= npix * cgroups) return;
  const int cg = static_cast<int>(gid % cgroups);
  const int64_t pix = gid / cgroups;
  const int wi = static_cast<int>(pix % d.W);
  const int hi = static_cast<int>((pix / d.W) % d.H);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(d.W) * d.H));
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int r = 0; r < d.ksize; ++r) {
    const int th = hi - d.off_h + d.pad - r * d.dil;
    if (th < 0 || th % d.stride) continue;
    const int ho = th / d.stride;
    if (ho >= d.Ho) continue;
    for (int s = 0; s < d.ksize; ++s) {
      const int tw = wi - d.off_w + d.pad - s * d.dil;
      if (tw < 0 || tw % d.stride) continue;
      const int wo = tw / d.stride;
      if (wo >= d.Wo) continue;
      const __half* dyp = p.dy + (static_cast<size_t>(n) * d.Ho * d.Wo + static_cast<size_t>(ho) * d.Wo + wo) * p.dcs;
      for (int co = 0; co < d.Cout; ++co) {
        const float g = __half2float(dyp[co]);
        const float* wp = p.w + co * p.so + r * d.ksize + s;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int ci = cg * 8 + j;
          if (ci < d.Cin) acc[j] = fmaf(g, wp[ci * p.si], acc[j]);
        }
      }
    }
  }
  __half* xp = p.dx + static_cast<size_t>(pix) * p.xcs + cg * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (cg * 8 + j < d.Cin) xp[j] = __float2half_rn(acc[j]);
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int conv_dgrad_launch(const fsb_conv_desc* d, const void* dy, int dcs, const void* wpacked_t, const float* w, int64_t so,
                      int64_t si, void* dx, int xcs, cudaStream_t stream) {
  // the tensor-core paths read dy and the packed weight through TMA (16-byte aligned bases); anything else takes the direct kernel
  const bool tc_ok = wpacked_t && aligned16(wpacked_t) && aligned16(dy) && !(d->flags & FSB_CONV_FORCE_DIRECT);
  if (d->stride == 1 && d->off_h == 0 && d->off_w == 0 && tc_ok) {
    fsb_conv_desc t = dgrad_as_fwd_desc(d, dcs, xcs);
    if (conv_tc_supported(&t)) return conv_tc_launch(conv_plan(&t, nullptr, false), &t, dy, wpacked_t, nullptr, nullptr, dx, nullptr, stream);
  }
  // stride 2: the input pixels of each (row, column) parity receive contributions from a fixed subset of filter taps; each
  // parity plane is a stride-1 implicit GEMM over dy with that tap subset, written to the plane through a strided tensor map
  if (d->stride == 2 && tc_ok && d->Cin % 8 == 0 && xcs % 8 == 0 && dcs % 8 == 0 && d->Cout >= 16 && aligned16(dx) &&
      opt(OPT_DGRAD_S2_DIRECT) <= 0) {
    fsb_conv_desc t = dgrad_as_fwd_desc(d, dcs, xcs);  // stride-1 problem over dy; geometry fields only feed the packer
    t.pad = 0;
    t.Ho = d->Ho;
    t.Wo = d->Wo;
    const int K = d->ksize;
    bool need_zero = false;
    ConvTcCustom planes[4];
    bool live[4];
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw) {
        ConvTcCustom& c = planes[ph * 2 + pw];
        memset(&c, 0, sizeof(c));
        const int Hl = (d->H - ph + 1) / 2, Wl = (d->W - pw + 1) / 2;
        for (int r = 0; r < K; ++r) {
          const int th = ph - d->off_h + d->pad - r * d->dil;
          if (th & 1) continue;
          for (int s = 0; s < K; ++s) {
            const int tw = pw - d->off_w + d->pad - s * d->dil;
            if (tw & 1) continue;
            c.dh[c.ntaps] = th / 2;  // exact: th is even (may be negative)
            c.dw[c.ntaps] = tw / 2;
            c.widx[c.ntaps] = (K - 1 - r) * K + (K - 1 - s);  // pack_dgrad_kernel stores the flipped filter
            ++c.ntaps;
          }
        }
        live[ph * 2 + pw] = c.ntaps > 0 && Hl > 0 && Wl > 0;
        if (c.ntaps == 0 && Hl > 0 && Wl > 0) need_zero = true;
        c.Ho = Hl;
        c.Wo = Wl;
        c.y_base = static_cast<const __half*>(dx) + (static_cast<size_t>(ph) * d->W + pw) * xcs;
        c.y_dims[0] = d->Cin;
        c.y_dims[1] = Wl;
        c.y_dims[2] = Hl;
        c.y_dims[3] = d->N;
        c.y_strides[0] = 2ull * xcs * 2;
        c.y_strides[1] = 2ull * d->W * xcs * 2;
        c.y_strides[2] = static_cast<uint64_t>(d->H) * d->W * xcs * 2;
      }
    if (conv_tc_supported(&t)) {
      ConvPlan plans[4];
      for (int i = 0; i < 4; ++i) {  // descriptor errors before the first write
        if (!live[i]) continue;
        plans[i] = conv_plan(&t, &planes[i]);
        if (plans[i].rc) return plans[i].rc;
      }
      // a parity plane without taps (1x1 stride 2) gets no MMA: zero the Cin channels of every pixel, not the whole pixel
      // stride, which belongs to the caller when dx is a channel slice
      if (need_zero) {
        cudaError_t e = cudaMemset2DAsync(dx, static_cast<size_t>(xcs) * 2, 0, static_cast<size_t>(d->Cin) * 2,
                                          static_cast<size_t>(d->N) * d->H * d->W, stream);
        if (e != cudaSuccess) return set_cuda_error(e, "conv_dgrad: memset");
      }
      for (int i = 0; i < 4; ++i) {
        if (!live[i]) continue;
        int rc = conv_tc_launch(plans[i], &t, dy, wpacked_t, nullptr, nullptr, dx, nullptr, stream, &planes[i]);
        if (rc) return rc;
      }
      return FSB_OK;
    }
  }
  if (!w) return set_error(FSB_ERR_INVALID, "conv_dgrad: the direct path needs the fp32 master weight");
  DgradParams p;
  p.d = *d;
  p.dy = static_cast<const __half*>(dy);
  p.dcs = dcs;
  p.w = w;
  p.so = so;
  p.si = si;
  p.dx = static_cast<__half*>(dx);
  p.xcs = xcs;
  const int64_t total = static_cast<int64_t>(d->N) * d->H * d->W * ((d->Cin + 7) / 8);
  FSB_LAUNCH(conv_dgrad_direct_kernel, dim3(static_cast<unsigned>((total + 127) / 128)), dim3(128), 0, stream, p);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "conv_dgrad_direct launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// conv wgrad: per tap a [Cout x Cin] GEMM over K = pixels.  CUDA-core tiled GEMM, split over pixel chunks with
// fp32 atomic accumulation: block = 64 co x 64 ci x one tap x one pixel chunk; 256 threads, 4x4 outputs each.
// ------------------------------------------------------------------------------------------
constexpr int kWgTile = 64;
constexpr int kWgK = 16;
struct WgradParams {
  fsb_conv_desc d;
  const __half* x;
  const __half* dy;
  int dcs;
  float* dw;
  int64_t so, si;
  float inv_gscale;
  int64_t chunk;  // pixels per block along K
};
__global__ void __launch_bounds__(256) conv_wgrad_kernel(const WgradParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const fsb_conv_desc& d = p.d;
  __shared__ float s_dy[kWgK][kWgTile + 1];
  __shared__ float s_x[kWgK][kWgTile + 1];
  const int co_tiles = (d.Cout + kWgTile - 1) / kWgTile;
  const int ci_tiles = (d.Cin + kWgTile - 1) / kWgTile;
  int b = blockIdx.x;
  const int co0 = (b % co_tiles) * kWgTile;
  b /= co_tiles;
  const int ci0 = (b % ci_tiles) * kWgTile;
  b /= ci_tiles;
  const int tap = b;
  const int r = tap / d.ksize, s = tap % d.ksize;
  const int64_t npix = static_cast<int64_t>(d.N) * d.Ho * d.Wo;
  const int64_t p0 = static_cast<int64_t>(blockIdx.y) * p.chunk;
  const int64_t p1 = min(npix, p0 + p.chunk);
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;  // ty -> co sub-tile, tx -> ci sub-tile
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int64_t pb = p0; pb < p1; pb += kWgK) {
    // cooperative load: 16 pixels x 64 channels of dy and of the tap-shifted x (zero outside the image)
    for (int i = threadIdx.x; i < kWgK * kWgTile; i += blockDim.x) {
      const int kk = i / kWgTile, c = i % kWgTile;
      const int64_t pp = pb + kk;
      float vdy = 0.f, vx = 0.f;
      if (pp < p1) {
        const int wo = static_cast<int>(pp % d.Wo);
        const int ho = static_cast<int>((pp / d.Wo) % d.Ho);
        const int n = static_cast<int>(pp / (static_cast<int64_t>(d.Wo) * d.Ho));
        if (co0 + c < d.Cout) vdy = __half2float(p.dy[pp * p.dcs + co0 + c]);
        const int hi = ho * d.stride + r * d.dil - d.pad + d.off_h;
        const int wi = wo * d.stride + s * d.dil - d.pad + d.off_w;
        if (ci0 + c < d.Cin && hi >= 0 && hi < d.H && wi >= 0 && wi < d.W)
          vx = __half2float(p.x[(static_cast<size_t>(n) * d.H * d.W + static_cast<size_t>(hi) * d.W + wi) * d.x_cstride + ci0 + c]);
      }
      s_dy[kk][c] = vdy;
      s_x[kk][c] = vx;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kWgK; ++kk) {
      float a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = s_dy[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bb[j] = s_x[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = co0 + ty * 4 + i;
    if (co >= d.Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = ci0 + tx * 4 + j;
      if (ci >= d.Cin) continue;
      atomicAdd(&p.dw[co * p.so + ci * p.si + tap], acc[i][j] * p.inv_gscale);
    }
  }
}
__global__ void zero_wgrad_kernel(float* dw, int64_t so, int64_t si, int Cout, int Cin, int taps) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(Cout) * Cin * taps;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i % taps);
    const int ci = static_cast<int>((i / taps) % Cin);
    const int co = static_cast<int>(i / (static_cast<int64_t>(taps) * Cin));
    dw[co * so + ci * si + t] = 0.f;
  }
}
// zeroes the [0,Cout) x [0,Cin) corner of the gradient before an accumulate = 0 weight gradient
int zero_wgrad_launch(const fsb_conv_desc* d, float* dw, int64_t so, int64_t si, cudaStream_t stream) {
  const int taps = d->ksize * d->ksize;
  const int64_t total = static_cast<int64_t>(d->Cout) * d->Cin * taps;
  FSB_LAUNCH(zero_wgrad_kernel, dim3(grid_for(total, 256)), dim3(256), 0, stream, dw, so, si, d->Cout, d->Cin, taps);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "zero_wgrad launch");
  return FSB_OK;
}
int conv_wgrad_launch(const fsb_conv_desc* d, const void* x, const void* dy, int dcs, float* dw, int64_t so, int64_t si,
                      int accumulate, float gscale, cudaStream_t stream) {
  const int taps = d->ksize * d->ksize;
  // the tensor-core kernel reads x and dy through TMA (16-byte aligned bases); the direct kernel has no alignment needs.  The
  // tensor-core launch zeroes dw itself, once its tensor maps are encoded, so that a call it rejects writes nothing.
  if (conv_wgrad_tc_supported(d, dcs) && aligned16(x) && aligned16(dy) && !(d->flags & FSB_CONV_FORCE_DIRECT))
    return conv_wgrad_tc_launch(d, x, dy, dcs, dw, so, si, accumulate, gscale, stream);
  if (!accumulate)
    if (int rc = zero_wgrad_launch(d, dw, so, si, stream)) return rc;
  WgradParams p;
  p.d = *d;
  p.x = static_cast<const __half*>(x);
  p.dy = static_cast<const __half*>(dy);
  p.dcs = dcs;
  p.dw = dw;
  p.so = so;
  p.si = si;
  p.inv_gscale = 1.0f / gscale;
  const int64_t npix = static_cast<int64_t>(d->N) * d->Ho * d->Wo;
  const int tiles = ((d->Cout + kWgTile - 1) / kWgTile) * ((d->Cin + kWgTile - 1) / kWgTile) * taps;
  // enough pixel chunks to fill the machine a few times over, each at least 256 pixels
  int64_t chunks = (132 * 4 + tiles - 1) / tiles;
  const int64_t max_chunks = (npix + 255) / 256;
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1 || opt(OPT_DETERMINISTIC) == 1) chunks = 1;  // deterministic mode: one owner per output element, no split-K atomics
  p.chunk = ((npix + chunks - 1) / chunks + kWgK - 1) / kWgK * kWgK;
  chunks = (npix + p.chunk - 1) / p.chunk;
  FSB_LAUNCH(conv_wgrad_kernel, dim3(static_cast<unsigned>(tiles), static_cast<unsigned>(chunks)), dim3(256), 0, stream, p);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "conv_wgrad launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// bilinear backward (gather form: one thread = one INPUT pixel x 8 channels)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bilinear_bwd_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ dy, int dcs,
                    const __half* __restrict__ ymask, int ycs, __half* __restrict__ dx, int xcs, float sh, float sw) {
  pdl_launch_dependents();
  pdl_wait();
  const int cvec = C >> 3;
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi * cvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int cv = static_cast<int>(gid % cvec);
  const int64_t pix = gid / cvec;
  const int wi = static_cast<int>(pix % Wi);
  const int hi = static_cast<int>((pix / Wi) % Hi);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wi) * Hi));
  int hlo, hhi, wlo, whi;
  cand_range(hi, sh, Ho, hlo, hhi);
  cand_range(wi, sw, Wo, wlo, whi);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int ho = hlo; ho <= hhi; ++ho) {
    const float wh = tap_weight(ho, hi, sh, Hi);
    if (wh == 0.f) continue;
    for (int wo = wlo; wo <= whi; ++wo) {
      const float ww = tap_weight(wo, wi, sw, Wi);
      if (ww == 0.f) continue;
      const size_t op = (static_cast<size_t>(n) * Ho + ho) * Wo + wo;
      float d[8];
      unpack8(*reinterpret_cast<const uint4*>(dy + op * dcs + cv * 8), d);
      if (ymask) {
        float yy[8];
        unpack8(*reinterpret_cast<const uint4*>(ymask + op * ycs + cv * 8), yy);
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = yy[j] > 0.f ? d[j] : 0.f;
      }
      const float wgt = wh * ww;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(wgt, d[j], acc[j]);
    }
  }
  *reinterpret_cast<uint4*>(dx + static_cast<size_t>(pix) * xcs + cv * 8) = pack8(acc);
}
int bilinear_bwd_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy, int dcs, const void* ymask, int ycs, void* dx,
                        int xcs, cudaStream_t stream) {
  if (!vec_ok(C, dcs, dy) || !vec_ok(C, xcs, dx) || (ymask && !vec_ok(C, ycs, ymask)))
    return set_error(FSB_ERR_INVALID, "bilinear_bwd: C/strides multiples of 8, pointers 16B aligned");
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi * (C / 8);
  FSB_LAUNCH(bilinear_bwd_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo,
             static_cast<const __half*>(dy), dcs, static_cast<const __half*>(ymask), ycs, static_cast<__half*>(dx), xcs,
             ac_scale_t(Hi, Ho), ac_scale_t(Wi, Wo));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bilinear_bwd launch");
  return FSB_OK;
}

// logits upsample backward: NCHW gradient (Ho x Wo) -> NHWC fp16 (Hi x Wi); one thread = one (n, hi, wi, c)
template <typename TIn>
__global__ void __launch_bounds__(256)
upsample_logits_bwd_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const TIn* __restrict__ dy, __half* __restrict__ dx,
                           int xcs, float sh, float sw, float gscale) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(N) * C * Hi * Wi;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wi = static_cast<int>(gid % Wi);
  const int hi = static_cast<int>((gid / Wi) % Hi);
  const int c = static_cast<int>((gid / (static_cast<int64_t>(Wi) * Hi)) % C);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(Wi) * Hi * C));
  int hlo, hhi, wlo, whi;
  cand_range(hi, sh, Ho, hlo, hhi);
  cand_range(wi, sw, Wo, wlo, whi);
  const TIn* plane = dy + (static_cast<size_t>(n) * C + c) * Ho * Wo;
  float acc = 0.f;
  for (int ho = hlo; ho <= hhi; ++ho) {
    const float wh = tap_weight(ho, hi, sh, Hi);
    if (wh == 0.f) continue;
    float row = 0.f;
    for (int wo = wlo; wo <= whi; ++wo) {
      const float ww = tap_weight(wo, wi, sw, Wi);
      if (ww != 0.f) row = fmaf(ww, static_cast<float>(plane[static_cast<size_t>(ho) * Wo + wo]), row);
    }
    acc = fmaf(wh, row, acc);
  }
  dx[((static_cast<size_t>(n) * Hi + hi) * Wi + wi) * xcs + c] = __float2half_rn(acc * gscale);
}
int upsample_logits_bwd_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* dy, int dy_is_f32, void* dx, int xcs,
                               float gscale, cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(N) * C * Hi * Wi;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
  if (dy_is_f32)
    FSB_LAUNCH(upsample_logits_bwd_kernel<float>, dim3(blocks), dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo,
               static_cast<const float*>(dy), static_cast<__half*>(dx), xcs, ac_scale_t(Hi, Ho), ac_scale_t(Wi, Wo), gscale);
  else
    FSB_LAUNCH(upsample_logits_bwd_kernel<__half>, dim3(blocks), dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo,
               static_cast<const __half*>(dy), static_cast<__half*>(dx), xcs, ac_scale_t(Hi, Ho), ac_scale_t(Wi, Wo), gscale);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_logits_bwd launch");
  return FSB_OK;
}

template <typename TIn>
__global__ void nchw_grad_to_nhwc_kernel(int N, int C, int H, int W, const TIn* __restrict__ x, __half* __restrict__ y, int ycs,
                                         float gscale) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const int64_t HW = static_cast<int64_t>(H) * W;
  const int n = blockIdx.z;
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const int64_t pp = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && pp < HW) ? static_cast<float>(x[(static_cast<int64_t>(n) * C + c) * HW + pp]) * gscale : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t pp = p0 + i;
    const int c = c0 + threadIdx.x;
    if (pp < HW && c < C) y[(static_cast<int64_t>(n) * HW + pp) * ycs + c] = __float2half_rn(tile[threadIdx.x][i]);
  }
}
int nchw_grad_to_nhwc_launch(int N, int C, int H, int W, const void* dy, int dy_is_f32, void* dx, int xcs, float gscale,
                             cudaStream_t stream) {
  const int64_t HW = static_cast<int64_t>(H) * W;
  dim3 block(32, 8), grid(static_cast<unsigned>((HW + 31) / 32), (C + 31) / 32, N);
  if (dy_is_f32)
    FSB_LAUNCH(nchw_grad_to_nhwc_kernel<float>, grid, block, 0, stream, N, C, H, W, static_cast<const float*>(dy),
               static_cast<__half*>(dx), xcs, gscale);
  else
    FSB_LAUNCH(nchw_grad_to_nhwc_kernel<__half>, grid, block, 0, stream, N, C, H, W, static_cast<const __half*>(dy),
               static_cast<__half*>(dx), xcs, gscale);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "nchw_grad_to_nhwc launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// K5: weighted multi-tensor sum
// ------------------------------------------------------------------------------------------
constexpr int kMaxWsum = 8;
struct WsumArgs {
  const __half* x[kMaxWsum];
  __half* dx[kMaxWsum];
  int xcs[kMaxWsum];
  int dxcs[kMaxWsum];
  int K;
};
__global__ void __launch_bounds__(256)
wsum_fwd_kernel(const WsumArgs a, int64_t pixels, int cvec, const float* __restrict__ wts, __half* __restrict__ out, int ocs) {
  pdl_launch_dependents();
  pdl_wait();
  float w[kMaxWsum];
#pragma unroll
  for (int k = 0; k < kMaxWsum; ++k) w[k] = k < a.K ? wts[k] : 0.f;
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t p = i / cvec;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxWsum; ++k) {
      if (k < a.K) {
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(a.x[k] + p * a.xcs[k] + cv * 8), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(w[k], v[j], acc[j]);
      }
    }
    *reinterpret_cast<uint4*>(out + p * ocs + cv * 8) = pack8(acc);
  }
}
__global__ void __launch_bounds__(256)
wsum_bwd_kernel(const WsumArgs a, int64_t pixels, int cvec, const __half* __restrict__ dout, int docs, const float* __restrict__ wts,
                float* __restrict__ dwts, float inv_gscale) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[kMaxWsum][8];
  float w[kMaxWsum], dot[kMaxWsum];
#pragma unroll
  for (int k = 0; k < kMaxWsum; ++k) {
    w[k] = k < a.K ? wts[k] : 0.f;
    dot[k] = 0.f;
  }
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t p = i / cvec;
    float g[8];
    unpack8(*reinterpret_cast<const uint4*>(dout + p * docs + cv * 8), g);
#pragma unroll
    for (int k = 0; k < kMaxWsum; ++k) {
      if (k < a.K) {
        if (dwts) {
          float v[8];
          unpack8(*reinterpret_cast<const uint4*>(a.x[k] + p * a.xcs[k] + cv * 8), v);
#pragma unroll
          for (int j = 0; j < 8; ++j) dot[k] = fmaf(g[j], v[j], dot[k]);
        }
        if (a.dx[k]) {
          float o[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = w[k] * g[j];
          *reinterpret_cast<uint4*>(a.dx[k] + p * a.dxcs[k] + cv * 8) = pack8(o);
        }
      }
    }
  }
  if (!dwts) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kMaxWsum; ++k) {
    float v = dot[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[k][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < kMaxWsum) {  // partial row of this block (rows 1..; row 0 = fixed-order total, written by rowsum_kernel)
    float v = 0.f;
    if (threadIdx.x < a.K)
      for (int wv = 0; wv < (blockDim.x >> 5); ++wv) v += red[threadIdx.x][wv];
    dwts[(static_cast<size_t>(blockIdx.x) + 1) * kMaxWsum + threadIdx.x] = v * inv_gscale;
  }
}
int wsum_rows(int64_t pixels, int C) {
  int64_t b = (pixels * (C / 8) + 255) / 256;
  if (b < 1) b = 1;
  if (b > 132 * 2) b = 132 * 2;
  return static_cast<int>(b);
}
int wsum_fwd_launch(int K, int64_t pixels, int C, const void* const* xs, const int* xcs, const float* wts, void* out, int ocs,
                    cudaStream_t stream) {
  if (K < 1 || K > kMaxWsum) return set_error(FSB_ERR_INVALID, "wsum: 1 <= K <= 8");
  WsumArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  for (int k = 0; k < K; ++k) {
    if (!vec_ok(C, xcs[k], xs[k])) return set_error(FSB_ERR_INVALID, "wsum: C/strides multiples of 8, pointers 16B aligned");
    a.x[k] = static_cast<const __half*>(xs[k]);
    a.xcs[k] = xcs[k];
  }
  if (!vec_ok(C, ocs, out)) return set_error(FSB_ERR_INVALID, "wsum: bad output view");
  FSB_LAUNCH(wsum_fwd_kernel, dim3(grid_for(pixels * (C / 8), 256)), dim3(256), 0, stream, a, pixels, C / 8, wts,
             static_cast<__half*>(out), ocs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "wsum_fwd launch");
  return FSB_OK;
}
int wsum_bwd_launch(int K, int64_t pixels, int C, const void* dout, int docs, const void* const* xs, const int* xcs,
                    const float* wts, void* const* dxs, const int* dxcs, float* dwts, float gscale, cudaStream_t stream) {
  if (K < 1 || K > kMaxWsum) return set_error(FSB_ERR_INVALID, "wsum: 1 <= K <= 8");
  WsumArgs a;
  memset(&a, 0, sizeof(a));
  a.K = K;
  for (int k = 0; k < K; ++k) {
    if (xs && xs[k]) {
      if (!vec_ok(C, xcs[k], xs[k])) return set_error(FSB_ERR_INVALID, "wsum_bwd: bad x view");
      a.x[k] = static_cast<const __half*>(xs[k]);
      a.xcs[k] = xcs[k];
    } else if (dwts) {
      return set_error(FSB_ERR_INVALID, "wsum_bwd: dwts needs every xs[k]");
    }
    if (dxs && dxs[k]) {
      if (!vec_ok(C, dxcs[k], dxs[k])) return set_error(FSB_ERR_INVALID, "wsum_bwd: bad dx view");
      a.dx[k] = static_cast<__half*>(dxs[k]);
      a.dxcs[k] = dxcs[k];
    }
  }
  if (!vec_ok(C, docs, dout)) return set_error(FSB_ERR_INVALID, "wsum_bwd: bad dout view");
  // with scalar gradients the grid is capped so that the (1 + rows) x 8 partial buffer stays small; dwts[0..8) = totals
  const unsigned grid = dwts ? static_cast<unsigned>(wsum_rows(pixels, C)) : grid_for(pixels * (C / 8), 256);
  FSB_LAUNCH(wsum_bwd_kernel, dim3(grid), dim3(256), 0, stream, a, pixels, C / 8,
             static_cast<const __half*>(dout), docs, wts, dwts, 1.0f / gscale);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "wsum_bwd launch");
  if (dwts) return rowsum_launch(kMaxWsum, dwts + kMaxWsum, static_cast<int>(grid), kMaxWsum, dwts, stream);
  return FSB_OK;
}

__global__ void __launch_bounds__(256)
add_inplace_kernel(int64_t pixels, int cvec, const __half* __restrict__ x, int xcs, __half* __restrict__ y, int ycs) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t p = i / cvec;
    float a[8], b[8];
    unpack8(*reinterpret_cast<const uint4*>(x + p * xcs + cv * 8), a);
    unpack8(*reinterpret_cast<const uint4*>(y + p * ycs + cv * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] += a[j];
    *reinterpret_cast<uint4*>(y + p * ycs + cv * 8) = pack8(b);
  }
}
int add_inplace_launch(int64_t pixels, int C, const void* x, int xcs, void* y, int ycs, cudaStream_t stream) {
  if (!vec_ok(C, xcs, x) || !vec_ok(C, ycs, y)) return set_error(FSB_ERR_INVALID, "add_inplace: bad views");
  FSB_LAUNCH(add_inplace_kernel, dim3(grid_for(pixels * (C / 8), 256)), dim3(256), 0, stream, pixels, C / 8,
             static_cast<const __half*>(x), xcs, static_cast<__half*>(y), ycs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "add_inplace launch");
  return FSB_OK;
}

}  // namespace fsb
