// conv_direct.cu -- CUDA-core convolution kernels + weight packing.
//   * pack_conv_weight_kernel : fp32 OIHW (max-width, sliced) -> fp16 [tap][Npad][Kpad] for the tensor-core kernels
//   * conv_direct_kernel      : generic NHWC fp16 direct conv on the same packed weights (Cin < 16, odd strides of
//                               the API, and the device-side cross-check of the tensor-core kernel in tests)
//   * stem_conv_nchw_kernel   : 3x3 s2 p1 RGB stem reading the caller's NCHW fp32/fp16 tensor directly, so the
//                               NCHW->NHWC layout change and the fp32->fp16 cast cost no extra HBM round trip
//                               (ConvNorm at train/model_seg.py:193, search/model_search.py:148)
#include <type_traits>

#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

int bn_stats_rows_launch(int64_t pixels, int C, const void* x, int xcs, int x_is_f32, float* rows, int SC, cudaStream_t stream);

// ------------------------------------------------------------------------------------------
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, int64_t so, int64_t si, int taps, int Cout, int Cin,
                                        int npad, int kpad, __half* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = static_cast<int64_t>(taps) * npad * kpad;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % kpad);
    const int n = static_cast<int>((i / kpad) % npad);
    const int tap = static_cast<int>(i / (static_cast<int64_t>(kpad) * npad));
    float v = 0.f;
    if (n < Cout && k < Cin) v = w[n * so + k * si + tap];
    out[i] = __float2half_rn(v);
  }
}

int pack_conv_weight(const fsb_conv_desc* d, const float* w, int64_t so, int64_t si, void* packed, cudaStream_t stream) {
  const ConvGeom g = conv_geom(d);
  const int64_t total = static_cast<int64_t>(g.taps) * g.npad * g.kpad;
  int blocks = static_cast<int>((total + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  FSB_LAUNCH(pack_conv_weight_kernel, dim3(blocks), dim3(256), 0, stream, w, so, si, g.taps, d->Cout, d->Cin, g.npad, g.kpad,
                                                      static_cast<__half*>(packed));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "pack_conv_weight");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// generic direct conv: one thread = one output pixel x 8 output channels
// ------------------------------------------------------------------------------------------
struct DirectParams {
  fsb_conv_desc d;
  int npad, kpad, taps;
  const __half* x;
  const __half* w;
  const float* scale;
  const float* shift;
  __half* y;
  float* stats;
};

__global__ void __launch_bounds__(128) conv_direct_kernel(const DirectParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const fsb_conv_desc& d = p.d;
  const int64_t npix = static_cast<int64_t>(d.N) * d.Ho * d.Wo;
  const int cgroups = (d.Cout + 7) / 8;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= npix * cgroups) return;
  const int cg = static_cast<int>(gid % cgroups);
  const int64_t pix = gid / cgroups;
  const int wo = static_cast<int>(pix % d.Wo);
  const int ho = static_cast<int>((pix / d.Wo) % d.Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(d.Wo) * d.Ho));
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int r = 0; r < d.ksize; ++r) {
    const int hi = ho * d.stride + r * d.dil - d.pad + d.off_h;
    if (hi < 0 || hi >= d.H) continue;
    for (int s = 0; s < d.ksize; ++s) {
      const int wi = wo * d.stride + s * d.dil - d.pad + d.off_w;
      if (wi < 0 || wi >= d.W) continue;
      const __half* xp = p.x + (static_cast<size_t>(n) * d.H * d.W + static_cast<size_t>(hi) * d.W + wi) * d.x_cstride;
      const __half* wp = p.w + (static_cast<size_t>(r * d.ksize + s) * p.npad + cg * 8) * p.kpad;
      for (int c = 0; c < d.Cin; ++c) {
        const float xv = __half2float(xp[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(xv, __half2float(wp[static_cast<size_t>(j) * p.kpad + c]), acc[j]);
      }
    }
  }
  __half* yp = p.y + static_cast<size_t>(pix) * d.y_cstride + cg * 8;
  float* yp32 = reinterpret_cast<float*>(p.y) + static_cast<size_t>(pix) * d.y_cstride + cg * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = cg * 8 + j;
    if (ch >= d.Cout) break;
    float v = acc[j];
    if (d.flags & FSB_CONV_AFFINE) v = v * (p.scale ? p.scale[ch] : 1.f) + (p.shift ? p.shift[ch] : 0.f);
    if (d.flags & FSB_CONV_RELU) v = fmaxf(v, 0.f);
    if (d.flags & FSB_CONV_OUT_F32)
      yp32[j] = v;
    else
      yp[j] = __float2half_rn(v);
  }
}

int conv_direct_launch(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                       void* y, float* stats, cudaStream_t stream) {
  const ConvGeom g = conv_geom(d);
  DirectParams p;
  p.d = *d;
  p.npad = g.npad;
  p.kpad = g.kpad;
  p.taps = g.taps;
  p.x = static_cast<const __half*>(x);
  p.w = static_cast<const __half*>(wpacked);
  p.scale = scale;
  p.shift = shift;
  p.y = static_cast<__half*>(y);
  // the statistics are taken in a second pass over the output (partial rows, no atomics: bn.cu)
  const bool want_stats = (d->flags & FSB_CONV_STATS) && stats;
  p.stats = nullptr;
  p.d.flags &= ~FSB_CONV_STATS;
  const int64_t total = static_cast<int64_t>(d->N) * d->Ho * d->Wo * ((d->Cout + 7) / 8);
  const int64_t blocks = (total + 127) / 128;
  FSB_LAUNCH(conv_direct_kernel, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, stream, p);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "conv_direct launch");
  if (want_stats) {
    if (d->flags & (FSB_CONV_AFFINE | FSB_CONV_RELU)) return set_error(FSB_ERR_INVALID, "conv_direct: STATS needs a raw (no epilogue) output");
    const int SC = d->stats_C > 0 ? d->stats_C : d->Cout;
    return bn_stats_rows_launch(static_cast<int64_t>(d->N) * d->Ho * d->Wo, d->Cout, y, d->y_cstride,
                                (d->flags & FSB_CONV_OUT_F32) ? 1 : 0, stats + d->stats_off, SC, stream);
  }
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// RGB stem: NCHW in (fp32 or fp16), NHWC fp16 out, 3x3 stride 2 pad 1, fused affine + ReLU.
// One thread = one output pixel x 16 output channels; weights (27 x Cout fp32) live in shared memory and are
// read as warp-wide broadcasts.  HBM-bound: 2*3*H*W*4 B in (fp32) + Cout*H*W/4*2 B out.
// ------------------------------------------------------------------------------------------
template <typename TIn>
__global__ void __launch_bounds__(256)
stem_conv_nchw_kernel(int N, int H, int W, int Cout, const TIn* __restrict__ x, const float* __restrict__ w,
                      const float* __restrict__ scale, const float* __restrict__ shift, __half* __restrict__ y,
                      int y_cstride, uint32_t flags) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_w[];  // [27][CoutPad16] then scale[CoutPad16], shift[CoutPad16]
  const int Ho = H / 2 + (H & 1), Wo = W / 2 + (W & 1);  // floor((H + 2 - 3)/2) + 1
  const int cpad = (Cout + 15) / 16 * 16;
  for (int i = threadIdx.x; i < 27 * cpad; i += blockDim.x) {
    const int co = i % cpad, t = i / cpad;  // t = ci*9 + r*3 + s (OIHW inner order)
    s_w[i] = (co < Cout) ? w[static_cast<size_t>(co) * 27 + t] : 0.f;
  }
  float* s_scale = s_w + 27 * cpad;
  float* s_shift = s_scale + cpad;
  for (int i = threadIdx.x; i < cpad; i += blockDim.x) {
    const bool aff = (flags & FSB_CONV_AFFINE) && i < Cout;
    s_scale[i] = (aff && scale) ? scale[i] : 1.f;
    s_shift[i] = (aff && shift) ? shift[i] : 0.f;
  }
  __syncthreads();
  const int groups = cpad / 16;
  const int wo = blockIdx.x * blockDim.x + threadIdx.x;
  const int ho = blockIdx.y;
  const int n = blockIdx.z / groups;
  const int grp = blockIdx.z % groups;
  if (wo >= Wo) return;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  const size_t plane = static_cast<size_t>(H) * W;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = ho * 2 + r - 1;
      const bool hok = hi >= 0 && hi < H;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int wi = wo * 2 + s - 1;
        float xv = 0.f;
        if (hok && wi >= 0 && wi < W) xv = static_cast<float>(x[(static_cast<size_t>(n) * 3 + ci) * plane + static_cast<size_t>(hi) * W + wi]);
        const float4* wp = reinterpret_cast<const float4*>(s_w + (ci * 9 + r * 3 + s) * cpad + grp * 16);
#pragma unroll
        for (int j4 = 0; j4 < 4; ++j4) {
          const float4 wv = wp[j4];
          acc[j4 * 4 + 0] = fmaf(xv, wv.x, acc[j4 * 4 + 0]);
          acc[j4 * 4 + 1] = fmaf(xv, wv.y, acc[j4 * 4 + 1]);
          acc[j4 * 4 + 2] = fmaf(xv, wv.z, acc[j4 * 4 + 2]);
          acc[j4 * 4 + 3] = fmaf(xv, wv.w, acc[j4 * 4 + 3]);
        }
      }
    }
  }
  const bool relu = flags & FSB_CONV_RELU;
  __half* yp = y + (static_cast<size_t>(n) * Ho * Wo + static_cast<size_t>(ho) * Wo + wo) * y_cstride + grp * 16;
  float f[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    float v = acc[j] * s_scale[grp * 16 + j] + s_shift[grp * 16 + j];
    f[j] = relu ? fmaxf(v, 0.f) : v;
  }
  const int remaining = Cout - grp * 16;
  if (remaining >= 16 && (reinterpret_cast<uintptr_t>(yp) & 15) == 0) {
    uint4 o0, o1;
    o0.x = pack_half2(f[0], f[1]);
    o0.y = pack_half2(f[2], f[3]);
    o0.z = pack_half2(f[4], f[5]);
    o0.w = pack_half2(f[6], f[7]);
    o1.x = pack_half2(f[8], f[9]);
    o1.y = pack_half2(f[10], f[11]);
    o1.z = pack_half2(f[12], f[13]);
    o1.w = pack_half2(f[14], f[15]);
    reinterpret_cast<uint4*>(yp)[0] = o0;
    reinterpret_cast<uint4*>(yp)[1] = o1;
  } else {
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (j < remaining) yp[j] = __float2half_rn(f[j]);
  }
}

// ------------------------------------------------------------------------------------------
// RGB stem on the tensor cores: a CTA (128 threads) owns 128 consecutive output pixels of one output row.  Thread t
// gathers the 27 inputs of its pixel straight from the NCHW tensor (warp-coalesced per (channel,row)), converts to
// fp16 and writes row t of a 128 x 32 K-major A tile in the SWIZZLE_64B canonical layout (K = 27 padded to 32); the
// OIHW weights are laid out the same way as the B tile.  The CTA is one warpgroup: four wgmma (two m64 halves x K = 16 each)
// produce the 128 x NP fp32 tile in registers, parked in shared memory as [channel][pixel]; the epilogue applies BN
// scale/shift + ReLU and each thread stores its pixel's Cout fp16 values contiguously (a warp writes 32 x 2*Cout contiguous
// bytes).  No im2col buffer, no fp16 NHWC copy of the image.
// ------------------------------------------------------------------------------------------
// TIn = uint8_t: the frame is the camera / dataset image itself, uint8 HWC (tools/engine/evaluator.py:206-225 hands the model
// `normalize(img, mean, std)` = (img / 255 - mean) / std as fp32 CHW, evaluator.py:329, tools/utils/img_utils.py:179-185).  The
// normalisation is a 3 x 256 lookup table of fp16 values (exactly the fp16 rounding of what the reference computes for each
// byte value), so the H2D copy shrinks 4x and the result is bit-identical to feeding the normalised fp32 image.
constexpr int kStemAccLd = 128 + 4;  // padded channel column of the parked accumulator (conflict-free stores and reads)

template <typename TIn, int NP>  // NP: wgmma N, Cout rounded up to 32 or 64
__global__ void __launch_bounds__(128)
stem_conv_tc_kernel(int N, int H, int W, int Cout, int npad, const TIn* __restrict__ x, const float* __restrict__ w,
                    const float* __restrict__ scale, const float* __restrict__ shift, __half* __restrict__ y,
                    int y_cstride, uint32_t flags, const __half* __restrict__ lut) {
  __shared__ __align__(1024) uint8_t s_a[128 * 64];
  __shared__ __half s_lut[std::is_same<TIn, uint8_t>::value ? 768 : 2];
  __shared__ __align__(1024) uint8_t s_b[64 * 64];
  __shared__ float s_scale[64];
  __shared__ float s_shift[64];
  __shared__ float s_acc[NP * kStemAccLd];
  pdl_launch_dependents();
  const int t = threadIdx.x;
  const int Ho = H / 2 + (H & 1), Wo = W / 2 + (W & 1);
  const int wo = blockIdx.x * 128 + t;
  const int ho = blockIdx.y;
  const int n = blockIdx.z;
  pdl_wait();  // weights / scale / shift may have been produced by the immediately preceding kernel
  if constexpr (std::is_same<TIn, uint8_t>::value) {
    for (int i = t; i < 768; i += 128) s_lut[i] = lut[i];
    __syncthreads();
  }
  // weights -> B tile rows (one thread per output channel, zero rows up to NP), fp32 OIHW is already [co][27]
  if (t < NP) {
    __half hv[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) hv[k] = __float2half_rn((t < Cout && k < 27) ? w[t * 27 + k] : 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint4*>(s_b + t * 64 + ((j ^ ((t >> 1) & 3)) << 4)) = *reinterpret_cast<const uint4*>(&hv[j * 8]);
    const bool aff = (flags & FSB_CONV_AFFINE) && t < Cout;
    s_scale[t] = (aff && scale) ? scale[t] : 1.f;
    s_shift[t] = (aff && shift) ? shift[t] : 0.f;
  }
  // im2col row of this thread's pixel
  {
    __half hv[32];
    const size_t plane = static_cast<size_t>(H) * W;
    const bool pix = wo < Wo;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int hi = ho * 2 + r - 1;
        const bool hok = pix && hi >= 0 && hi < H;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int wi = wo * 2 + s - 1;
          if constexpr (std::is_same<TIn, uint8_t>::value) {
            __half hvv = __float2half_rn(0.f);   // zero padding of the NORMALISED image, like the reference's conv
            if (hok && wi >= 0 && wi < W)
              hvv = s_lut[ci * 256 + x[((static_cast<size_t>(n) * H + hi) * W + wi) * 3 + ci]];
            hv[ci * 9 + r * 3 + s] = hvv;
          } else {
            float v = 0.f;
            if (hok && wi >= 0 && wi < W) v = static_cast<float>(x[(static_cast<size_t>(n) * 3 + ci) * plane + static_cast<size_t>(hi) * W + wi]);
            hv[ci * 9 + r * 3 + s] = __float2half_rn(v);
          }
        }
      }
    }
#pragma unroll
    for (int k = 27; k < 32; ++k) hv[k] = __float2half_rn(0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint4*>(s_a + t * 64 + ((j ^ ((t >> 1) & 3)) << 4)) = *reinterpret_cast<const uint4*>(&hv[j * 8]);
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy smem writes -> visible to the MMA (async proxy)
  __syncthreads();
  {
    float acc[2][NP / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) acc[h][i] = 0.f;
    const uint64_t da = wgmma_desc_kmajor(smem_u32(s_a), 64);
    const uint64_t db = wgmma_desc_kmajor(smem_u32(s_b), 64);
    constexpr uint64_t kHalf = (64 * 64) >> 4;  // pixel rows 64..127 of the A tile
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k) {  // K = 32 = two steps of 16 fp16 (32 B, +2 in the address field)
      wgmma_f16<NP, 0>(acc[0], da + 2 * k, db + 2 * k);
      wgmma_f16<NP, 0>(acc[1], da + kHalf + 2 * k, db + 2 * k);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NP / 2; ++i) s_acc[wgmma_col(t, i) * kStemAccLd + 64 * h + wgmma_row(t, i)] = acc[h][i];
  }
  __syncthreads();
  const bool relu = flags & FSB_CONV_RELU;
  __half* yp = y + (static_cast<size_t>(n) * Ho * Wo + static_cast<size_t>(ho) * Wo + wo) * y_cstride;
  for (int c = 0; c < npad; c += 16) {
    float f[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float a = s_acc[(c + j) * kStemAccLd + t] * s_scale[c + j] + s_shift[c + j];
      f[j] = relu ? fmaxf(a, 0.f) : a;
    }
    if (wo < Wo) {
      const int remaining = Cout - c;
      if (remaining >= 16 && (reinterpret_cast<uintptr_t>(yp + c) & 15) == 0) {
        uint4 o0, o1;
        o0.x = pack_half2(f[0], f[1]);
        o0.y = pack_half2(f[2], f[3]);
        o0.z = pack_half2(f[4], f[5]);
        o0.w = pack_half2(f[6], f[7]);
        o1.x = pack_half2(f[8], f[9]);
        o1.y = pack_half2(f[10], f[11]);
        o1.z = pack_half2(f[12], f[13]);
        o1.w = pack_half2(f[14], f[15]);
        reinterpret_cast<uint4*>(yp + c)[0] = o0;
        reinterpret_cast<uint4*>(yp + c)[1] = o1;
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (j < remaining) yp[c + j] = __float2half_rn(f[j]);
      }
    }
  }
}

int stem_conv_nchw_launch(int N, int H, int W, int Cout, const void* x, int x_is_f32, const float* w, const float* scale,
                          const float* shift, void* y, int y_cstride, uint32_t flags, cudaStream_t stream) {
  const int Ho = H / 2 + (H & 1), Wo = W / 2 + (W & 1);
  const int cpad = (Cout + 15) / 16 * 16;
  if (cpad <= 64 && !(flags & FSB_CONV_FORCE_DIRECT)) {
    dim3 grid_tc((Wo + 127) / 128, Ho, N);
    const __half* no_lut = nullptr;
    if (x_is_f32) {
      if (cpad <= 32)
        FSB_LAUNCH(stem_conv_tc_kernel<float, 32>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, static_cast<const float*>(x), w,
                   scale, shift, static_cast<__half*>(y), y_cstride, flags, no_lut);
      else
        FSB_LAUNCH(stem_conv_tc_kernel<float, 64>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, static_cast<const float*>(x), w,
                   scale, shift, static_cast<__half*>(y), y_cstride, flags, no_lut);
    } else {
      if (cpad <= 32)
        FSB_LAUNCH(stem_conv_tc_kernel<__half, 32>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, static_cast<const __half*>(x),
                   w, scale, shift, static_cast<__half*>(y), y_cstride, flags, no_lut);
      else
        FSB_LAUNCH(stem_conv_tc_kernel<__half, 64>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, static_cast<const __half*>(x),
                   w, scale, shift, static_cast<__half*>(y), y_cstride, flags, no_lut);
    }
    cudaError_t e2 = last_launch_error();
    if (e2 != cudaSuccess) return set_cuda_error(e2, "stem_conv_tc launch");
    return FSB_OK;
  }
  const int groups = cpad / 16;
  const size_t smem = static_cast<size_t>(27 + 2) * cpad * sizeof(float);
  dim3 block(Wo >= 256 ? 256 : 128);
  dim3 grid((Wo + block.x - 1) / block.x, Ho, N * groups);
  if (x_is_f32)
    FSB_LAUNCH(stem_conv_nchw_kernel<float>, dim3(grid), dim3(block), smem, stream, N, H, W, Cout, static_cast<const float*>(x), w, scale, shift,
                                                                static_cast<__half*>(y), y_cstride, flags);
  else
    FSB_LAUNCH(stem_conv_nchw_kernel<__half>, dim3(grid), dim3(block), smem, stream, N, H, W, Cout, static_cast<const __half*>(x), w, scale,
                                                                 shift, static_cast<__half*>(y), y_cstride, flags);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "stem_conv_nchw launch");
  return FSB_OK;
}

int stem_conv_u8hwc_launch(int N, int H, int W, int Cout, const uint8_t* x, const void* lut, const float* w, const float* scale,
                           const float* shift, void* y, int y_cstride, uint32_t flags, cudaStream_t stream) {
  const int Ho = H / 2 + (H & 1), Wo = W / 2 + (W & 1);
  const int cpad = (Cout + 15) / 16 * 16;
  if (cpad > 64) return set_error(FSB_ERR_UNSUPPORTED, "stem_conv_u8hwc: Cout <= 64");
  dim3 grid_tc((Wo + 127) / 128, Ho, N);
  if (cpad <= 32)
    FSB_LAUNCH(stem_conv_tc_kernel<uint8_t, 32>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, x, w, scale, shift,
               static_cast<__half*>(y), y_cstride, flags, static_cast<const __half*>(lut));
  else
    FSB_LAUNCH(stem_conv_tc_kernel<uint8_t, 64>, grid_tc, dim3(128), 0, stream, N, H, W, Cout, cpad, x, w, scale, shift,
               static_cast<__half*>(y), y_cstride, flags, static_cast<const __half*>(lut));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "stem_conv_u8hwc launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// confusion matrix of a predicted label map against the ground truth (tools/seg_opr/metric.py:7-15 hist_info):
//   k = (gt >= 0) & (gt < n_cl);  hist[n_cl * gt + pred] += 1 over k;  labeled = sum(k);  correct = sum(pred == gt over k)
// per-block shared-memory histogram, then integer atomics (exact and order-independent).  out: int64 [n_cl * n_cl + 2].
// ------------------------------------------------------------------------------------------
template <typename TGt>
__global__ void __launch_bounds__(256)
confusion_kernel(int64_t n, const uint8_t* __restrict__ pred, const TGt* __restrict__ gt, int n_cl, unsigned long long* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ unsigned int s_hist[];  // n_cl * n_cl + 2
  const int cells = n_cl * n_cl + 2;
  for (int i = threadIdx.x; i < cells; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const long long g = static_cast<long long>(gt[i]);
    if (g < 0 || g >= n_cl) continue;
    const int p = pred[i];
    if (p < n_cl) atomicAdd(&s_hist[g * n_cl + p], 1u);
    atomicAdd(&s_hist[n_cl * n_cl], 1u);
    if (p == g) atomicAdd(&s_hist[n_cl * n_cl + 1], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cells; i += blockDim.x)
    if (s_hist[i]) atomicAdd(&out[i], static_cast<unsigned long long>(s_hist[i]));
}
int confusion_launch(int64_t n, const uint8_t* pred, const void* gt, int gt_bytes, int n_cl, long long* out, cudaStream_t stream) {
  if (n_cl < 1 || n_cl > 64) return set_error(FSB_ERR_INVALID, "confusion_matrix: 1 <= n_cl <= 64");
  int64_t blocks = (n + 256 * 16 - 1) / (256 * 16);
  if (blocks < 1) blocks = 1;
  if (blocks > 132 * 8) blocks = 132 * 8;
  const size_t smem = static_cast<size_t>(n_cl * n_cl + 2) * sizeof(unsigned int);
  unsigned long long* o = reinterpret_cast<unsigned long long*>(out);
  if (gt_bytes == 1)
    FSB_LAUNCH(confusion_kernel<uint8_t>, dim3(static_cast<unsigned>(blocks)), dim3(256), smem, stream, n, pred, static_cast<const uint8_t*>(gt), n_cl, o);
  else if (gt_bytes == 4)
    FSB_LAUNCH(confusion_kernel<int32_t>, dim3(static_cast<unsigned>(blocks)), dim3(256), smem, stream, n, pred, static_cast<const int32_t*>(gt), n_cl, o);
  else if (gt_bytes == 8)
    FSB_LAUNCH(confusion_kernel<long long>, dim3(static_cast<unsigned>(blocks)), dim3(256), smem, stream, n, pred, static_cast<const long long*>(gt), n_cl, o);
  else
    return set_error(FSB_ERR_INVALID, "confusion_matrix: ground truth must be uint8, int32 or int64");
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "confusion_matrix launch");
  return FSB_OK;
}

}  // namespace fsb
