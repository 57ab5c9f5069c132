// bn.cu -- BatchNorm kernels: eval-mode folding, training statistics (K2), running-stat update (K3), apply.
// nn.BatchNorm2d semantics of the reference (search/operations.py:79-83 etc., USBatchNorm2d search/slimmable_ops.py:51-70):
//   eval : y = (x - running_mean) / sqrt(running_var + eps) * gamma + beta
//   train: batch mean, BIASED var for normalisation; running = (1-m)*running + m*{mean, UNBIASED var}
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

__global__ void bn_fold_kernel(int C, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                               const float* conv_bias, float* scale, float* shift) {
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float g = gamma ? gamma[c] : 1.f;
  const float b = beta ? beta[c] : 0.f;
  const float s = g / sqrtf(var[c] + eps);
  float sh = b - mean[c] * s;
  if (conv_bias) sh += conv_bias[c] * s;
  scale[c] = s;
  shift[c] = sh;
}
int bn_fold_launch(int C, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                   const float* conv_bias, float* scale, float* shift, cudaStream_t stream) {
  FSB_LAUNCH(bn_fold_kernel, dim3((C + 127) / 128), dim3(128), 0, stream, C, gamma, beta, mean, var, eps, conv_bias, scale, shift);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bn_fold launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// Deterministic statistics.  No kernel of this library accumulates BatchNorm statistics with floating-point atomics
// (their arrival order changes from run to run, and a chain of BatchNorm layers amplifies the last-bit differences into
// percent-level gradient differences).  Instead every producer CTA writes ONE partial row
//     row[r][0 .. SC)  = per-channel sum,   row[r][SC .. 2*SC) = per-channel sum of squares   (row stride 2*SC floats)
// and the consumer adds the rows in index order (bn_finalize folds that in; rowsum_kernel is the stand-alone form).
// ------------------------------------------------------------------------------------------
// FactorizedReduce at maximum width (captured training graphs): conv1 writes raw channels [0, hmax), conv2 [hmax, 2*hmax),
// but with an active half-width h < hmax the BatchNorm set and every consumer see the COMPACT order [conv1[0..h) | conv2[0..h) |
// inactive...].  remap() is the bijection compact channel -> raw ("expanded") channel; all quantities are multiples of 8 and
// the kernels apply it per 8-channel vector.  hmax == 0 disables it.
__host__ __device__ __forceinline__ int split_remap(int c, int h, int hmax) {
  if (hmax <= 0) return c;
  if (c < h) return c;
  if (c < 2 * h) return hmax + (c - h);
  const int k = c - 2 * h;
  return k < hmax - h ? h + k : hmax + h + (k - (hmax - h));
}

int stat_rows(int64_t pixels) {
  int64_t b = (pixels + 255) / 256;
  if (b < 1) b = 1;
  if (b > 132 * 2) b = 132 * 2;
  return static_cast<int>(b);
}

// out[c] = sum_r rows[r * stride + c], r ascending, accumulated in double: one block = 32 columns x 8 row lanes
__global__ void __launch_bounds__(256) rowsum_kernel(int L, const float* __restrict__ rows, int P, int stride, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sh[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  double acc = 0.0;
  if (c < L)
    for (int r = ty; r < P; r += 8) acc += static_cast<double>(rows[static_cast<size_t>(r) * stride + c]);
  sh[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < L) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sh[k][tx];
    out[c] = static_cast<float>(t);
  }
}
int rowsum_launch(int L, const float* rows, int P, int stride, float* out, cudaStream_t stream) {
  FSB_LAUNCH(rowsum_kernel, dim3((L + 31) / 32), dim3(256), 0, stream, L, rows, P, stride, out);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "rowsum launch");
  return FSB_OK;
}

// per-channel sum / sumsq of an fp16 NHWC tensor.  Block = 256 threads = (256 / cvec_lanes) pixel rows x channel
// vectors; each thread owns 8 channels (one 16-byte load per pixel), accumulates in fp32 registers, then the block
// reduces through shared memory in a fixed order and writes its partial row (blockIdx.x).
__global__ void __launch_bounds__(256)
bn_stats_kernel(int64_t pixels, int C, const __half* __restrict__ x, int xcs, float* __restrict__ rows_out, int SC) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float red[];  // [rows][C*2]
  const int cvec = C >> 3;
  const int rows = blockDim.x / cvec;
  const int cv = threadIdx.x % cvec;
  const int row = threadIdx.x / cvec;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  if (row < rows) {
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * rows + row; p < pixels; p += static_cast<int64_t>(gridDim.x) * rows) {
      const uint4 v = *reinterpret_cast<const uint4*>(x + p * xcs + cv * 8);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        s[2 * j] += f.x;
        q[2 * j] += f.x * f.x;
        s[2 * j + 1] += f.y;
        q[2 * j + 1] += f.y * f.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      red[(row * C + cv * 8 + j) * 2 + 0] = s[j];
      red[(row * C + cv * 8 + j) * 2 + 1] = q[j];
    }
  }
  __syncthreads();
  float* out = rows_out + static_cast<size_t>(blockIdx.x) * 2 * SC;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < rows; ++r) {
      a += red[(r * C + c) * 2 + 0];
      b += red[(r * C + c) * 2 + 1];
    }
    out[c] = a;
    out[SC + c] = b;
  }
}
// generic (any C / stride) fallback: block = 32 channels x 8 pixel rows
template <typename T>
__global__ void __launch_bounds__(256)
bn_stats_generic_kernel(int64_t pixels, int C, const T* __restrict__ x, int xcs, float* __restrict__ rows_out, int SC) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[8][32][2];
  const int c = blockIdx.y * 32 + (threadIdx.x & 31);
  const int row = threadIdx.x >> 5;
  float s = 0.f, q = 0.f;
  if (c < C)
    for (int64_t p = static_cast<int64_t>(blockIdx.x) * 8 + row; p < pixels; p += static_cast<int64_t>(gridDim.x) * 8) {
      const float v = static_cast<float>(x[p * xcs + c]);
      s += v;
      q += v * v;
    }
  red[row][threadIdx.x & 31][0] = s;
  red[row][threadIdx.x & 31][1] = q;
  __syncthreads();
  if (row == 0 && c < C) {
    for (int r = 1; r < 8; ++r) {
      s += red[r][threadIdx.x][0];
      q += red[r][threadIdx.x][1];
    }
    float* out = rows_out + static_cast<size_t>(blockIdx.x) * 2 * SC;
    out[c] = s;
    out[SC + c] = q;
  }
}

// writes stat_rows(pixels) partial rows (row stride 2*SC; `rows` already points at the channel offset of this tensor)
int bn_stats_rows_launch(int64_t pixels, int C, const void* x, int xcs, int x_is_f32, float* rows, int SC, cudaStream_t stream) {
  const int P = stat_rows(pixels);
  if (x_is_f32 || C % 8 || xcs % 8 || C > 2048 || (reinterpret_cast<uintptr_t>(x) & 15)) {
    if (x_is_f32)
      FSB_LAUNCH(bn_stats_generic_kernel<float>, dim3(static_cast<unsigned>(P), (C + 31) / 32), dim3(256), 0, stream, pixels, C,
                 static_cast<const float*>(x), xcs, rows, SC);
    else
      FSB_LAUNCH(bn_stats_generic_kernel<__half>, dim3(static_cast<unsigned>(P), (C + 31) / 32), dim3(256), 0, stream, pixels, C,
                 static_cast<const __half*>(x), xcs, rows, SC);
    cudaError_t e0 = last_launch_error();
    if (e0 != cudaSuccess) return set_cuda_error(e0, "bn_stats_generic launch");
    return FSB_OK;
  }
  const int cvec = C / 8;
  const int threads = 256;
  if (cvec > threads) return set_error(FSB_ERR_INVALID, "bn_stats: C too large");
  const int rows_per = threads / cvec;
  const size_t smem = static_cast<size_t>(rows_per) * C * 2 * sizeof(float);
  FSB_LAUNCH(bn_stats_kernel, dim3(static_cast<unsigned>(P)), dim3(threads), smem, stream, pixels, C, static_cast<const __half*>(x), xcs, rows, SC);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bn_stats launch");
  return FSB_OK;
}
// buf: (1 + stat_rows(pixels)) rows of 2*C floats; row 0 receives the totals
int bn_stats_launch(int64_t pixels, int C, const void* x, int xcs, int x_is_f32, float* buf, cudaStream_t stream) {
  int rc = bn_stats_rows_launch(pixels, C, x, xcs, x_is_f32, buf + 2 * C, C, stream);
  if (rc) return rc;
  return rowsum_launch(2 * C, buf + 2 * C, stat_rows(pixels), 2 * C, buf, stream);
}

// One block = 32 channels x 16 row lanes: adds the partial rows in index order (double), then finalises.
// sel != nullptr ("selected" mode, used by the captured training graphs): the BatchNorm parameter set of this launch is
// chosen ON THE DEVICE -- sel[*width_idx] -- and channels >= its active width get scale = shift = 0, i.e. the unit runs at
// its maximum width with the inactive tail forced to zero (USBatchNorm2d / USConv2d semantics, search/slimmable_ops.py:36-69).
__global__ void __launch_bounds__(512)
bn_finalize_kernel(int C, const float* __restrict__ stats, int P, int SC, double count, const float* gamma, const float* beta, float eps,
                   float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                   float* save_mean, float* save_invstd, long long* num_batches_tracked, const fsb_bn_sel* sel, const int* width_idx,
                   int hmax) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double sh[16][32][2];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  int active = C;
  if (sel) {
    const fsb_bn_sel s = sel[*width_idx];
    gamma = s.gamma;
    beta = s.beta;
    running_mean = s.running_mean;
    running_var = s.running_var;
    num_batches_tracked = s.num_batches_tracked;
    active = s.C;
  }
  double s = 0.0, q = 0.0;
  if (c < C) {
    const size_t stride = 2 * static_cast<size_t>(SC);
    const int src = split_remap(c, active / 2, hmax);  // statistics columns are in raw channel order
    for (int r = ty; r < P; r += 16) {
      s += static_cast<double>(stats[r * stride + src]);
      q += static_cast<double>(stats[r * stride + SC + src]);
    }
  }
  sh[ty][tx][0] = s;
  sh[ty][tx][1] = q;
  __syncthreads();
  if (ty != 0) return;
  if (c == 0 && num_batches_tracked) *num_batches_tracked += 1;
  if (c >= C) return;
  s = 0.0;
  q = 0.0;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    s += sh[k][tx][0];
    q += sh[k][tx][1];
  }
  if (c >= active) {  // inactive tail of a slimmable unit running at max width
    if (scale) scale[c] = 0.f;
    if (shift) shift[c] = 0.f;
    if (save_mean) save_mean[c] = 0.f;
    if (save_invstd) save_invstd[c] = 0.f;
    return;
  }
  const double mean = s / count;
  double var = q / count - mean * mean;
  if (var < 0) var = 0;
  const float invstd = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  const float g = gamma ? gamma[c] : 1.f;
  const float b = beta ? beta[c] : 0.f;
  if (scale) scale[c] = g * invstd;
  if (shift) shift[c] = b - static_cast<float>(mean) * g * invstd;
  if (save_mean) save_mean[c] = static_cast<float>(mean);
  if (save_invstd) save_invstd[c] = invstd;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * static_cast<float>(mean);
  if (running_var) {
    const double unbiased = count > 1.0 ? var * (count / (count - 1.0)) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * static_cast<float>(unbiased);
  }
}
int bn_finalize_launch(int C, const float* stats, int P, int SC, double count, const float* gamma, const float* beta, float eps,
                       float momentum, float* running_mean, float* running_var, float* scale, float* shift, float* save_mean,
                       float* save_invstd, cudaStream_t stream, long long* num_batches_tracked, const fsb_bn_sel* sel,
                       const int* width_idx, int hmax) {
  FSB_LAUNCH(bn_finalize_kernel, dim3((C + 31) / 32), dim3(512), 0, stream, C, stats, P, SC, count, gamma, beta, eps, momentum,
             running_mean, running_var, scale, shift, save_mean, save_invstd, num_batches_tracked, sel, width_idx, hmax);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bn_finalize launch");
  return FSB_OK;
}

template <typename T>
__device__ __forceinline__ void load8f(const T* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load8f<__half>(const __half* p, float (&f)[8]) {
  const uint4 v = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = __half22float2(h[j]);
    f[2 * j] = t.x;
    f[2 * j + 1] = t.y;
  }
}
template <>
__device__ __forceinline__ void load8f<float>(const float* p, float (&f)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p);
  const float4 b = *reinterpret_cast<const float4*>(p + 4);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

template <typename T>
__global__ void __launch_bounds__(256)
affine_act_kernel(int64_t pixels, int cvec, const T* __restrict__ x, int xcs, const float* __restrict__ scale,
                  const float* __restrict__ shift, __half* __restrict__ y, int ycs, int relu, const fsb_bn_sel* sel,
                  const int* width_idx, int hmax) {
  pdl_launch_dependents();
  pdl_wait();
  const int h8 = (sel && hmax > 0) ? sel[*width_idx].C / 16 : 0;  // active half-width in 8-channel vectors (x is in raw order)
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t pix = i / cvec;
    float xin[8];
    load8f<T>(x + pix * xcs + split_remap(cv, h8, hmax >> 3) * 8, xin);
    const float4 s0 = *reinterpret_cast<const float4*>(scale + cv * 8);
    const float4 s1 = *reinterpret_cast<const float4*>(scale + cv * 8 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(shift + cv * 8);
    const float4 b1 = *reinterpret_cast<const float4*>(shift + cv * 8 + 4);
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float sf[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    uint4 out;
    uint32_t* o = reinterpret_cast<uint32_t*>(&out);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float r0 = xin[2 * j] * sc[2 * j] + sf[2 * j];
      float r1 = xin[2 * j + 1] * sc[2 * j + 1] + sf[2 * j + 1];
      if (relu) {
        r0 = fmaxf(r0, 0.f);
        r1 = fmaxf(r1, 0.f);
      }
      o[j] = pack_half2(r0, r1);
    }
    *reinterpret_cast<uint4*>(y + pix * ycs + cv * 8) = out;
  }
}
int affine_act_launch(int64_t pixels, int C, const void* x, int xcs, const float* scale, const float* shift, void* y, int ycs,
                      uint32_t flags, cudaStream_t stream, const fsb_bn_sel* sel, const int* width_idx, int hmax) {
  if (hmax > 0 && (!sel || !width_idx || hmax % 8 || C != 2 * hmax)) return set_error(FSB_ERR_INVALID, "affine_act: bad split arguments");
  if (C % 8 || xcs % 8 || ycs % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) ||
      (reinterpret_cast<uintptr_t>(scale) & 15) || (reinterpret_cast<uintptr_t>(shift) & 15))
    return set_error(FSB_ERR_INVALID, "affine_act: C/strides multiples of 8, pointers 16B aligned");
  const int64_t total = pixels * (C / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  if (flags & FSB_ACT_IN_F32)
    FSB_LAUNCH(affine_act_kernel<float>, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, pixels, C / 8,
               static_cast<const float*>(x), xcs, scale, shift, static_cast<__half*>(y), ycs, (flags & FSB_CONV_RELU) ? 1 : 0, sel,
               width_idx, hmax);
  else
    FSB_LAUNCH(affine_act_kernel<__half>, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, pixels, C / 8,
               static_cast<const __half*>(x), xcs, scale, shift, static_cast<__half*>(y), ycs, (flags & FSB_CONV_RELU) ? 1 : 0, sel,
               width_idx, hmax);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "affine_act launch");
  return FSB_OK;
}

}  // namespace fsb
