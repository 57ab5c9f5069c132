// resize.cu -- K4 / K9: bilinear (align_corners=True) resize kernels and layout plumbing, all HBM-bound:
// 16-byte vector loads/stores over the channel dimension of NHWC fp16, fp32 interpolation arithmetic.
// Reference call sites: F.interpolate at search/operations.py:271,275,437,444; search/model_search.py:339-343,353-357;
// train/model_seg.py:305,310,317,359-365.  Coordinate rule and interpolation: src_index / bilinear8 (fsb_common.cuh).
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

// one thread = one output pixel x 8 channels
__global__ void __launch_bounds__(256)
bilinear_nhwc_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                     __half* __restrict__ y, int ycs, float sh, float sw, int relu) {
  pdl_launch_dependents();
  pdl_wait();
  const int cvec = C >> 3;
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo * cvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int cv = static_cast<int>(gid % cvec);
  const int64_t pix = gid / cvec;
  const int wo = static_cast<int>(pix % Wo);
  const int ho = static_cast<int>((pix / Wo) % Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wo) * Ho));
  int h0, h1, w0, w1;
  float lh, lw;
  src_index(ho, sh, Hi, h0, h1, lh);
  src_index(wo, sw, Wi, w0, w1, lw);
  const __half* base = x + static_cast<size_t>(n) * Hi * Wi * xcs + cv * 8;
  const uint4 v00 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h0) * Wi + w0) * xcs);
  const uint4 v01 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h0) * Wi + w1) * xcs);
  const uint4 v10 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h1) * Wi + w0) * xcs);
  const uint4 v11 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h1) * Wi + w1) * xcs);
  *reinterpret_cast<uint4*>(y + static_cast<size_t>(pix) * ycs + cv * 8) = bilinear8(v00, v01, v10, v11, lh, lw, relu != 0);
}

// Exact x2 upsample (Ho = 2Hi, Wo = 2Wi) that also stores the bilinear /2 of its own output (Hi x Wi, y_half): one thread = one
// 2x2 output block x 8 channels.  Each of the four outputs is bilinear_nhwc_kernel's value; the /2 pixel (k, l) reads only rows
// 2k, 2k+1 and columns 2l, 2l+1 of the output (kBilinearLocalMax), i.e. this thread's four fp16 results.
__global__ void __launch_bounds__(256)
bilinear_up2_half_nhwc_kernel(int N, int C, int Hi, int Wi, const __half* __restrict__ x, int xcs, __half* __restrict__ y, int ycs,
                              __half* __restrict__ yh, int yhcs, float sh, float sw, float dh, float dw, int relu) {
  pdl_launch_dependents();
  pdl_wait();
  const int cvec = C >> 3;
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi * cvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int cv = static_cast<int>(gid % cvec);
  const int64_t blk = gid / cvec;
  const int l = static_cast<int>(blk % Wi);
  const int k = static_cast<int>((blk / Wi) % Hi);
  const int n = static_cast<int>(blk / (static_cast<int64_t>(Wi) * Hi));
  const int Ho = 2 * Hi, Wo = 2 * Wi;
  const __half* base = x + static_cast<size_t>(n) * Hi * Wi * xcs + cv * 8;
  __half* ybase = y + static_cast<size_t>(n) * Ho * Wo * ycs + cv * 8;
  uint4 r[2][2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    int h0, h1;
    float lh;
    src_index(2 * k + a, sh, Hi, h0, h1, lh);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      int w0, w1;
      float lw;
      src_index(2 * l + b, sw, Wi, w0, w1, lw);
      const uint4 v00 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h0) * Wi + w0) * xcs);
      const uint4 v01 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h0) * Wi + w1) * xcs);
      const uint4 v10 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h1) * Wi + w0) * xcs);
      const uint4 v11 = *reinterpret_cast<const uint4*>(base + (static_cast<size_t>(h1) * Wi + w1) * xcs);
      r[a][b] = bilinear8(v00, v01, v10, v11, lh, lw, relu != 0);
      *reinterpret_cast<uint4*>(ybase + (static_cast<size_t>(2 * k + a) * Wo + 2 * l + b) * ycs) = r[a][b];
    }
  }
  int h0, h1, w0, w1;
  float lh, lw;
  src_index(k, dh, Ho, h0, h1, lh);
  src_index(l, dw, Wo, w0, w1, lw);
  auto at = [&](int hh, int ww) {  // selects, not a dynamically indexed (local-memory) array
    const bool a = hh != 2 * k, b = ww != 2 * l;
    return a ? (b ? r[1][1] : r[1][0]) : (b ? r[0][1] : r[0][0]);
  };
  *reinterpret_cast<uint4*>(yh + (static_cast<size_t>(n) * Hi * Wi + static_cast<size_t>(k) * Wi + l) * yhcs + cv * 8) =
      bilinear8(at(h0, w0), at(h0, w1), at(h1, w0), at(h1, w1), lh, lw, false);
}

int bilinear_up2_half_launch(int N, int C, int Hi, int Wi, const void* x, int xcs, void* y, int ycs, void* y_half, int yhcs,
                             uint32_t flags, cudaStream_t stream) {
  if (C % 8 || xcs % 8 || ycs % 8 || yhcs % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) ||
      (reinterpret_cast<uintptr_t>(y_half) & 15))
    return set_error(FSB_ERR_INVALID, "bilinear_fwd_half: C, strides must be multiples of 8 and pointers 16B aligned");
  if (2 * Hi > kBilinearLocalMax || 2 * Wi > kBilinearLocalMax)
    return set_error(FSB_ERR_UNSUPPORTED, "bilinear_fwd_half: output extent beyond kBilinearLocalMax");
  const int64_t total = static_cast<int64_t>(N) * Hi * Wi * (C / 8);
  const int64_t blocks = (total + 255) / 256;
  FSB_LAUNCH(bilinear_up2_half_nhwc_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream,
      N, C, Hi, Wi, static_cast<const __half*>(x), xcs, static_cast<__half*>(y), ycs, static_cast<__half*>(y_half), yhcs,
      ac_scale(Hi, 2 * Hi), ac_scale(Wi, 2 * Wi), ac_scale(2 * Hi, Hi), ac_scale(2 * Wi, Wi), (flags & FSB_CONV_RELU) ? 1 : 0);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bilinear_fwd_half launch");
  return FSB_OK;
}

int bilinear_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int ycs, uint32_t flags,
                    cudaStream_t stream) {
  if (C % 8 || xcs % 8 || ycs % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return set_error(FSB_ERR_INVALID, "bilinear: C, strides must be multiples of 8 and pointers 16B aligned");
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo * (C / 8);
  const int64_t blocks = (total + 255) / 256;
  FSB_LAUNCH(bilinear_nhwc_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, 
      N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs, static_cast<__half*>(y), ycs, ac_scale(Hi, Ho),
      ac_scale(Wi, Wo), (flags & FSB_CONV_RELU) ? 1 : 0);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "bilinear launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// final logits upsample: NHWC fp16 low-res (C classes) -> NCHW out.  One thread = 8 consecutive output columns of
// one output row, all classes; per class the warp writes 32 x 16 B = 512 B contiguous.
// ------------------------------------------------------------------------------------------
template <typename TOut, int MAXC>
__global__ void __launch_bounds__(128)
upsample_logits_nchw_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                            TOut* __restrict__ y, float sh, float sw) {
  pdl_launch_dependents();
  pdl_wait();
  const int wvec = (Wo + 7) >> 3;
  const int64_t total = static_cast<int64_t>(N) * Ho * wvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wv = static_cast<int>(gid % wvec);
  const int ho = static_cast<int>((gid / wvec) % Ho);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(wvec) * Ho));
  int h0, h1;
  float lh;
  src_index(ho, sh, Hi, h0, h1, lh);
  const __half* r0 = x + (static_cast<size_t>(n) * Hi + h0) * Wi * xcs;
  const __half* r1 = x + (static_cast<size_t>(n) * Hi + h1) * Wi * xcs;
  int w0[8], w1[8];
  float lw[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) src_index(min(wv * 8 + j, Wo - 1), sw, Wi, w0[j], w1[j], lw[j]);
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  TOut* yrow = y + static_cast<size_t>(n) * C * plane + static_cast<size_t>(ho) * Wo + wv * 8;
  const bool full = (wv * 8 + 8 <= Wo) && ((reinterpret_cast<uintptr_t>(yrow) & (sizeof(TOut) * 8 - 1)) == 0) &&
                    ((plane * sizeof(TOut)) % (sizeof(TOut) * 8) == 0);
  for (int c = 0; c < C; ++c) {
    float o[8];
    int prev = -1;
    float a0 = 0.f, a1 = 0.f;  // row-interpolated values at column w0 / w1 of the current source pair
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (w0[j] != prev) {
        const float t0 = __half2float(r0[static_cast<size_t>(w0[j]) * xcs + c]);
        const float b0 = __half2float(r1[static_cast<size_t>(w0[j]) * xcs + c]);
        const float t1 = __half2float(r0[static_cast<size_t>(w1[j]) * xcs + c]);
        const float b1 = __half2float(r1[static_cast<size_t>(w1[j]) * xcs + c]);
        a0 = (1.f - lh) * t0 + lh * b0;
        a1 = (1.f - lh) * t1 + lh * b1;
        prev = w0[j];
      }
      o[j] = (1.f - lw[j]) * a0 + lw[j] * a1;
    }
    TOut* dst = yrow + static_cast<size_t>(c) * plane;
    if (full) {
      if (sizeof(TOut) == 2) {
        uint4 v;
        v.x = pack_half2(o[0], o[1]);
        v.y = pack_half2(o[2], o[3]);
        v.z = pack_half2(o[4], o[5]);
        v.w = pack_half2(o[6], o[7]);
        *reinterpret_cast<uint4*>(dst) = v;
      } else {
        float4* d4 = reinterpret_cast<float4*>(dst);
        d4[0] = make_float4(o[0], o[1], o[2], o[3]);
        d4[1] = make_float4(o[4], o[5], o[6], o[7]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (wv * 8 + j < Wo) dst[j] = static_cast<TOut>(o[j]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// tiled variant (the x8 / x16 / x32 logits upsample of model_seg.py:359-365): a block owns kRows output rows x kCols
// output columns.  The (few) source rows/columns it touches are staged in shared memory as fp32 [row][class][col];
// per output row the vertical lerp is done once into a [class][col] line, and each thread then produces 8 consecutive
// output columns of one class from <= 3 line entries -> one 16-byte store; a warp writes 512 contiguous bytes.
// HBM traffic = output bytes (+ the tiny source), i.e. the kernel is a pure streaming write.
// ------------------------------------------------------------------------------------------
constexpr int kUpRows = 4;
constexpr int kUpCols = 512;

template <typename TOut>
__global__ void __launch_bounds__(256)
upsample_logits_tiled_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                             TOut* __restrict__ y, float sh, float sw, int max_rows, int max_cols) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_up[];  // [max_rows][C][max_cols] window, then [C][max_cols] line
  const int n = blockIdx.z;
  const int ho0 = blockIdx.y * kUpRows;
  const int wo0 = blockIdx.x * kUpCols;
  const int ho_last = min(ho0 + kUpRows, Ho) - 1;
  const int wo_last = min(wo0 + kUpCols, Wo) - 1;
  int hs0, hs1, ws0, ws1, tmp;
  float ftmp;
  src_index(ho0, sh, Hi, hs0, tmp, ftmp);
  src_index(ho_last, sh, Hi, tmp, hs1, ftmp);
  src_index(wo0, sw, Wi, ws0, tmp, ftmp);
  src_index(wo_last, sw, Wi, tmp, ws1, ftmp);
  const int nrows = hs1 - hs0 + 1;  // <= max_rows by construction on the host
  const int ncols = ws1 - ws0 + 1;  // <= max_cols
  float* win = s_up;
  float* line = s_up + static_cast<size_t>(max_rows) * C * max_cols;
  // ---- stage the source window (NHWC fp16 -> [row][class][col] fp32) ----
  const int cvec = (C + 7) >> 3;
  const int items = nrows * ncols * cvec;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int cv = i % cvec;
    const int col = (i / cvec) % ncols;
    const int row = i / (cvec * ncols);
    const uint4 v = *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * Hi + hs0 + row) * Wi + ws0 + col) * xcs + cv * 8);
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = cv * 8 + j;
      if (c < C) win[(static_cast<size_t>(row) * C + c) * max_cols + col] = __half2float(hv[j]);
    }
  }
  __syncthreads();
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  // thread -> (column vector v, class group cg): the 8 horizontal taps of a thread are the same for every class and
  // every output row, so they are computed once and kept in registers
  constexpr int kVecs = kUpCols / 8;            // 64
  const int v = threadIdx.x % kVecs;
  const int cg = threadIdx.x / kVecs;           // 0..3
  const int cgs = blockDim.x / kVecs;
  const int wo = wo0 + v * 8;
  int wofs[8];
  float lwj[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int w0, w1;
    src_index(min(wo + j, Wo - 1), sw, Wi, w0, w1, lwj[j]);
    wofs[j] = (w0 - ws0) | ((w1 - w0) << 16);
  }
  const bool active = wo <= wo_last;
  for (int r = 0; r <= ho_last - ho0; ++r) {
    const int ho = ho0 + r;
    int h0, h1;
    float lh;
    src_index(ho, sh, Hi, h0, h1, lh);
    const float* r0 = win + static_cast<size_t>(h0 - hs0) * C * max_cols;
    const float* r1 = win + static_cast<size_t>(h1 - hs0) * C * max_cols;
    for (int i = threadIdx.x; i < C * ncols; i += blockDim.x) {
      const int c = i / ncols, col = i % ncols;
      line[c * max_cols + col] = (1.f - lh) * r0[c * max_cols + col] + lh * r1[c * max_cols + col];
    }
    __syncthreads();
    if (active) {
      for (int c = cg; c < C; c += cgs) {
        const float* ln = line + c * max_cols;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int a = wofs[j] & 0xffff;
          const float x0 = ln[a], x1 = ln[a + (wofs[j] >> 16)];
          o[j] = x0 + lwj[j] * (x1 - x0);
        }
        TOut* dst = y + (static_cast<size_t>(n) * C + c) * plane + static_cast<size_t>(ho) * Wo + wo;
        if (wo + 8 <= Wo && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
          if (sizeof(TOut) == 2) {
            uint4 pk;
            pk.x = pack_half2(o[0], o[1]);
            pk.y = pack_half2(o[2], o[3]);
            pk.z = pack_half2(o[4], o[5]);
            pk.w = pack_half2(o[6], o[7]);
            *reinterpret_cast<uint4*>(dst) = pk;
          } else {
            float4* d4 = reinterpret_cast<float4*>(dst);
            d4[0] = make_float4(o[0], o[1], o[2], o[3]);
            d4[1] = make_float4(o[4], o[5], o[6], o[7]);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (wo + j < Wo) dst[j] = static_cast<TOut>(o[j]);
        }
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// EXPERIMENTAL (FSB_UPSAMPLE_V2=1, default off): same tiling idea without the per-row barriers.
// The tiled kernel above synchronises twice per output row (build the vertically interpolated line in smem, consume it),
// i.e. 8 barriers for 78 KB of stores -- it reaches 2.4 TB/s of the 6.6 TB/s the 80 MB logits write could stream at.
// For upsampling factors >= 8 the 8 consecutive output columns of a thread read at most 3 consecutive source columns, so
// a thread can interpolate them vertically in registers (6 smem loads per (row, class)) and needs no shared line at all:
// one barrier per block (after staging the source window), 8 output rows per block.
// Arithmetic is expression-for-expression the one of the kernel above: (1 - lh) * top + lh * bottom, then x0 + lw * (x1 - x0).
// ------------------------------------------------------------------------------------------
constexpr int kUp2Rows = 8;

template <typename TOut>
__global__ void __launch_bounds__(256)
upsample_logits_rows_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                            TOut* __restrict__ y, float sh, float sw, int max_rows, int max_cols) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float s_up[];  // [max_rows][C][max_cols] source window as fp32
  const int n = blockIdx.z;
  const int ho0 = blockIdx.y * kUp2Rows;
  const int wo0 = blockIdx.x * kUpCols;
  const int ho_last = min(ho0 + kUp2Rows, Ho) - 1;
  const int wo_last = min(wo0 + kUpCols, Wo) - 1;
  int hs0, hs1, ws0, ws1, tmp;
  float ftmp;
  src_index(ho0, sh, Hi, hs0, tmp, ftmp);
  src_index(ho_last, sh, Hi, tmp, hs1, ftmp);
  src_index(wo0, sw, Wi, ws0, tmp, ftmp);
  src_index(wo_last, sw, Wi, tmp, ws1, ftmp);
  const int nrows = hs1 - hs0 + 1;  // <= max_rows by construction on the host
  const int ncols = ws1 - ws0 + 1;  // <= max_cols
  float* win = s_up;
  const int cvec = (C + 7) >> 3;
  const int items = nrows * ncols * cvec;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int cv = i % cvec;
    const int col = (i / cvec) % ncols;
    const int row = i / (cvec * ncols);
    const uint4 v = *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * Hi + hs0 + row) * Wi + ws0 + col) * xcs + cv * 8);
    const __half* hv = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = cv * 8 + j;
      if (c < C) win[(static_cast<size_t>(row) * C + c) * max_cols + col] = __half2float(hv[j]);
    }
  }
  __syncthreads();
  constexpr int kVecs = kUpCols / 8;  // 64 column vectors per block row
  const int v = threadIdx.x % kVecs;
  const int cg = threadIdx.x / kVecs;  // class group 0..3
  const int cgs = blockDim.x / kVecs;
  const int wo = wo0 + v * 8;
  if (wo > wo_last) return;  // no barrier below this point
  // horizontal taps of the 8 columns, relative to the first source column this thread touches (span <= 3 columns)
  int rel0[8], rel1[8];
  float lwj[8];
  int base = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int w0, w1;
    src_index(min(wo + j, Wo - 1), sw, Wi, w0, w1, lwj[j]);
    if (j == 0) base = w0;
    rel0[j] = w0 - base;
    rel1[j] = w1 - base;
  }
  const int col0 = base - ws0;
  const int k1 = min(col0 + 1, ncols - 1) - col0;  // clamp the 2nd / 3rd column into the staged window
  const int k2 = min(col0 + 2, ncols - 1) - col0;
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  for (int ho = ho0; ho <= ho_last; ++ho) {
    int h0, h1;
    float lh;
    src_index(ho, sh, Hi, h0, h1, lh);
    const float* r0 = win + static_cast<size_t>(h0 - hs0) * C * max_cols + col0;
    const float* r1 = win + static_cast<size_t>(h1 - hs0) * C * max_cols + col0;
    for (int c = cg; c < C; c += cgs) {
      const float* p0 = r0 + c * max_cols;
      const float* p1 = r1 + c * max_cols;
      const float s0 = (1.f - lh) * p0[0] + lh * p1[0];
      const float s1 = (1.f - lh) * p0[k1] + lh * p1[k1];
      const float s2 = (1.f - lh) * p0[k2] + lh * p1[k2];
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float x0 = rel0[j] == 0 ? s0 : (rel0[j] == 1 ? s1 : s2);
        const float x1 = rel1[j] == 0 ? s0 : (rel1[j] == 1 ? s1 : s2);
        o[j] = x0 + lwj[j] * (x1 - x0);
      }
      TOut* dst = y + (static_cast<size_t>(n) * C + c) * plane + static_cast<size_t>(ho) * Wo + wo;
      if (wo + 8 <= Wo && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        if (sizeof(TOut) == 2) {
          uint4 pk;
          pk.x = pack_half2(o[0], o[1]);
          pk.y = pack_half2(o[2], o[3]);
          pk.z = pack_half2(o[4], o[5]);
          pk.w = pack_half2(o[6], o[7]);
          *reinterpret_cast<uint4*>(dst) = pk;
        } else {
          float4* d4 = reinterpret_cast<float4*>(dst);
          d4[0] = make_float4(o[0], o[1], o[2], o[3]);
          d4[1] = make_float4(o[4], o[5], o[6], o[7]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (wo + j < Wo) dst[j] = static_cast<TOut>(o[j]);
      }
    }
  }
}

int upsample_logits_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int out_dtype,
                           cudaStream_t stream) {
  // tiled path: upsampling only, source window must fit in shared memory, 16-byte addressable source pixels
  const float sh = ac_scale(Hi, Ho), sw = ac_scale(Wi, Wo);
  const bool v2_on = opt(OPT_UPSAMPLE_V2) == 1;
  // v2 needs the 8 columns of a thread to span <= 3 source columns: 7 * sw + 1 < 2  <=>  upsampling factor > 7
  if (v2_on && sh <= 1.f && sw * 7.f < 0.999f && xcs % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && xcs >= (C + 7) / 8 * 8) {
    const int max_rows = static_cast<int>(sh * (kUp2Rows - 1)) + 3;
    const int max_cols = static_cast<int>(sw * (kUpCols - 1)) + 3;
    const size_t smem = static_cast<size_t>(max_rows) * C * max_cols * sizeof(float);
    if (smem <= 48 * 1024) {
      dim3 grid((Wo + kUpCols - 1) / kUpCols, (Ho + kUp2Rows - 1) / kUp2Rows, N);
      if (out_dtype == 0)
        FSB_LAUNCH(upsample_logits_rows_kernel<__half>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo,
                   static_cast<const __half*>(x), xcs, static_cast<__half*>(y), sh, sw, max_rows, max_cols);
      else
        FSB_LAUNCH(upsample_logits_rows_kernel<float>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo,
                   static_cast<const __half*>(x), xcs, static_cast<float*>(y), sh, sw, max_rows, max_cols);
      cudaError_t e3 = last_launch_error();
      if (e3 != cudaSuccess) return set_cuda_error(e3, "upsample_logits_rows launch");
      return FSB_OK;
    }
  }
  if (sh <= 1.f && sw <= 1.f && xcs % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && xcs >= (C + 7) / 8 * 8) {
    const int max_rows = static_cast<int>(sh * (kUpRows - 1)) + 3;
    const int max_cols = static_cast<int>(sw * (kUpCols - 1)) + 3;
    const size_t smem = (static_cast<size_t>(max_rows) * C * max_cols + static_cast<size_t>(C) * max_cols) * sizeof(float);
    if (smem <= 48 * 1024) {
      dim3 grid((Wo + kUpCols - 1) / kUpCols, (Ho + kUpRows - 1) / kUpRows, N);
      if (out_dtype == 0)
        FSB_LAUNCH(upsample_logits_tiled_kernel<__half>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo,
                   static_cast<const __half*>(x), xcs, static_cast<__half*>(y), sh, sw, max_rows, max_cols);
      else
        FSB_LAUNCH(upsample_logits_tiled_kernel<float>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo,
                   static_cast<const __half*>(x), xcs, static_cast<float*>(y), sh, sw, max_rows, max_cols);
      cudaError_t e2 = last_launch_error();
      if (e2 != cudaSuccess) return set_cuda_error(e2, "upsample_logits_tiled launch");
      return FSB_OK;
    }
  }
  const int64_t total = static_cast<int64_t>(N) * Ho * ((Wo + 7) / 8);
  const int64_t blocks = (total + 127) / 128;
  if (out_dtype == 0)
    FSB_LAUNCH(upsample_logits_nchw_kernel<__half, 32>, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, stream, 
        N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs, static_cast<__half*>(y), ac_scale(Hi, Ho), ac_scale(Wi, Wo));
  else
    FSB_LAUNCH(upsample_logits_nchw_kernel<float, 32>, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, stream, 
        N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs, static_cast<float*>(y), ac_scale(Hi, Ho), ac_scale(Wi, Wo));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_logits launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// fused upsample + argmax.  One work item = 4 consecutive output columns wv*4.. of output row ho of image n: the argmax over
// the C classes of the bilinear (align_corners) value at each.  Columns past Wo repeat the last column.  Both the label kernel
// and the confusion kernel below call this, so their labels are the same bits.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void upsample_argmax4(int C, int Hi, int Wi, int Wo, const __half* __restrict__ x, int xcs, float sh,
                                                 float sw, int n, int ho, int wv, int (&arg)[4]) {
  int h0, h1;
  float lh;
  src_index(ho, sh, Hi, h0, h1, lh);
  const __half* r0 = x + (static_cast<size_t>(n) * Hi + h0) * Wi * xcs;
  const __half* r1 = x + (static_cast<size_t>(n) * Hi + h1) * Wi * xcs;
  int w0[4], w1[4];
  float lw[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) src_index(min(wv * 4 + j, Wo - 1), sw, Wi, w0[j], w1[j], lw[j]);
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 4; ++j) arg[j] = 0;
  for (int c = 0; c < C; ++c) {
    int prev = -1;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (w0[j] != prev) {
        const float t0 = __half2float(r0[static_cast<size_t>(w0[j]) * xcs + c]);
        const float b0 = __half2float(r1[static_cast<size_t>(w0[j]) * xcs + c]);
        const float t1 = __half2float(r0[static_cast<size_t>(w1[j]) * xcs + c]);
        const float b1 = __half2float(r1[static_cast<size_t>(w1[j]) * xcs + c]);
        a0 = (1.f - lh) * t0 + lh * b0;
        a1 = (1.f - lh) * t1 + lh * b1;
        prev = w0[j];
      }
      const float v = (1.f - lw[j]) * a0 + lw[j] * a1;
      if (v > best[j]) {  // strict '>' => first maximum wins, like torch/np argmax
        best[j] = v;
        arg[j] = c;
      }
    }
  }
}

// -> uint8 labels.  One thread = 4 consecutive output columns (one 32-bit store).
__global__ void __launch_bounds__(128)
upsample_argmax_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                       uint8_t* __restrict__ labels, float sh, float sw) {
  pdl_launch_dependents();
  pdl_wait();
  const int wvec = (Wo + 3) >> 2;
  const int64_t total = static_cast<int64_t>(N) * Ho * wvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wv = static_cast<int>(gid % wvec);
  const int ho = static_cast<int>((gid / wvec) % Ho);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(wvec) * Ho));
  int arg[4];
  upsample_argmax4(C, Hi, Wi, Wo, x, xcs, sh, sw, n, ho, wv, arg);
  uint8_t* dst = labels + (static_cast<size_t>(n) * Ho + ho) * Wo + wv * 4;
  if (wv * 4 + 4 <= Wo && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
    *reinterpret_cast<uint32_t*>(dst) = static_cast<uint32_t>(arg[0]) | (static_cast<uint32_t>(arg[1]) << 8) |
                                        (static_cast<uint32_t>(arg[2]) << 16) | (static_cast<uint32_t>(arg[3]) << 24);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (wv * 4 + j < Wo) dst[j] = static_cast<uint8_t>(arg[j]);
  }
}

int upsample_argmax_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, uint8_t* labels,
                           cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(N) * Ho * ((Wo + 3) / 4);
  const int64_t blocks = (total + 127) / 128;
  FSB_LAUNCH(upsample_argmax_kernel, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x),
                                                                         xcs, labels, ac_scale(Hi, Ho), ac_scale(Wi, Wo));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_argmax launch");
  return FSB_OK;
}

// upsample + argmax + confusion matrix (tools/seg_opr/metric.py:7-15 hist_info) without writing the label map: the labels of
// upsample_argmax4 go straight into a per-CTA shared-memory histogram, flushed with integer atomics (exact, order-independent).
// Counting rule of confusion_kernel (conv_direct.cu): gt outside [0, n_cl) is ignored, hist[n_cl * gt + pred] += 1,
// labeled += 1, correct += (pred == gt).  out: int64 [n_cl * n_cl + 2], accumulated into.  Grid-stride over the work items.
template <typename TGt>
__global__ void __launch_bounds__(256)
upsample_argmax_confusion_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                                 const TGt* __restrict__ gt, float sh, float sw, unsigned long long* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ unsigned int s_cm[];  // C * C + 2
  const int cells = C * C + 2;
  for (int i = threadIdx.x; i < cells; i += blockDim.x) s_cm[i] = 0;
  __syncthreads();
  const int wvec = (Wo + 3) >> 2;
  const int64_t total = static_cast<int64_t>(N) * Ho * wvec;
  unsigned int labeled = 0, correct = 0;
  for (int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; gid < total;
       gid += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int wv = static_cast<int>(gid % wvec);
    const int ho = static_cast<int>((gid / wvec) % Ho);
    const int n = static_cast<int>(gid / (static_cast<int64_t>(wvec) * Ho));
    int arg[4];
    upsample_argmax4(C, Hi, Wi, Wo, x, xcs, sh, sw, n, ho, wv, arg);
    const TGt* g = gt + (static_cast<size_t>(n) * Ho + ho) * Wo + wv * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (wv * 4 + j >= Wo) break;
      const long long t = static_cast<long long>(g[j]);
      if (t < 0 || t >= C) continue;
      atomicAdd(&s_cm[t * C + arg[j]], 1u);
      ++labeled;
      correct += arg[j] == t ? 1u : 0u;
    }
  }
  if (labeled) atomicAdd(&s_cm[C * C], labeled);
  if (correct) atomicAdd(&s_cm[C * C + 1], correct);
  __syncthreads();
  for (int i = threadIdx.x; i < cells; i += blockDim.x)
    if (s_cm[i]) atomicAdd(&out[i], static_cast<unsigned long long>(s_cm[i]));
}

int upsample_argmax_confusion_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const void* gt, int gt_bytes,
                                     long long* out, cudaStream_t stream) {
  if (C < 1 || C > 64) return set_error(FSB_ERR_INVALID, "upsample_argmax_confusion: 1 <= n_cl <= 64");
  const int64_t total = static_cast<int64_t>(N) * Ho * ((Wo + 3) / 4);
  // at most 4 CTAs per SM (2 are resident at this kernel's register count): large maps run several work items per thread, which
  // amortises the histogram's clear and flush
  int64_t blocks = (total + 255) / 256;
  if (blocks > static_cast<int64_t>(sm_count()) * 4) blocks = static_cast<int64_t>(sm_count()) * 4;
  if (blocks < 1) blocks = 1;
  const size_t smem = static_cast<size_t>(C * C + 2) * sizeof(unsigned int);
  const __half* xh = static_cast<const __half*>(x);
  const float sh = ac_scale(Hi, Ho), sw = ac_scale(Wi, Wo);
  unsigned long long* o = reinterpret_cast<unsigned long long*>(out);
  const dim3 grid(static_cast<unsigned>(blocks));
  if (gt_bytes == 1)
    FSB_LAUNCH(upsample_argmax_confusion_kernel<uint8_t>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo, xh, xcs,
               static_cast<const uint8_t*>(gt), sh, sw, o);
  else if (gt_bytes == 4)
    FSB_LAUNCH(upsample_argmax_confusion_kernel<int32_t>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo, xh, xcs,
               static_cast<const int32_t*>(gt), sh, sw, o);
  else if (gt_bytes == 8)
    FSB_LAUNCH(upsample_argmax_confusion_kernel<long long>, grid, dim3(256), smem, stream, N, C, Hi, Wi, Ho, Wo, xh, xcs,
               static_cast<const long long*>(gt), sh, sw, o);
  else
    return set_error(FSB_ERR_INVALID, "upsample_argmax_confusion: ground truth must be uint8, int32 or int64");
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_argmax_confusion launch");
  return FSB_OK;
}

// upsample + argmax -> the two uint8 images the reference's test-set writer saves (train/test.py:49-69,
// tools/utils/visualize.py:6-21): ids[p] = lut[label] and viz[p] = the BGR bytes of palette[label] (B, G, R, use_image), or of the
// RGB image pixel reversed where use_image is set.  Labels are upsample_argmax4's, so they are upsample_argmax_kernel's bits.  One
// thread = 4 consecutive output columns: one 32-bit store of ids, three of viz, where the row allows.  The tables live in shared
// memory (C <= 255 entries).
__global__ void __launch_bounds__(128)
upsample_argmax_map_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs, float sh, float sw,
                           const uint8_t* __restrict__ lut, uint8_t* __restrict__ ids, const uint8_t* __restrict__ palette,
                           const uint8_t* __restrict__ image, uint8_t* __restrict__ viz) {
  __shared__ uint8_t s_lut[256];
  __shared__ uchar4 s_pal[256];
  pdl_launch_dependents();
  pdl_wait();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    s_lut[i] = lut ? lut[i] : static_cast<uint8_t>(i);
    if (palette) s_pal[i] = make_uchar4(palette[4 * i], palette[4 * i + 1], palette[4 * i + 2], palette[4 * i + 3]);
  }
  __syncthreads();
  const int wvec = (Wo + 3) >> 2;
  const int64_t total = static_cast<int64_t>(N) * Ho * wvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wv = static_cast<int>(gid % wvec);
  const int ho = static_cast<int>((gid / wvec) % Ho);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(wvec) * Ho));
  int arg[4];
  upsample_argmax4(C, Hi, Wi, Wo, x, xcs, sh, sw, n, ho, wv, arg);
  const size_t pix = (static_cast<size_t>(n) * Ho + ho) * Wo + wv * 4;
  const bool full = wv * 4 + 4 <= Wo;
  if (ids) {
    uint8_t* dst = ids + pix;
    if (full && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
      *reinterpret_cast<uint32_t*>(dst) = static_cast<uint32_t>(s_lut[arg[0]]) | (static_cast<uint32_t>(s_lut[arg[1]]) << 8) |
                                          (static_cast<uint32_t>(s_lut[arg[2]]) << 16) | (static_cast<uint32_t>(s_lut[arg[3]]) << 24);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (wv * 4 + j < Wo) dst[j] = s_lut[arg[j]];
    }
  }
  if (viz) {
    uint8_t b[12];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uchar4 c = s_pal[arg[j]];
      if (c.w && wv * 4 + j < Wo) {   // set_img_color leaves the pixel alone: the image's RGB, written reversed
        const uint8_t* s = image + (pix + j) * 3;
        b[3 * j] = s[2];
        b[3 * j + 1] = s[1];
        b[3 * j + 2] = s[0];
      } else {
        b[3 * j] = c.x;
        b[3 * j + 1] = c.y;
        b[3 * j + 2] = c.z;
      }
    }
    uint8_t* dst = viz + pix * 3;
    if (full && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        reinterpret_cast<uint32_t*>(dst)[k] = static_cast<uint32_t>(b[4 * k]) | (static_cast<uint32_t>(b[4 * k + 1]) << 8) |
                                              (static_cast<uint32_t>(b[4 * k + 2]) << 16) | (static_cast<uint32_t>(b[4 * k + 3]) << 24);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (wv * 4 + j < Wo) {
          dst[3 * j] = b[3 * j];
          dst[3 * j + 1] = b[3 * j + 1];
          dst[3 * j + 2] = b[3 * j + 2];
        }
    }
  }
}

int upsample_argmax_map_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, const uint8_t* lut, uint8_t* ids,
                               const uint8_t* palette, const uint8_t* image, uint8_t* viz, cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(N) * Ho * ((Wo + 3) / 4);
  const int64_t blocks = (total + 127) / 128;
  FSB_LAUNCH(upsample_argmax_map_kernel, dim3(static_cast<unsigned>(blocks)), dim3(128), 0, stream, N, C, Hi, Wi, Ho, Wo,
             static_cast<const __half*>(x), xcs, ac_scale(Hi, Ho), ac_scale(Wi, Wo), lut, ids, palette, image, viz);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_argmax_map launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// nearest (latency/ deployment network): torch's legacy 'nearest' index rule, scale and product in fp32 -- for sizes like
// 5 -> 2 or 2 -> 5 the float rounding IS the behaviour, so no integer shortcut.  Pure copies: outputs are bit-exact.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int nearest_src(int dst, int n_in, int n_out) {
  const float scale = static_cast<float>(n_in) / static_cast<float>(n_out);
  const int s = static_cast<int>(floorf(static_cast<float>(dst) * scale));
  return s < n_in - 1 ? s : n_in - 1;
}

// one thread = one output pixel x 8 channels
__global__ void __launch_bounds__(256)
nearest_nhwc_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs, __half* __restrict__ y,
                    int ycs) {
  pdl_launch_dependents();
  pdl_wait();
  const int cvec = C >> 3;
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo * cvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int cv = static_cast<int>(gid % cvec);
  const int64_t pix = gid / cvec;
  const int wo = static_cast<int>(pix % Wo);
  const int ho = static_cast<int>((pix / Wo) % Ho);
  const int n = static_cast<int>(pix / (static_cast<int64_t>(Wo) * Ho));
  const int hs = nearest_src(ho, Hi, Ho), ws = nearest_src(wo, Wi, Wo);
  *reinterpret_cast<uint4*>(y + static_cast<size_t>(pix) * ycs + cv * 8) =
      *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * Hi + hs) * Wi + ws) * xcs + cv * 8);
}

int nearest_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int ycs, cudaStream_t stream) {
  if (C % 8 || xcs % 8 || ycs % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return set_error(FSB_ERR_INVALID, "nearest: C, strides must be multiples of 8 and pointers 16B aligned");
  const int64_t total = static_cast<int64_t>(N) * Ho * Wo * (C / 8);
  FSB_LAUNCH(nearest_nhwc_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo,
             static_cast<const __half*>(x), xcs, static_cast<__half*>(y), ycs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "nearest launch");
  return FSB_OK;
}

// final nearest logits upsample: NHWC fp16 -> NCHW.  One thread = 8 consecutive output columns of one output row, all classes;
// per class it stores one 16-byte vector (fp16) or two (fp32), so a warp writes 512 / 1024 contiguous bytes.  The kernel is
// bound by these writes; the source values (one or two pixels per thread at x8) come from L1.
template <typename TOut>
__global__ void __launch_bounds__(128)
upsample_logits_nearest_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                               TOut* __restrict__ y) {
  pdl_launch_dependents();
  pdl_wait();
  const int wvec = (Wo + 7) >> 3;
  const int64_t total = static_cast<int64_t>(N) * Ho * wvec;
  const int64_t gid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (gid >= total) return;
  const int wv = static_cast<int>(gid % wvec);
  const int ho = static_cast<int>((gid / wvec) % Ho);
  const int n = static_cast<int>(gid / (static_cast<int64_t>(wvec) * Ho));
  const __half* row = x + (static_cast<size_t>(n) * Hi + nearest_src(ho, Hi, Ho)) * Wi * xcs;
  int ws[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) ws[j] = nearest_src(min(wv * 8 + j, Wo - 1), Wi, Wo);
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  TOut* yrow = y + static_cast<size_t>(n) * C * plane + static_cast<size_t>(ho) * Wo + wv * 8;
  const bool full = (wv * 8 + 8 <= Wo) && ((reinterpret_cast<uintptr_t>(yrow) & 15) == 0) && ((plane * sizeof(TOut)) % 16 == 0);
  for (int c = 0; c < C; ++c) {
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o[j] = (j > 0 && ws[j] == ws[j - 1]) ? o[j - 1] : __half2float(row[static_cast<size_t>(ws[j]) * xcs + c]);
    TOut* dst = yrow + static_cast<size_t>(c) * plane;
    if (full) {
      if (sizeof(TOut) == 2) {
        uint4 v;
        v.x = pack_half2(o[0], o[1]);
        v.y = pack_half2(o[2], o[3]);
        v.z = pack_half2(o[4], o[5]);
        v.w = pack_half2(o[6], o[7]);
        *reinterpret_cast<uint4*>(dst) = v;
      } else {
        float4* d4 = reinterpret_cast<float4*>(dst);
        d4[0] = make_float4(o[0], o[1], o[2], o[3]);
        d4[1] = make_float4(o[4], o[5], o[6], o[7]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (wv * 8 + j < Wo) dst[j] = static_cast<TOut>(o[j]);
    }
  }
}

int upsample_logits_nearest_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, void* y, int out_dtype,
                                   cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(N) * Ho * ((Wo + 7) / 8);
  const dim3 grid(static_cast<unsigned>((total + 127) / 128));
  if (out_dtype == 0)
    FSB_LAUNCH(upsample_logits_nearest_kernel<__half>, grid, dim3(128), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x),
               xcs, static_cast<__half*>(y));
  else
    FSB_LAUNCH(upsample_logits_nearest_kernel<float>, grid, dim3(128), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x),
               xcs, static_cast<float*>(y));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_logits_nearest launch");
  return FSB_OK;
}

// nearest upsample + argmax -> uint8 labels.  A block owns kLabRows x kLabCols output pixels.  The nearest index is monotone,
// so the source rows (columns) the tile touches are a run src0..src_last when upsampling (in <= out: consecutive outputs
// differ by 0 or 1) and one distinct source per output when downsampling (in > out: they differ by >= 1).  The block takes
// the argmax once per distinct source pixel into shared memory, then every thread stores 8 replicated labels (one 8-byte store).
// Arithmetic: strict '>' over the fp16 values widened to fp32, i.e. the argmax of the logits kernel's output (which holds the
// same values), first maximum winning.
constexpr int kLabRows = 8;
constexpr int kLabCols = 256;

__global__ void __launch_bounds__(256)
upsample_argmax_nearest_kernel(int N, int C, int Hi, int Wi, int Ho, int Wo, const __half* __restrict__ x, int xcs,
                               uint8_t* __restrict__ labels) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int s_hsrc[kLabRows], s_wsrc[kLabCols];      // source row / column of each distinct slot
  __shared__ int s_hslot[kLabRows], s_wslot[kLabCols];    // slot of each output row / column of the tile
  __shared__ uint8_t s_lab[kLabRows][kLabCols];
  const int n = blockIdx.z;
  const int ho0 = blockIdx.y * kLabRows, wo0 = blockIdx.x * kLabCols;
  const int nrows = min(kLabRows, Ho - ho0), ncols = min(kLabCols, Wo - wo0);
  const int t = threadIdx.x;
  const bool up_h = Hi <= Ho, up_w = Wi <= Wo;
  const int hs0 = nearest_src(ho0, Hi, Ho), ws0 = nearest_src(wo0, Wi, Wo);
  if (t < ncols) {
    const int ws = nearest_src(wo0 + t, Wi, Wo);
    const int slot = up_w ? ws - ws0 : t;
    s_wslot[t] = slot;
    s_wsrc[slot] = ws;  // upsampling: threads of one slot write the same value
  }
  if (t < nrows) {
    const int hs = nearest_src(ho0 + t, Hi, Ho);
    const int slot = up_h ? hs - hs0 : t;
    s_hslot[t] = slot;
    s_hsrc[slot] = hs;
  }
  __syncthreads();
  const int srows = up_h ? nearest_src(ho0 + nrows - 1, Hi, Ho) - hs0 + 1 : nrows;
  const int scols = up_w ? nearest_src(wo0 + ncols - 1, Wi, Wo) - ws0 + 1 : ncols;
  for (int i = t; i < srows * scols; i += blockDim.x) {
    const int r = i / scols, c = i - r * scols;
    const __half* px = x + ((static_cast<size_t>(n) * Hi + s_hsrc[r]) * Wi + s_wsrc[c]) * xcs;
    float best = -INFINITY;
    int arg = 0;
    for (int k = 0; k < C; ++k) {
      const float v = __half2float(px[k]);
      if (v > best) {
        best = v;
        arg = k;
      }
    }
    s_lab[r][c] = static_cast<uint8_t>(arg);
  }
  __syncthreads();
  const int r = t / (kLabCols / 8);
  const int c0 = (t % (kLabCols / 8)) * 8;
  if (r >= nrows || c0 >= ncols) return;
  const uint8_t* lab = s_lab[s_hslot[r]];
  uint8_t* dst = labels + (static_cast<size_t>(n) * Ho + ho0 + r) * Wo + wo0 + c0;
  if (c0 + 8 <= ncols && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo |= static_cast<uint32_t>(lab[s_wslot[c0 + j]]) << (8 * j);
      hi |= static_cast<uint32_t>(lab[s_wslot[c0 + 4 + j]]) << (8 * j);
    }
    *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
  } else {
    for (int j = 0; j < 8 && c0 + j < ncols; ++j) dst[j] = lab[s_wslot[c0 + j]];
  }
}

int upsample_argmax_nearest_launch(int N, int C, int Hi, int Wi, int Ho, int Wo, const void* x, int xcs, uint8_t* labels,
                                   cudaStream_t stream) {
  const dim3 grid((Wo + kLabCols - 1) / kLabCols, (Ho + kLabRows - 1) / kLabRows, N);
  FSB_LAUNCH(upsample_argmax_nearest_kernel, grid, dim3(256), 0, stream, N, C, Hi, Wi, Ho, Wo, static_cast<const __half*>(x), xcs,
             labels);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "upsample_argmax_nearest launch");
  return FSB_OK;
}

// ------------------------------------------------------------------------------------------
// layout plumbing
// ------------------------------------------------------------------------------------------
template <typename TIn>
__global__ void nchw_to_nhwc_kernel(int N, int C, int H, int W, const TIn* __restrict__ x, __half* __restrict__ y, int ycs) {
  pdl_launch_dependents();
  pdl_wait();
  // tile transpose through shared memory: 32 pixels x 32 channels
  __shared__ float tile[32][33];
  const int64_t HW = static_cast<int64_t>(H) * W;
  const int n = blockIdx.z;
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const int64_t pp = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && pp < HW) ? static_cast<float>(x[(static_cast<int64_t>(n) * C + c) * HW + pp]) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t pp = p0 + i;
    const int c = c0 + threadIdx.x;
    if (pp < HW && c < C) y[(static_cast<int64_t>(n) * HW + pp) * ycs + c] = __float2half_rn(tile[threadIdx.x][i]);
  }
}
template <typename TOut>
__global__ void nhwc_to_nchw_kernel(int N, int C, int H, int W, const __half* __restrict__ x, int xcs, TOut* __restrict__ y) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float tile[32][33];
  const int64_t HW = static_cast<int64_t>(H) * W;
  const int n = blockIdx.z;
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t pp = p0 + i;
    const int c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (pp < HW && c < C) ? __half2float(x[(static_cast<int64_t>(n) * HW + pp) * xcs + c]) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const int64_t pp = p0 + threadIdx.x;
    if (c < C && pp < HW) y[(static_cast<int64_t>(n) * C + c) * HW + pp] = static_cast<TOut>(tile[threadIdx.x][i]);
  }
}

int nchw_to_nhwc_launch(int N, int C, int H, int W, const void* x, int x_is_f32, void* y, int ycs, cudaStream_t stream) {
  const int64_t HW = static_cast<int64_t>(H) * W;
  dim3 block(32, 8), grid(static_cast<unsigned>((HW + 31) / 32), (C + 31) / 32, N);
  if (x_is_f32)
    FSB_LAUNCH(nchw_to_nhwc_kernel<float>, dim3(grid), dim3(block), 0, stream, N, C, H, W, static_cast<const float*>(x), static_cast<__half*>(y), ycs);
  else
    FSB_LAUNCH(nchw_to_nhwc_kernel<__half>, dim3(grid), dim3(block), 0, stream, N, C, H, W, static_cast<const __half*>(x), static_cast<__half*>(y), ycs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "nchw_to_nhwc launch");
  return FSB_OK;
}
int nhwc_to_nchw_launch(int N, int C, int H, int W, const void* x, int xcs, void* y, int y_is_f32, cudaStream_t stream) {
  const int64_t HW = static_cast<int64_t>(H) * W;
  dim3 block(32, 8), grid(static_cast<unsigned>((HW + 31) / 32), (C + 31) / 32, N);
  if (y_is_f32)
    FSB_LAUNCH(nhwc_to_nchw_kernel<float>, dim3(grid), dim3(block), 0, stream, N, C, H, W, static_cast<const __half*>(x), xcs, static_cast<float*>(y));
  else
    FSB_LAUNCH(nhwc_to_nchw_kernel<__half>, dim3(grid), dim3(block), 0, stream, N, C, H, W, static_cast<const __half*>(x), xcs, static_cast<__half*>(y));
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "nhwc_to_nchw launch");
  return FSB_OK;
}

__global__ void copy_channels_kernel(int64_t pixels, int cvec, const __half* __restrict__ x, int xcs, __half* __restrict__ y,
                                     int ycs) {
  pdl_launch_dependents();
  pdl_wait();
  const int64_t total = pixels * cvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(i % cvec);
    const int64_t pix = i / cvec;
    *reinterpret_cast<uint4*>(y + pix * ycs + cv * 8) = *reinterpret_cast<const uint4*>(x + pix * xcs + cv * 8);
  }
}
int copy_channels_launch(int64_t pixels, int C, const void* x, int xcs, void* y, int ycs, cudaStream_t stream) {
  if (C % 8 || xcs % 8 || ycs % 8 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15))
    return set_error(FSB_ERR_INVALID, "copy_channels: C, strides must be multiples of 8 and pointers 16B aligned");
  const int64_t total = pixels * (C / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  FSB_LAUNCH(copy_channels_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream, pixels, C / 8, static_cast<const __half*>(x), xcs,
                                                                        static_cast<__half*>(y), ycs);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "copy_channels launch");
  return FSB_OK;
}

}  // namespace fsb
