// trainpre.cu -- K15: the drivers' training augmentation (TrainPre, train/dataloader.py:14-31, same in search/dataloader.py) on the
// device.  One launch per batch; every output element is computed independently from the uint8 source, so the kernel is a gather
// that is bound by memory latency.
//
// The arithmetic reproduces OpenCV's cv::resize for 8-bit images exactly (checked against opencv-python 4.13.0 on x86-64):
//   INTER_LINEAR (resizeGeneric_ with HResizeLinear<uchar, int, short, 2048> and VResizeLinear's vector form):
//     scale = 1.0 / ((double)dst / src);  f = (float)((d + 0.5) * scale - 0.5);  s = floor(f);  f -= s;
//     coefficients (saturate_cast<short>((1 - f) * 2048), saturate_cast<short>(f * 2048)), round half to even;
//     columns: s < 0 -> (s, f) = (0, 0);  s >= src - 1 -> (s, f) = (src - 1, 0);  taps s and min(s + 1, src - 1);
//     rows: the coefficients are NOT clamped, only the two row indices s and s + 1 are clamped to [0, src - 1];
//     horizontal pass in int32: S = p[s] * a0 + p[s + 1] * a1;
//     vertical pass: ((((S0 >> 4) * b0) >> 16) + (((S1 >> 4) * b1) >> 16) + 2) >> 2, saturated to [0, 255].
//   INTER_NEAREST (resizeNN):  s = min(floor(d * (1.0 / ((double)dst / src))), src - 1)  per axis, in double.
// The double expressions use explicitly rounded intrinsics so that nvcc cannot contract them into FMAs that OpenCV's build does
// not use.
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

namespace {

constexpr int kGeom = 8;  // H, W, mirror, sh, sw, pos_h, pos_w, pixel offset of the image in the source buffers

// cv::resize INTER_LINEAR coefficient of destination index d (dst = scaled size, src = source size)
__device__ __forceinline__ void linear_coef(int d, int src, int dst, bool clamp, int& s, int& a0, int& a1) {
  const double scale = __drcp_rn(__ddiv_rn(static_cast<double>(dst), static_cast<double>(src)));
  float f = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), scale), -0.5));
  s = static_cast<int>(floorf(f));
  f = __fsub_rn(f, static_cast<float>(s));
  if (clamp) {
    if (s < 0) s = 0, f = 0.f;
    if (s >= src - 1) s = src - 1, f = 0.f;
  }
  a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  a1 = __float2int_rn(__fmul_rn(f, 2048.f));
}

// cv::resize INTER_NEAREST source index of destination index d
__device__ __forceinline__ int nearest_src(int d, int src, int dst) {
  const double ifx = __drcp_rn(__ddiv_rn(static_cast<double>(dst), static_cast<double>(src)));
  const int s = static_cast<int>(floor(__dmul_rn(static_cast<double>(d), ifx)));
  return s < src - 1 ? s : src - 1;
}

// pad_image_to_shape (tools/utils/img_utils.py:60-74) after the crop of random_crop_pad_to_shape (:24-39): crop index c of an
// axis whose scaled size is `scaled` and crop start `pos` -> scaled-frame index, or -1 in the padding
__device__ __forceinline__ int crop_src(int c, int crop, int scaled, int pos) {
  const int kept = min(crop, scaled - pos);
  const int lo = (crop - kept) / 2;
  const int k = c - lo;
  return (k >= 0 && k < kept) ? pos + k : -1;
}

// grid (ceil(crop_w / 128), crop_h, N); thread (x, y) of image n writes the 3 image channels of crop pixel (y, x) and, when
// (y, x) lies inside the label_h x label_w map, that label
__global__ void __launch_bounds__(128) train_pre_kernel(int crop_h, int crop_w, int label_h, int label_w,
                                                        const uint8_t* __restrict__ img, const uint8_t* __restrict__ gt,
                                                        const int32_t* __restrict__ geom, const float* __restrict__ lut,
                                                        float* __restrict__ out_img, long long* __restrict__ out_gt) {
  pdl_launch_dependents();
  pdl_wait();
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int n = blockIdx.z;
  if (x >= crop_w) return;
  const int32_t* g = geom + n * kGeom;
  const int H = g[0], W = g[1], mirror = g[2], sh = g[3], sw = g[4], ph = g[5], pw = g[6];
  const int64_t off = static_cast<int64_t>(static_cast<uint32_t>(g[7]));

  // image: mirror -> INTER_LINEAR to (sh, sw) -> normalize (LUT) -> crop / pad with 0
  const size_t plane = static_cast<size_t>(crop_h) * crop_w;
  float* o = out_img + static_cast<size_t>(n) * 3 * plane + static_cast<size_t>(y) * crop_w + x;
  const int ys = crop_src(y, crop_h, sh, ph), xs = crop_src(x, crop_w, sw, pw);
  if (ys < 0 || xs < 0) {
    o[0] = 0.f;
    o[plane] = 0.f;
    o[2 * plane] = 0.f;
  } else {
    int sy, b0, b1, sx, a0, a1;
    linear_coef(ys, H, sh, false, sy, b0, b1);
    linear_coef(xs, W, sw, true, sx, a0, a1);
    const int r0 = min(max(sy, 0), H - 1), r1 = min(max(sy + 1, 0), H - 1);
    int c0 = sx, c1 = min(sx + 1, W - 1);
    if (mirror) c0 = W - 1 - c0, c1 = W - 1 - c1;  // coefficients live in the flipped frame; the source is read unflipped
    const uint8_t* p = img + off * 3;
    const uint8_t* p00 = p + (static_cast<int64_t>(r0) * W + c0) * 3;
    const uint8_t* p01 = p + (static_cast<int64_t>(r0) * W + c1) * 3;
    const uint8_t* p10 = p + (static_cast<int64_t>(r1) * W + c0) * 3;
    const uint8_t* p11 = p + (static_cast<int64_t>(r1) * W + c1) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int s0 = static_cast<int>(p00[c]) * a0 + static_cast<int>(p01[c]) * a1;
      const int s1 = static_cast<int>(p10[c]) * a0 + static_cast<int>(p11[c]) * a1;
      int v = ((((s0 >> 4) * b0) >> 16) + (((s1 >> 4) * b1) >> 16) + 2) >> 2;
      v = min(max(v, 0), 255);
      o[c * plane] = __ldg(lut + c * 256 + v);
    }
  }

  // label: mirror -> INTER_NEAREST to (sh, sw) -> crop / pad with 255 -> INTER_NEAREST to (label_h, label_w)
  if (y < label_h && x < label_w) {
    const int yc = crop_src(nearest_src(y, crop_h, label_h), crop_h, sh, ph);
    const int xc = crop_src(nearest_src(x, crop_w, label_w), crop_w, sw, pw);
    long long v = 255;
    if (yc >= 0 && xc >= 0) {
      const int r = nearest_src(yc, H, sh);
      int c = nearest_src(xc, W, sw);
      if (mirror) c = W - 1 - c;
      v = gt[off + static_cast<int64_t>(r) * W + c];
    }
    out_gt[(static_cast<size_t>(n) * label_h + y) * label_w + x] = v;
  }
}

}  // namespace

int train_pre_launch(const fsb_train_pre_desc& d, const uint8_t* img, const uint8_t* gt, const int32_t* geom, const float* lut,
                     float* out_img, long long* out_gt, cudaStream_t stream) {
  const dim3 grid(static_cast<unsigned>((d.crop_w + 127) / 128), static_cast<unsigned>(d.crop_h), static_cast<unsigned>(d.n));
  FSB_LAUNCH(train_pre_kernel, grid, dim3(128), 0, stream, d.crop_h, d.crop_w, d.label_h, d.label_w, img, gt, geom, lut, out_img,
             out_gt);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "train_pre launch");
  return FSB_OK;
}

}  // namespace fsb
