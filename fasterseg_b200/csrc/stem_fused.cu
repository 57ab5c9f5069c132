// stem_fused.cu -- K1f: the RGB stem (stem.0, 3x3 s2 3 -> C0) and the first conv of stem.1 (3x3 s2 C0 -> 64) as ONE kernel, so
// the 1/2-resolution map between them never goes through HBM (ConvNorm at train/model_seg.py:193 followed by conv1 of
// BasicResidual2x, search/operations.py:280-359).  Inference only: BN folded into scale / shift, ReLU after both convs.
//
// A CTA (256 threads = two warpgroups, persistent over output tiles, 2 CTAs per SM) owns 16 x 8 output pixels of stem.1.conv1 at a
// time (the K1 per-tap tile of that conv) and keeps both weight sets in shared memory for its whole life.  Per tile:
//   1. stem.0 on the 17 x 33 window of the 1/2 map the tile needs: window pixels in chunks of 128 (5 chunks, a warpgroup takes
//      every other one); a thread gathers the 27 inputs of its pixel exactly as stem_conv_tc_kernel does (same fp16 rounding, same
//      zero padding of the normalised image), two m64n32k16 wgmma per m64 half, BN + ReLU, fp16.  The result goes to four parity
//      planes (window row / column parity), 9 rows x 17 pixels each, 64 B per pixel in the SWIZZLE_64B K-major layout, the swizzle
//      applied to absolute shared-memory address bits as TMA would.  Window pixels outside the 1/2 map are stem.1's zero padding
//      and are written as 0.
//   2. stem.1.conv1: tap (r, s) of the stride-2 conv is a dense 8 x 16 block of plane (r & 1, s & 1) shifted by (r >> 1, s >> 1)
//      pixels, read through a shifted descriptor (as K1's window mode does with its halo window).  Warpgroup h computes the m64
//      half made of tile columns 8h..8h+7 (8-pixel groups = tile rows, group stride = the plane pitch): tap-major, one K = 32
//      chunk per tap, N = 64 -- the MMA sequence K1 runs for this conv, so the result is bit-identical to the two-kernel path.
//   3. BN + ReLU on the fragments, fp16, staged in the 128B-swizzled layout of K1's TMA-store epilogue and written with one TMA
//      store (channel offset / stride of the destination in the tensor map).
#include <type_traits>

#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

namespace {
constexpr int kThreadsF = 256;
constexpr int kTw = 16, kTh = 8;                       // stem.1.conv1 tile (output pixels)
constexpr int kWinH = 2 * kTh + 1, kWinW = 2 * kTw + 1;  // 17 x 33 pixels of the 1/2 map
constexpr int kWinPix = kWinH * kWinW;                 // 561
constexpr int kChunks = (kWinPix + 127) / 128;         // 5
constexpr int kPitch = kTw + 1;                        // plane pitch (pixels): 17 columns of the even planes
constexpr int kPlaneBytes = ((kTh + 1) * kPitch * 64 + 1023) / 1024 * 1024;
// dynamic shared memory (offsets from the 1024-aligned base)
constexpr uint32_t kOffB1 = 0;                               // stem.1 weights [9 taps][64 rows][64 B]
constexpr uint32_t kOffB0 = kOffB1 + 9 * 64 * 64;            // stem.0 weights [32 rows][64 B]
constexpr uint32_t kOffPlanes = kOffB0 + 32 * 64;            // 4 parity planes
constexpr uint32_t kOffA0 = kOffPlanes + 4 * kPlaneBytes;    // stem.0 A tiles, one per warpgroup [128][64 B]; also the output staging
constexpr uint32_t kSmemF = kOffA0 + 128 * 128 + 1024;       // + the slack that aligns the base
}  // namespace

// byte offset of 16-byte chunk `chunk` of row `row` (64-byte rows) in a SWIZZLE_64B region whose base is 512-aligned
__device__ __forceinline__ uint32_t sw64(uint32_t row_off, int chunk) {
  return row_off + ((static_cast<uint32_t>(chunk) ^ ((row_off >> 7) & 3u)) << 4);
}

template <typename TIn>
__global__ void __launch_bounds__(kThreadsF, 2)
stem_fused_tc_kernel(int N, int H, int W, int C0, const TIn* __restrict__ x, const __half* __restrict__ lut,
                     const float* __restrict__ w0, const float* __restrict__ scale0, const float* __restrict__ shift0,
                     const __half* __restrict__ w1, const float* __restrict__ scale1, const float* __restrict__ shift1,
                     const __grid_constant__ CUtensorMap tmap_y, int tiles_w, int tiles_h) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __half s_lut[std::is_same<TIn, uint8_t>::value ? 768 : 2];
  __shared__ float s_scale0[32], s_shift0[32], s_scale1[64], s_shift1[64];
  pdl_launch_dependents();
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x;
  const int wg = tid >> 7;   // warpgroup
  const int t = tid & 127;   // thread inside the warpgroup
  const int H0 = H / 2 + (H & 1), W0 = W / 2 + (W & 1);  // 1/2 map
  pdl_wait();  // weights / scale / shift / input may have been produced by the immediately preceding kernel

  // ---- once per CTA: LUT, epilogue vectors, both weight sets ----
  if constexpr (std::is_same<TIn, uint8_t>::value)
    for (int i = tid; i < 768; i += kThreadsF) s_lut[i] = lut[i];
  if (tid < 32) {
    const bool ok = tid < C0;
    s_scale0[tid] = ok ? scale0[tid] : 1.f;
    s_shift0[tid] = ok ? shift0[tid] : 0.f;
  } else if (tid >= 64 && tid < 128) {
    s_scale1[tid - 64] = scale1[tid - 64];
    s_shift1[tid - 64] = shift1[tid - 64];
  } else if (tid >= 128 && tid < 160) {
    // stem.0 weights -> B rows (one thread per output channel, zero rows up to 32): fp32 OIHW is already [co][27]
    const int co = tid - 128;
    __half hv[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) hv[k] = __float2half_rn((co < C0 && k < 27) ? w0[co * 27 + k] : 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint4*>(smem + sw64(kOffB0 + co * 64, j)) = *reinterpret_cast<const uint4*>(&hv[j * 8]);
  }
  // stem.1 weights: packed fp16 [tap][64][32] (K1's layout, npad = 64, kpad = 32), 16 B per (tap, row, chunk)
  for (int i = tid; i < 9 * 64 * 4; i += kThreadsF) {
    const int row = i >> 2;  // tap * 64 + output channel
    *reinterpret_cast<uint4*>(smem + sw64(kOffB1 + row * 64, i & 3)) = reinterpret_cast<const uint4*>(w1)[i];
  }
  fence_proxy_async_smem();  // the weights are read by the MMAs (async proxy) after the first barrier of the tile loop

  uint8_t* a0 = smem + kOffA0 + wg * (128 * 64);
  uint8_t* stage = smem + kOffA0;  // output staging (128 pixels x 128 B), reuses both A tiles after the stem.0 phase
  const uint32_t sbase = smem_u32(smem);
  const size_t plane = static_cast<size_t>(H) * W;
  const int tiles = tiles_w * tiles_h * N;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int tx = tile % tiles_w;
    const int ty = (tile / tiles_w) % tiles_h;
    const int n = tile / (tiles_w * tiles_h);
    const int ow0 = tx * kTw, oh0 = ty * kTh;
    // the previous tile's TMA store has read the staging area and every MMA of it has retired: A tiles and planes are free
    if (tid == 0) tma_store_wait_read();
    __syncthreads();

    // ================= 1. stem.0 on the window: 1/2-map rows 2*oh0-1 .. 2*oh0+15, columns 2*ow0-1 .. 2*ow0+31 =================
    for (int ch = wg; ch < kChunks; ch += 2) {
      const int q = ch * 128 + t;
      const int wr = q / kWinW, wc = q - (q / kWinW) * kWinW;
      const int y0 = 2 * oh0 - 1 + wr, x0 = 2 * ow0 - 1 + wc;
      const bool inside = q < kWinPix && y0 >= 0 && y0 < H0 && x0 >= 0 && x0 < W0;
      __half hv[32];
      const int xl = x0 * 2 - 1;  // leftmost input column of the pixel's 3 x 3 window
      const bool ok0 = xl >= 0, ok2 = xl + 2 < W;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int hi = y0 * 2 + r - 1;
        const bool hok = inside && hi >= 0 && hi < H;
        const bool sok[3] = {hok && ok0, hok, hok && ok2};
        if constexpr (std::is_same<TIn, uint8_t>::value) {
          const uint8_t* rp = x + ((static_cast<size_t>(n) * H + (hok ? hi : 0)) * W + xl) * 3;
#pragma unroll
          for (int s = 0; s < 3; ++s)
#pragma unroll
            for (int ci = 0; ci < 3; ++ci)  // zero padding of the NORMALISED image, like the reference's conv
              hv[ci * 9 + r * 3 + s] = sok[s] ? s_lut[ci * 256 + rp[s * 3 + ci]] : __float2half_rn(0.f);
        } else {
          const TIn* rp = x + (static_cast<size_t>(n) * 3 * H + (hok ? hi : 0)) * W + xl;
#pragma unroll
          for (int ci = 0; ci < 3; ++ci)
#pragma unroll
            for (int s = 0; s < 3; ++s)
              hv[ci * 9 + r * 3 + s] = __float2half_rn(sok[s] ? static_cast<float>(rp[ci * plane + s]) : 0.f);
        }
      }
#pragma unroll
      for (int k = 27; k < 32; ++k) hv[k] = __float2half_rn(0.f);
      named_bar_sync(1 + wg, 128);  // this warpgroup's previous chunk has retired its MMAs
#pragma unroll
      for (int j = 0; j < 4; ++j) *reinterpret_cast<uint4*>(a0 + sw64(t * 64, j)) = *reinterpret_cast<const uint4*>(&hv[j * 8]);
      fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the MMA (async proxy)
      named_bar_sync(1 + wg, 128);
      float acc[2][16];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[h][i] = 0.f;
      {
        const uint64_t da = wgmma_desc_kmajor(smem_u32(a0), 64);
        const uint64_t db = wgmma_desc_kmajor(sbase + kOffB0, 64);
        constexpr uint64_t kHalf = (64 * 64) >> 4;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          wgmma_f16<32, 0>(acc[0], da + 2 * k, db + 2 * k);
          wgmma_f16<32, 0>(acc[1], da + kHalf + 2 * k, db + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<0>();
      }
      // BN + ReLU -> fp16 -> parity plane (pairs of adjacent channels per 4-byte store).  The accumulator is read on every path
      // (a read under a branch makes ptxas serialise the wgmma of the kernel); rows past the window store nothing.
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
          const int m = ch * 128 + 64 * h + wgmma_row(t, i);
          const int r2 = m / kWinW, c2 = m - (m / kWinW) * kWinW;
          const int yy = 2 * oh0 - 1 + r2, xx = 2 * ow0 - 1 + c2;
          const int c = wgmma_col(t, i);
          const float f0 = acc[h][i] * s_scale0[c] + s_shift0[c];
          const float f1 = acc[h][i + 1] * s_scale0[c + 1] + s_shift0[c + 1];
          const uint32_t v = pack_half2(fmaxf(f0, 0.f), fmaxf(f1, 0.f));
          const bool in_map = yy >= 0 && yy < H0 && xx >= 0 && xx < W0;  // outside the 1/2 map: stem.1's zero padding
          const uint32_t row_off = kOffPlanes + ((r2 & 1) * 2 + (c2 & 1)) * kPlaneBytes + ((r2 >> 1) * kPitch + (c2 >> 1)) * 64;
          if (m < kWinPix) *reinterpret_cast<uint32_t*>(smem + sw64(row_off, c >> 3) + (c & 7) * 2) = in_map ? v : 0u;
        }
    }
    fence_proxy_async_smem();
    __syncthreads();

    // ================= 2. stem.1.conv1: warpgroup wg = m64 half of tile columns 8*wg .. 8*wg+7 =================
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    // shared-memory base re-read per tile: left loop-invariant, the 18 descriptors below are hoisted out of the tile loop and spilled
    uint32_t sb;
    asm volatile("mov.u32 %0, %1;" : "=r"(sb) : "r"(sbase));
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int r = tap / 3, s = tap - 3 * (tap / 3);
      const uint32_t a_off = kOffPlanes + ((r & 1) * 2 + (s & 1)) * kPlaneBytes + ((r >> 1) * kPitch + (s >> 1) + 8 * wg) * 64;
      const uint64_t da = wgmma_desc(sb + a_off, 16, kPitch * 64, 64);
      const uint64_t db = wgmma_desc_kmajor(sb + kOffB1 + tap * 64 * 64, 64);
#pragma unroll
      for (int k = 0; k < 2; ++k) wgmma_f16<64, 0>(acc, da + 2 * k, db + 2 * k);
    }
    wgmma_commit();
    wgmma_wait<0>();

    // ================= 3. BN + ReLU -> fp16 staged as K1's TMA-store slab, one TMA store =================
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int row = wgmma_row(t, i);
      const int m = (row >> 3) * kTw + 8 * wg + (row & 7);  // tile pixel (row-major 16 x 8)
      const int c = wgmma_col(t, i);
      float f0 = acc[i] * s_scale1[c] + s_shift1[c];
      float f1 = acc[i + 1] * s_scale1[c + 1] + s_shift1[c + 1];
      *reinterpret_cast<uint32_t*>(stage + m * 128 + (((c >> 3) ^ (m & 7)) << 4) + (c & 7) * 2) = pack_half2(fmaxf(f0, 0.f), fmaxf(f1, 0.f));
    }
    fence_proxy_async_smem();  // generic-proxy smem writes -> visible to the TMA engine
    __syncthreads();
    if (tid == 0) {
      tma_store_4d(&tmap_y, stage, 0, ow0, oh0, n);
      tma_store_commit();
    }
  }
  if (tid == 0) tma_store_wait_read();  // smem must outlive the bulk reads
}

// in_kind: 0 = fp32 NCHW, 1 = fp16 NCHW, 2 = uint8 HWC + lut
int stem_fused_launch(int N, int H, int W, int in_kind, const void* x, const void* lut, int C0, const float* w0, const float* scale0,
                      const float* shift0, int C1, const void* w1, const float* scale1, const float* shift1, void* y, int y_cstride,
                      cudaStream_t stream) {
  if (C0 < 16 || C0 > 32 || C1 != 64)
    return set_error(FSB_ERR_UNSUPPORTED, "stem_fused: stem.0 with 16..32 output channels and stem.1.conv1 with 64");
  if ((reinterpret_cast<uintptr_t>(w1) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) || (y_cstride % 8) != 0)
    return set_error(FSB_ERR_UNSUPPORTED, "stem_fused: 16-byte aligned packed weights and output, y_cstride a multiple of 8");
  const int H0 = H / 2 + (H & 1), W0 = W / 2 + (W & 1);
  const int H1 = (H0 - 1) / 2 + 1, W1 = (W0 - 1) / 2 + 1;
  const int tiles_w = (W1 + kTw - 1) / kTw, tiles_h = (H1 + kTh - 1) / kTh;
  CUtensorMap tmap;
  {
    const uint64_t ycs = static_cast<uint64_t>(y_cstride) * 2;
    const uint64_t dims[4] = {static_cast<uint64_t>(C1), static_cast<uint64_t>(W1), static_cast<uint64_t>(H1), static_cast<uint64_t>(N)};
    const uint64_t str[3] = {ycs, ycs * W1, ycs * W1 * H1};
    const uint32_t box[4] = {64u, static_cast<uint32_t>(kTw), static_cast<uint32_t>(kTh), 1u};
    if (int rc = encode_tiled(&tmap, y, 4, dims, str, box, 128)) return rc;
  }
  const int tiles = tiles_w * tiles_h * N;
  int grid = 2 * sm_count();
  if (grid > tiles) grid = tiles;
  const __half* l = static_cast<const __half*>(lut);
  const __half* wp = static_cast<const __half*>(w1);
  const void* entry = in_kind == 0 ? reinterpret_cast<const void*>(stem_fused_tc_kernel<float>)
                      : in_kind == 1 ? reinterpret_cast<const void*>(stem_fused_tc_kernel<__half>)
                                     : reinterpret_cast<const void*>(stem_fused_tc_kernel<uint8_t>);
  if (int rc = ensure_dyn_smem(entry, kSmemF, "cudaFuncSetAttribute(stem_fused)")) return rc;
  if (in_kind == 0)
    FSB_LAUNCH(stem_fused_tc_kernel<float>, dim3(grid), dim3(kThreadsF), kSmemF, stream, N, H, W, C0, static_cast<const float*>(x), l, w0,
               scale0, shift0, wp, scale1, shift1, tmap, tiles_w, tiles_h);
  else if (in_kind == 1)
    FSB_LAUNCH(stem_fused_tc_kernel<__half>, dim3(grid), dim3(kThreadsF), kSmemF, stream, N, H, W, C0, static_cast<const __half*>(x), l,
               w0, scale0, shift0, wp, scale1, shift1, tmap, tiles_w, tiles_h);
  else
    FSB_LAUNCH(stem_fused_tc_kernel<uint8_t>, dim3(grid), dim3(kThreadsF), kSmemF, stream, N, H, W, C0, static_cast<const uint8_t*>(x), l,
               w0, scale0, shift0, wp, scale1, shift1, tmap, tiles_w, tiles_h);
  cudaError_t e = last_launch_error();
  if (e != cudaSuccess) return set_cuda_error(e, "stem_fused launch");
  return FSB_OK;
}

}  // namespace fsb
