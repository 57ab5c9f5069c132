// wgrad_tc.cu -- K7: convolution weight gradient on Hopper tensor cores (wgmma, sm_90a).
//
//   dW[co, ci, r, s] = sum over output pixels p of  dy[p, co] * x[p * stride + (r, s) - pad, ci]
//
// Per filter tap this is a GEMM  D[M = co, N = ci] = A^T[M, K] * B[K, N]  with K = output pixels.  Both operands live in
// memory as NHWC, i.e. pixel-major rows of channel-contiguous data, which is exactly the wgmma "MN-major" canonical layout:
// a TMA box {64 channels, tw, th, 1} lands in shared memory as 128 rows (pixels = K) x 128 bytes (64 channels = M or N),
// 128B-swizzled; 8-pixel groups are 1024 B apart (stride byte offset) and successive 64-channel blocks of the same pixels are
// separate boxes, one tile (16 KB) apart (leading byte offset).  The x tile of tap (r,s) is the dy tile's pixel block
// shifted by the tap (out-of-image pixels zero-filled by TMA; stride-2 convs read the matching parity plane), exactly like
// the forward kernel's A operand.  No transposes, no im2col.
// A CTA owns (co tile of 128, ci tile of 64 or 128, tap, pixel chunk): warp 0 streams the pixel chunk 128 pixels per
// pipeline stage, the warpgroup of warps 4-7 accumulates the 128 x ci_tile fp32 tile in registers (two m64 halves) and adds
// it into the fp32 master-layout gradient with atomics (pixel chunks of the same tile race benignly), scaled by 1/loss-scale.
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

constexpr int kWgThreads = 256;
constexpr int kWgMaxStages = 6;
constexpr int kWgPix = 128;           // K per stage
constexpr int kWgSub = kWgPix * 128;  // bytes of one [128 pixels x 64 channels] sub-tile

struct WgradTcParams {
  CUtensorMap tmap_dy;     // {Cout, Wo, Ho, N}, box {64, tw, th, 1}
  CUtensorMap tmap_x[4];   // input (parity planes for stride 2), box {64, tw, th, 1}
  int taps, ksize;
  int tap_map[9], tap_dh[9], tap_dw[9];
  int tiles_w, tiles_h, n_img;  // pixel tiling of the OUTPUT map
  int tw, th;
  int Cout, Cin;
  int co_tiles, ci_tiles;
  int chunks;                       // pixel-tile chunks (grid.y)
  int stages;
  float inv_gscale;
  float* dw;
  long long so, si;
};

template <int NT>  // ci tile: 64 or 128
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_tc_kernel(const __grid_constant__ WgradTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kWgMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kWgMaxStages];

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kSub = NT / 64;                     // x sub-tiles per stage
  constexpr uint32_t kStageBytes = static_cast<uint32_t>(2 + kSub) * kWgSub;

  int b = blockIdx.x;
  const int co_t = b % p.co_tiles;
  b /= p.co_tiles;
  const int ci_t = b % p.ci_tiles;
  b /= p.ci_tiles;
  const int tap = b;
  const int co0 = co_t * 128, ci0 = ci_t * NT;
  const int total_tiles = p.tiles_w * p.tiles_h * p.n_img;
  const int per = (total_tiles + p.chunks - 1) / p.chunks;
  const int t_begin = blockIdx.y * per;
  const int t_end = min(total_tiles, t_begin + per);
  const int n_iters = t_end - t_begin;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmap_dy);
    tma_prefetch_desc(&p.tmap_x[p.tap_map[tap]]);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);  // one arrival per warp of the MMA warpgroup
    }
    mbar_fence_init();
  }
  pdl_wait();
  __syncthreads();
  if (n_iters <= 0) {
    // nothing to do for this chunk (more chunks than tiles)
  } else if (warp == 0) {
    // converged warp, only the TMA issue under elect.sync
    const CUtensorMap* mx = &p.tmap_x[p.tap_map[tap]];
    RingPos rp;
    uint8_t* st = smem;
    int tile_w = t_begin % p.tiles_w, tile_h = (t_begin / p.tiles_w) % p.tiles_h, img = t_begin / (p.tiles_w * p.tiles_h);
    for (int it = 0; it < n_iters; ++it) {
      const int w0 = tile_w * p.tw, h0 = tile_h * p.th;
      mbar_wait_inline(&empty_bar[rp.s], rp.phase ^ 1u);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full_bar[rp.s], kStageBytes);
        tma_load_4d(st, &p.tmap_dy, &full_bar[rp.s], co0, w0, h0, img);
        tma_load_4d(st + kWgSub, &p.tmap_dy, &full_bar[rp.s], co0 + 64, w0, h0, img);
        for (int j = 0; j < kSub; ++j)
          tma_load_4d(st + static_cast<size_t>(2 + j) * kWgSub, mx, &full_bar[rp.s], ci0 + j * 64, w0 + p.tap_dw[tap],
                      h0 + p.tap_dh[tap], img);
      }
      __syncwarp();
      st += kStageBytes;
      rp.advance(p.stages);
      if (rp.s == 0) st = smem;
      if (++tile_w == p.tiles_w) {   // next spatial tile without integer division
        tile_w = 0;
        if (++tile_h == p.tiles_h) {
          tile_h = 0;
          ++img;
        }
      }
    }
  } else if (warp >= 4) {
    const int tw = threadIdx.x - 128;  // thread index inside the warpgroup
    float acc[2][NT / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[h][i] = 0.f;
    const uint32_t s0 = smem_u32(smem);
    RingPos rp;
    uint32_t soff = 0;
    int prev = -1;
    for (int it = 0; it < n_iters; ++it) {
      mbar_wait_inline(&full_bar[rp.s], rp.phase);
      wgmma_fence();
      const uint32_t sa = s0 + soff;
      const uint32_t sb = sa + 2 * kWgSub;
#pragma unroll
      for (int k = 0; k < kWgPix / 16; ++k) {
        // 16 pixels = two 8-row groups = 2048 B further down each sub-tile; co 0-63 / 64-127 are the two dy sub-tiles
        const uint64_t db = wgmma_desc(sb + k * 2048, kWgSub, 1024, 128);
        wgmma_f16<NT, 1>(acc[0], wgmma_desc(sa + k * 2048, kWgSub, 1024, 128), db);
        wgmma_f16<NT, 1>(acc[1], wgmma_desc(sa + kWgSub + k * 2048, kWgSub, 1024, 128), db);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous stage's MMAs have read their operands: hand that slot back to the producer
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = rp.s;
      soff += kStageBytes;
      rp.advance(p.stages);
      if (rp.s == 0) soff = 0;
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) {
        const int co = co0 + 64 * h + wgmma_row(tw, i), ci = ci0 + wgmma_col(tw, i);
        if (co < p.Cout && ci < p.Cin)
          atomicAdd(p.dw + static_cast<long long>(co) * p.so + tap + static_cast<long long>(ci) * p.si, acc[h][i] * p.inv_gscale);
      }
  }
  __syncthreads();
}

int encode_tiled_generic(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box, int swizzle_bytes);

static inline int floordiv2(int a) { return (a >= 0) ? a / 2 : -((-a + 1) / 2); }

int conv_wgrad_tc_supported(const fsb_conv_desc* d, int dy_cstride) {
  if (!(d->ksize == 1 || d->ksize == 3) || !(d->stride == 1 || d->stride == 2) || d->dil != 1) return 0;
  if (d->Cin < 16 || d->Cout < 16 || (d->x_cstride % 8) != 0 || (dy_cstride % 8) != 0) return 0;
  if (opt(OPT_WGRAD_TC) == 0) return 0;
  return 1;
}

int conv_wgrad_tc_launch(const fsb_conv_desc* d, const void* x, const void* dy, int dcs, float* dw, int64_t so, int64_t si,
                         float gscale, cudaStream_t stream) {
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(dy) & 15))
    return set_error(FSB_ERR_INVALID, "wgrad_tc: x / dy must be 16-byte aligned");
  WgradTcParams p;
  memset(&p, 0, sizeof(p));
  p.ksize = d->ksize;
  p.taps = d->ksize * d->ksize;
  p.tw = d->Wo >= 16 ? 16 : 8;
  p.th = kWgPix / p.tw;
  p.tiles_w = (d->Wo + p.tw - 1) / p.tw;
  p.tiles_h = (d->Ho + p.th - 1) / p.th;
  p.n_img = d->N;
  p.Cout = d->Cout;
  p.Cin = d->Cin;
  p.co_tiles = (d->Cout + 127) / 128;
  const int ci64 = (d->Cin + 63) / 64 * 64;
  // ci tile of 64 or 128 channels: two m64 x ci_tile accumulators = at most 128 registers per thread
  const int ci_tile = ci64 % 128 == 0 ? 128 : 64;
  p.ci_tiles = ci64 / ci_tile;
  p.inv_gscale = 1.0f / gscale;
  p.dw = dw;
  p.so = so;
  p.si = si;
  const int total_tiles = p.tiles_w * p.tiles_h * d->N;
  const int fixed = p.co_tiles * p.ci_tiles * p.taps;
  int chunks = (sm_count() * 2 + fixed - 1) / fixed;
  if (chunks > total_tiles) chunks = total_tiles;
  // deterministic mode (FSB_DETERMINISTIC=1 / fsb_set_option): no split over pixels, so every gradient element has exactly one
  // writer and the fp32 accumulation order is fixed (slower: co_tiles * ci_tiles * taps CTAs only)
  if (chunks < 1 || opt(OPT_DETERMINISTIC) == 1) chunks = 1;
  p.chunks = chunks;
  const size_t stage_bytes = static_cast<size_t>(2 + ci_tile / 64) * kWgSub;
  int stages = static_cast<int>((192 * 1024) / stage_bytes);
  if (stages > kWgMaxStages) stages = kWgMaxStages;
  const int per = (total_tiles + chunks - 1) / chunks;
  if (stages > per) stages = per;
  if (stages < 1) stages = 1;
  p.stages = stages;
  const size_t smem_bytes = stage_bytes * stages + 1024;

  const uint32_t box[4] = {64u, static_cast<uint32_t>(p.tw), static_cast<uint32_t>(p.th), 1u};
  {
    const uint64_t cs = static_cast<uint64_t>(dcs) * 2;
    const uint64_t dims[4] = {static_cast<uint64_t>(d->Cout), static_cast<uint64_t>(d->Wo), static_cast<uint64_t>(d->Ho),
                              static_cast<uint64_t>(d->N)};
    const uint64_t str[3] = {cs, cs * d->Wo, cs * d->Wo * d->Ho};
    int rc = encode_tiled_generic(&p.tmap_dy, dy, 4, dims, str, box, 128);
    if (rc) return rc;
  }
  const __half* xb = static_cast<const __half*>(x);
  const uint64_t cs = static_cast<uint64_t>(d->x_cstride) * 2;
  if (d->stride == 1) {
    const uint64_t dims[4] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(d->W), static_cast<uint64_t>(d->H),
                              static_cast<uint64_t>(d->N)};
    const uint64_t str[3] = {cs, cs * d->W, cs * d->W * d->H};
    int rc = encode_tiled_generic(&p.tmap_x[0], xb, 4, dims, str, box, 128);
    if (rc) return rc;
    for (int r = 0; r < d->ksize; ++r)
      for (int s = 0; s < d->ksize; ++s) {
        const int tp = r * d->ksize + s;
        p.tap_map[tp] = 0;
        p.tap_dh[tp] = r - d->pad + d->off_h;
        p.tap_dw[tp] = s - d->pad + d->off_w;
      }
  } else {
    bool used[4] = {false, false, false, false};
    for (int r = 0; r < d->ksize; ++r)
      for (int s = 0; s < d->ksize; ++s) {
        const int tp = r * d->ksize + s;
        const int qh = r - d->pad + d->off_h, qw = s - d->pad + d->off_w;
        const int ph = ((qh % 2) + 2) % 2, pw = ((qw % 2) + 2) % 2;
        p.tap_map[tp] = ph * 2 + pw;
        p.tap_dh[tp] = floordiv2(qh);
        p.tap_dw[tp] = floordiv2(qw);
        used[ph * 2 + pw] = true;
      }
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw) {
        if (!used[ph * 2 + pw]) continue;
        const int Hp = (d->H - ph + 1) / 2, Wp = (d->W - pw + 1) / 2;
        if (Hp <= 0 || Wp <= 0) return set_error(FSB_ERR_INVALID, "wgrad_tc: empty parity plane");
        const uint64_t dims[4] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(Wp), static_cast<uint64_t>(Hp),
                                  static_cast<uint64_t>(d->N)};
        const uint64_t str[3] = {2 * cs, 2 * cs * d->W, cs * d->W * d->H};
        int rc = encode_tiled_generic(&p.tmap_x[ph * 2 + pw], xb + (static_cast<size_t>(ph) * d->W + pw) * d->x_cstride, 4, dims,
                                      str, box, 128);
        if (rc) return rc;
      }
  }
  const void* kernel = ci_tile == 128 ? reinterpret_cast<const void*>(conv_wgrad_tc_kernel<128>)
                                      : reinterpret_cast<const void*>(conv_wgrad_tc_kernel<64>);
  if (int rc = ensure_dyn_smem(kernel, 220 * 1024, "cudaFuncSetAttribute(conv_wgrad_tc)")) return rc;
  dim3 grid(static_cast<unsigned>(fixed), static_cast<unsigned>(chunks));
  const cudaError_t e = ci_tile == 128 ? launch_kernel(conv_wgrad_tc_kernel<128>, grid, dim3(kWgThreads), smem_bytes, stream, p)
                                       : launch_kernel(conv_wgrad_tc_kernel<64>, grid, dim3(kWgThreads), smem_bytes, stream, p);
  if (e != cudaSuccess) return set_cuda_error(e, "conv_wgrad_tc launch");
  return FSB_OK;
}

}  // namespace fsb
