// conv_tc.cu -- K1: im2col-free implicit-GEMM convolution on Hopper tensor cores (wgmma, sm_90a).
//
// Replaces F.conv2d (+ BatchNorm eval + ReLU) for every 3x3 / 1x1 conv of the FasterSeg hot path
// (reference call sites: search/slimmable_ops.py:47, search/operations.py:72-83,146-150,..., search/seg_oprs.py:21-39).
//
// GEMM view:  D[M = 128 output pixels (th x tw tile), N = Cout tile] += A[M, K] * B[N, K]^T,
//             K = taps * Cin, walked as (tap, 64- or 32-channel chunk).
//   A tile  : for tap (r,s) the 128 x BK slab is ONE TMA box {BK, tw, th, 1} of the NHWC input at the
//             tap-shifted coordinate; out-of-image rows/cols and channel tails are zero-filled by TMA, so
//             padding costs nothing and no im2col buffer exists.  Stride-2 convs address one of four
//             parity planes of the input (each its own tensor map), which keeps every box dense.
//             3x3 stride-1 convs run in window mode instead (K walked as (64-channel chunk, tap)): one halo window of
//             the input per chunk, the nine taps read from it through shifted descriptors (see below).
//   B tile  : packed fp16 weights [tap][Npad][Kpad] (K-major), one TMA box {BK, NT, 1}.
//   D       : fp32 accumulator in the registers of one warpgroup (two m64 halves of the 128-pixel tile, NT <= 128
//             columns each: at most 128 accumulator registers per thread).
// Warp roles (256 threads): warp 0 = TMA producer (warps 1-3 only join the final barrier), warps 4-7 = the MMA warpgroup.
// After the main loop the warpgroup parks the accumulator in shared memory as [channel][pixel] and runs the epilogue on it
// (BN scale/shift -> ReLU -> fp16 -> NHWC store with channel offset/stride, which is how torch.cat(dim=1) call sites
// become free), one pixel per thread.
#include "fsb_common.cuh"
#include "fsb_internal.h"

namespace fsb {

constexpr int kTileM = 128;
constexpr int kMaxStages = 8;
constexpr int kThreads = 256;
constexpr int kAccLd = kTileM + 4;  // padded channel column of the parked accumulator: conflict-free fragment stores and row reads

struct ConvTcParams {
  CUtensorMap tmap_a[4];
  CUtensorMap tmap_b;
  CUtensorMap tmap_y[2];  // output maps for the TMA-store epilogue: [0] 64-channel slabs (SW128), [1] tail slab (dense)
  int tma_store;          // 1: fp16 tile staged in smem and written with cp.async.bulk.tensor (full-line, clipped stores)
  int tail_w;             // channels in the last slab of an N tile when n_tile % 64 != 0
  int taps;
  int tap_map[9];
  int tap_dh[9];
  int tap_dw[9];
  int tap_widx[9];  // which [tap] slice of the packed weights each tap multiplies (identity for plain convs)
  int k_chunks;
  int Ho, Wo;
  int tiles_w, tiles_h;
  int tw, th;
  // window mode only (see conv_tc_kernel): window = win_rows x win_pitch input pixels of 128 B; A row (half h, 8-row group g,
  // row i) of tap (r,s) is window pixel (r * win_pitch + s) + h * win_half + g * win_sbo / 128 + i, which is tile pixel
  // h * m_half + g * m_grp + i
  int win_pitch, win_rows;
  int win_sbo;     // bytes between 8-pixel groups (wgmma stride byte offset)
  int win_half;    // pixels between the two m64 halves
  int win_stride;  // bytes per window buffer (1024-aligned)
  int m_half, m_grp;
  int Cout;
  int stages;
  int y_cstride;
  uint32_t flags;
  const float* scale;
  const float* shift;
  __half* y;
  float* stats;   // partial rows (one per spatial tile = blockIdx.x), see bn.cu "Deterministic statistics"
  int stats_C;    // row half-width (row stride = 2 * stats_C floats)
  int stats_off;  // channel offset of this conv's output inside a row
};

// Parameters of the FSB_CONV_Y_UP2 instances: the staged output goes to y_reps = 4 lattices (one per 2x2 parity), lattice 0
// through p.tmap_y, lattice l >= 1 through tmap_up[2l - 2] (64-channel slabs) and tmap_up[2l - 1] (tail slab).  A struct of its
// own, so that every other launch keeps ConvTcParams' size (kernel-parameter bytes are uploaded per launch).
struct ConvTcUp2Params {
  ConvTcParams p;
  int y_reps;
  CUtensorMap tmap_up[6];
};

// shared memory after the main loop: [0, kOutBytes) = statistics partials or the TMA-store staging slabs,
// [kOutBytes, + NT * kAccLd * 4) = the parked accumulator; both reuse the (then idle) stage ring
template <int NT>
__host__ __device__ constexpr uint32_t conv_tc_out_bytes() { return static_cast<uint32_t>((NT + 63) / 64) * kTileM * 128; }
template <int NT>
__host__ __device__ constexpr uint32_t conv_tc_epilogue_bytes() { return conv_tc_out_bytes<NT>() + static_cast<uint32_t>(NT) * kAccLd * 4; }

// Window mode (WIN: 3x3 stride-1 dilation-1 convs without custom tap tables).  Per 64-channel chunk the producer loads the
// (th + 2) x (tw + 2) input pixels the tile needs (halo included, out-of-image pixels and channels >= Cin zero-filled by TMA)
// ONCE into a window buffer (ring of 2); the operand of tap (r,s) is the same window read through a descriptor whose start
// address is shifted by r window rows and s pixels (TMA and wgmma both apply the 128B swizzle to absolute shared-memory
// address bits, so a 128B-multiple shift inside the 1024B-aligned window reads back what TMA wrote).  Only the weights stream
// per (chunk, tap), through the stage ring.  Every input byte of a tile crosses L2 -> SM about 1.4x per chunk instead of 9x.
// Each m64 half of the 128-pixel tile must be 8 groups of 8 window-contiguous pixels at one stride:
//   16 x 8 tiles: half h = the 8 x 8 block at columns 8h..8h+7, groups = tile rows (stride tw + 2 pixels);
//   8 x 16 tiles: half h = tile rows 8h..8h+7, groups = tile rows (stride tw + 2 pixels);
//   row strip (128 x 1 tiles, FSB_CONV_TC2=2): half h = pixels 64h..64h+63 of the row, groups 8 pixels apart.

// The kernel body.  UP2 (FSB_CONV_Y_UP2) only adds the stores of each staged slab to lattices 1 .. y_reps - 1; it is compiled
// into instances of its own (conv_tc_up2_kernel) so that the instances every other call runs keep their registers.
template <int BK, int NT, bool WIN, bool UP2>
__device__ __forceinline__ void conv_tc_body(const ConvTcParams& p, const CUtensorMap* tmap_up, int y_reps) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(8) uint64_t win_full[2];
  __shared__ __align__(8) uint64_t win_empty[2];
  __shared__ float s_scale[NT];
  __shared__ float s_shift[NT];

  pdl_launch_dependents();  // let the next kernel's prologue overlap our main loop / tail
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr uint32_t kABytes = kTileM * BK * 2;
  constexpr uint32_t kStageBytes = WIN ? NT * BK * 2 : kABytes + NT * BK * 2;
  static_assert(!WIN || BK == 64, "windows are 128B-swizzled 64-channel rows");
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  // tile coordinates
  int t = blockIdx.x;
  const int tile_w = t % p.tiles_w;
  t /= p.tiles_w;
  const int tile_h = t % p.tiles_h;
  const int img = t / p.tiles_h;
  const int w0 = tile_w * p.tw;
  const int h0 = tile_h * p.th;
  const int n0 = blockIdx.y * NT;
  const int k_iters = p.taps * p.k_chunks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.tmap_a[0]);
    tma_prefetch_desc(&p.tmap_b);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);  // one arrival per warp of the MMA warpgroup
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&win_full[w], 1);
      mbar_init(&win_empty[w], 4);
    }
    mbar_fence_init();
  }
  pdl_wait();  // predecessor's outputs (our x) and anything it still reads (our y) are safe from here on
  // epilogue constants
  for (int c = threadIdx.x; c < NT; c += kThreads) {
    const int ch = n0 + c;
    const bool ok = ch < p.Cout;
    s_scale[c] = (ok && (p.flags & FSB_CONV_AFFINE) && p.scale) ? p.scale[ch] : 1.0f;
    s_shift[c] = (ok && (p.flags & FSB_CONV_AFFINE) && p.shift) ? p.shift[ch] : 0.0f;
  }
  __syncthreads();

  if (WIN && warp == 0) {
    // ================= TMA producer, window mode: one input window per chunk, one weight tile per (chunk, tap) =================
    uint8_t* bring = smem + 2 * p.win_stride;
    const uint32_t win_bytes = static_cast<uint32_t>(p.win_rows * p.win_pitch) * 128u;
    RingPos rp, rw;
    for (int kc = 0; kc < p.k_chunks; ++kc) {
      mbar_wait_inline(&win_empty[rw.s], rw.phase ^ 1u);
      if (elect_one()) {
        mbar_arrive_expect_tx(&win_full[rw.s], win_bytes);
        tma_load_4d(smem + rw.s * p.win_stride, &p.tmap_a[0], &win_full[rw.s], kc * BK, w0 + p.tap_dw[0], h0 + p.tap_dh[0], img);
      }
      __syncwarp();
      rw.advance(2);
      for (int tap = 0; tap < 9; ++tap) {
        mbar_wait_inline(&empty_bar[rp.s], rp.phase ^ 1u);
        if (elect_one()) {
          mbar_arrive_expect_tx(&full_bar[rp.s], kStageBytes);
          tma_load_3d(bring + rp.s * kStageBytes, &p.tmap_b, &full_bar[rp.s], kc * BK, n0, tap);
        }
        __syncwarp();
        rp.advance(p.stages);
      }
    }
  } else if (warp == 0) {
    // ================= TMA producer (converged warp, one elected lane issues) =================
    RingPos rp;
    uint8_t* sa = smem;
    for (int tap = 0; tap < p.taps; ++tap) {
      const CUtensorMap* ma = &p.tmap_a[p.tap_map[tap]];
      const int cw = w0 + p.tap_dw[tap];
      const int chh = h0 + p.tap_dh[tap];
      const int wi = p.tap_widx[tap];
      for (int kc = 0; kc < p.k_chunks; ++kc) {
        mbar_wait_inline(&empty_bar[rp.s], rp.phase ^ 1u);
        if (elect_one()) {
          mbar_arrive_expect_tx(&full_bar[rp.s], kStageBytes);
          tma_load_4d(sa, ma, &full_bar[rp.s], kc * BK, cw, chh, img);
          tma_load_3d(sa + kABytes, &p.tmap_b, &full_bar[rp.s], kc * BK, n0, wi);
        }
        __syncwarp();
        sa += kStageBytes;
        rp.advance(p.stages);
        if (rp.s == 0) sa = smem;
      }
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroup: wgmma over the stage ring, one stage in flight behind the current one =================
    const int tw = threadIdx.x - 128;  // thread index inside the warpgroup
    float acc[2][NT / 2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[h][i] = 0.f;
    // descriptors of stage s = descriptors of stage 0 + s * (kStageBytes >> 4) in the start-address field (shared-memory
    // addresses stay below 256 KB, so the 14-bit field never carries)
    const uint32_t sa0 = smem_u32(smem);
    const uint64_t da0 = wgmma_desc_kmajor(sa0, BK * 2);
    const uint64_t db0 = wgmma_desc_kmajor(sa0 + kABytes, BK * 2);
    constexpr uint32_t kHalf = (64 * BK * 2) >> 4;  // pixel rows 64..127 of the A tile
    if constexpr (WIN) {
      const uint64_t dw0 = wgmma_desc(sa0, 16, p.win_sbo, 128);                // window 0, tap (0,0)
      const uint64_t dbr = wgmma_desc_kmajor(sa0 + 2 * p.win_stride, 128);    // weight ring, stage 0
      const uint64_t whalf = static_cast<uint64_t>(p.win_half * 8);           // win_half pixels x 128 B >> 4
      RingPos rp, rw;
      int prev = -1, prev_w = -1;
      for (int kc = 0; kc < p.k_chunks; ++kc) {
        mbar_wait_inline(&win_full[rw.s], rw.phase);
        const uint64_t dwin = dw0 + static_cast<uint64_t>(rw.s * (p.win_stride >> 4));
        for (int tap = 0; tap < 9; ++tap) {
          const int r = tap / 3, sx = tap - 3 * r;
          mbar_wait_inline(&full_bar[rp.s], rp.phase);
          wgmma_fence();
          const uint64_t da = dwin + static_cast<uint64_t>((r * p.win_pitch + sx) * 8);   // (r rows, sx pixels) x 128 B >> 4
          const uint64_t db = dbr + static_cast<uint64_t>(rp.s * (kStageBytes >> 4));
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            wgmma_f16<NT, 0>(acc[0], da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k));
            wgmma_f16<NT, 0>(acc[1], da + whalf + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k));
          }
          wgmma_commit();
          wgmma_wait<1>();  // the previous group has read its operands
          if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
          if (tap == 0 && prev_w >= 0 && lane == 0) mbar_arrive(&win_empty[prev_w]);  // last group of the previous chunk retired
          prev = rp.s;
          rp.advance(p.stages);
        }
        prev_w = rw.s;
        rw.advance(2);
      }
    } else {
    RingPos rp;
    uint32_t doff = 0;
    int prev = -1;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait_inline(&full_bar[rp.s], rp.phase);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // advance 16 fp16 = 32 B along K inside the swizzle atom: +2 in the (addr >> 4) field
        const uint64_t da = da0 + doff + static_cast<uint64_t>(2 * k), db = db0 + doff + static_cast<uint64_t>(2 * k);
        wgmma_f16<NT, 0>(acc[0], da, db);
        wgmma_f16<NT, 0>(acc[1], da + kHalf, db);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the MMAs of the previous stage have read their operands: hand that slot back to the producer
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = rp.s;
      doff += kStageBytes >> 4;
      rp.advance(p.stages);
      if (rp.s == 0) doff = 0;
    }
    }
    wgmma_wait<0>();
    // park the accumulator as [channel][pixel] behind the epilogue's output area (the stage ring is idle now: every load
    // has been consumed and every MMA has retired in all four warps once the barrier below is passed)
    float* s_acc = reinterpret_cast<float*>(smem + conv_tc_out_bytes<NT>());
    named_bar_sync(1, 128);
    if constexpr (WIN) {
      // this thread's fragment rows are row0 and row0 + 8 (8-row groups g0 and g0 + 1) of each half
      const int row0 = wgmma_row(tw, 0);
      const int m0 = (row0 >> 3) * p.m_grp + (row0 & 7);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float* s_h = s_acc + h * p.m_half + m0;
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) s_h[wgmma_col(tw, i) * kAccLd + ((i >> 1) & 1) * p.m_grp] = acc[h][i];
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) s_acc[wgmma_col(tw, i) * kAccLd + 64 * h + wgmma_row(tw, i)] = acc[h][i];
    }
    named_bar_sync(1, 128);

    // ================= epilogue: thread m of the warpgroup owns pixel m of the tile =================
    const int q = warp & 3;
    const int m = q * 32 + lane;
    const int oh = h0 + m / p.tw;
    const int ow = w0 + m % p.tw;
    const bool pix_ok = (oh < p.Ho) && (ow < p.Wo);
    __half* yrow = p.y + (static_cast<size_t>(img) * p.Ho * p.Wo + static_cast<size_t>(oh) * p.Wo + ow) * p.y_cstride + n0;
    const bool out_f32 = (p.flags & FSB_CONV_OUT_F32) != 0;
    float* yrow32 = reinterpret_cast<float*>(p.y) +
                    (static_cast<size_t>(img) * p.Ho * p.Wo + static_cast<size_t>(oh) * p.Wo + ow) * p.y_cstride + n0;
    const bool vec_ok = out_f32 ? ((reinterpret_cast<uintptr_t>(yrow32) & 15) == 0) : ((reinterpret_cast<uintptr_t>(yrow) & 15) == 0);
    const bool relu = (p.flags & FSB_CONV_RELU) != 0;
    const bool do_stats = (p.flags & FSB_CONV_STATS) != 0 && p.stats != nullptr;
    // per-warp channel statistics of this tile: [4 warps][sum | sumsq][NT] in the output area
    float* s_stat = reinterpret_cast<float*>(smem);
    for (int c0 = 0; c0 < NT; c0 += 64) {
      const int nb = min(4, (NT - c0) >> 4);
#pragma unroll
      for (int b = 0; b < 4; ++b) {
      if (b >= nb) break;
      const int c = c0 + 16 * b;
      float f[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) f[j] = s_acc[(c + j) * kAccLd + m];
      if (do_stats) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          float a = pix_ok ? f[j] : 0.f;
          float b = a * a;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
          }
          if (lane == 0) {
            s_stat[(q * 2 + 0) * NT + c + j] = a;
            s_stat[(q * 2 + 1) * NT + c + j] = b;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float x = f[j] * s_scale[c + j] + s_shift[c + j];
        f[j] = relu ? fmaxf(x, 0.f) : x;
      }
      if (pix_ok && out_f32) {
        const int remaining = p.Cout - (n0 + c);
        if (remaining >= 16 && vec_ok) {
          float4* dst = reinterpret_cast<float4*>(yrow32 + c);
          dst[0] = make_float4(f[0], f[1], f[2], f[3]);
          dst[1] = make_float4(f[4], f[5], f[6], f[7]);
          dst[2] = make_float4(f[8], f[9], f[10], f[11]);
          dst[3] = make_float4(f[12], f[13], f[14], f[15]);
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (j < remaining) yrow32[c + j] = f[j];
        }
      } else if (p.tma_store) {
        // stage this thread's 16 channels of pixel m: slab = 64 channels; full slabs use the 128B-swizzled layout of the
        // output tensor map, the tail slab is dense (tail_w * 2 bytes per pixel)
        uint4 o0, o1;
        o0.x = pack_half2(f[0], f[1]);
        o0.y = pack_half2(f[2], f[3]);
        o0.z = pack_half2(f[4], f[5]);
        o0.w = pack_half2(f[6], f[7]);
        o1.x = pack_half2(f[8], f[9]);
        o1.y = pack_half2(f[10], f[11]);
        o1.z = pack_half2(f[12], f[13]);
        o1.w = pack_half2(f[14], f[15]);
        uint8_t* slab = smem + static_cast<size_t>(c0 >> 6) * (kTileM * 128);
        const int ch16 = (c - c0) >> 3;  // 16-byte chunk index inside the slab row
        if (NT - c0 >= 64) {
          *reinterpret_cast<uint4*>(slab + m * 128 + ((ch16 ^ (m & 7)) << 4)) = o0;
          *reinterpret_cast<uint4*>(slab + m * 128 + (((ch16 + 1) ^ (m & 7)) << 4)) = o1;
        } else {
          uint8_t* row = slab + m * (p.tail_w * 2) + (ch16 << 4);
          *reinterpret_cast<uint4*>(row) = o0;
          *reinterpret_cast<uint4*>(row + 16) = o1;
        }
      } else if (pix_ok) {
        const int remaining = p.Cout - (n0 + c);
        if (remaining >= 16 && vec_ok) {
          uint4 o0, o1;
          o0.x = pack_half2(f[0], f[1]);
          o0.y = pack_half2(f[2], f[3]);
          o0.z = pack_half2(f[4], f[5]);
          o0.w = pack_half2(f[6], f[7]);
          o1.x = pack_half2(f[8], f[9]);
          o1.y = pack_half2(f[10], f[11]);
          o1.z = pack_half2(f[12], f[13]);
          o1.w = pack_half2(f[14], f[15]);
          uint4* dst = reinterpret_cast<uint4*>(yrow + c);
          dst[0] = o0;
          dst[1] = o1;
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (j < remaining) yrow[c + j] = __float2half_rn(f[j]);
        }
      }
      }  // 16-column chunk
      if (p.tma_store) {
        fence_proxy_async_smem();           // generic-proxy smem writes -> visible to the TMA engine
        named_bar_sync(1, 128);             // the 4 epilogue warps
        if (warp == 4 && lane == 0) {
          const bool full = (NT - c0) >= 64;
          tma_store_4d(&p.tmap_y[full ? 0 : 1], smem + static_cast<size_t>(c0 >> 6) * (kTileM * 128), n0 + c0, w0, h0, img);
          if constexpr (UP2)
            for (int l = 1; l < y_reps; ++l)
              tma_store_4d(&tmap_up[2 * l - 2 + (full ? 0 : 1)], smem + static_cast<size_t>(c0 >> 6) * (kTileM * 128), n0 + c0, w0,
                           h0, img);
          tma_store_commit();
        }
      }
    }  // 64-column batch
    if (p.tma_store && warp == 4 && lane == 0) tma_store_wait_read();  // smem must outlive the bulk reads
    if (do_stats) {
      // no atomics: the four warp partials are added in warp order and written as this tile's partial row; the consumer
      // (bn_finalize / rowsum) adds the rows in index order, so the statistics are bit-reproducible run to run
      named_bar_sync(2, 128);
      float* row = p.stats + static_cast<size_t>(blockIdx.x) * 2 * p.stats_C + p.stats_off;
      for (int ch = static_cast<int>(threadIdx.x) - 128; ch < NT; ch += 128) {
        if (n0 + ch >= p.Cout) continue;
        float a = s_stat[0 * NT + ch], b = s_stat[1 * NT + ch];
#pragma unroll
        for (int w = 1; w < 4; ++w) {
          a += s_stat[(w * 2 + 0) * NT + ch];
          b += s_stat[(w * 2 + 1) * NT + ch];
        }
        row[n0 + ch] = a;
        row[p.stats_C + n0 + ch] = b;
      }
    }
  }
  __syncthreads();
}

template <int BK, int NT, bool WIN>
__global__ void __launch_bounds__(kThreads, NT <= 64 ? 2 : 1)
conv_tc_kernel(const __grid_constant__ ConvTcParams p) {
  conv_tc_body<BK, NT, WIN, false>(p, nullptr, 1);
}

template <int BK, int NT, bool WIN>
__global__ void __launch_bounds__(kThreads, NT <= 64 ? 2 : 1)
conv_tc_up2_kernel(const __grid_constant__ ConvTcUp2Params q) {
  conv_tc_body<BK, NT, WIN, true>(q.p, q.tmap_up, q.y_reps);
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static int encode_tiled(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                        const uint32_t* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error(FSB_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bdim[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                 : (swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE));
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr,
                   bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf),
             "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u] base %p stride0 %llu",
             static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1],
             rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, base, (unsigned long long)strides_bytes[0]);
    return set_error(FSB_ERR_CUDA, buf);
  }
  return FSB_OK;
}

int encode_tiled_generic(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box, int swizzle_bytes) {
  return encode_tiled(map, base, rank, dims, strides_bytes, box, swizzle_bytes);
}

static inline int floordiv(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

ConvGeom conv_geom(const fsb_conv_desc* d) {
  ConvGeom g;
  g.taps = d->ksize * d->ksize;
  g.bk = (d->Cin % 64 == 0) ? 64 : 32;
  g.kpad = (d->Cin + g.bk - 1) / g.bk * g.bk;
  g.npad = (d->Cout + 15) / 16 * 16;
  return g;
}

// Which conv_tc mode can run d (without custom tap tables).  3x3 stride-1 dilation-1 convs may use the window mode on their
// 16 x 8 / 8 x 16 tiles: the per-tap mode moves every input byte of a tile from L2 to the SM nine times, and on large maps
// L2 -> SM bandwidth, not HBM or the tensor cores, bounds the kernel (DESIGN.md section 3.3); conv_tc_launch takes it when the
// grid has more CTAs than SMs.  FSB_CONV_TC2=0 forces the per-tap mode and 1 the window mode (for A/B measurements and tests);
// FSB_CONV_TC2=2 selects the row strip (128 x 1 tiles, Cin % 64 == 0, no statistics), which is slower: its two 50 KB windows
// allow one CTA per SM.
enum ConvTcMode { kPerTap, kWindow, kStrip };
static ConvTcMode conv_tc_mode(const fsb_conv_desc* d) {
  if (d->ksize != 3 || d->stride != 1 || d->dil != 1) return kPerTap;
  const int o = opt(OPT_CONV_TC2);
  if (o == 0) return kPerTap;
  if (o == 2 && d->Cin % 64 == 0 && !(d->flags & FSB_CONV_STATS)) return kStrip;
  return kWindow;
}
bool conv_tc_strip(const fsb_conv_desc* d) { return conv_tc_mode(d) == kStrip; }

// spatial tiles (= CTAs along M = partial statistic rows) of conv_tc
int conv_tc_m_tiles(const fsb_conv_desc* d) {
  if (conv_tc_strip(d)) return ((d->Wo + kTileM - 1) / kTileM) * d->Ho * d->N;
  const int tw = d->Wo >= 16 ? 16 : 8, th = kTileM / tw;
  return ((d->Wo + tw - 1) / tw) * ((d->Ho + th - 1) / th) * d->N;
}

int conv_tc_supported(const fsb_conv_desc* d) {
  if (d->Cin < 16 || (d->x_cstride % 8) != 0) return 0;
  if (!(d->ksize == 1 || d->ksize == 3) || !(d->stride == 1 || d->stride == 2)) return 0;
  return 1;
}

template <int BK, int NT, bool WIN = false>
static int conv_tc_run(dim3 grid, size_t smem_bytes, cudaStream_t stream, const ConvTcUp2Params& q) {
  const bool up2 = q.y_reps > 1;
  const void* kernel = up2 ? reinterpret_cast<const void*>(conv_tc_up2_kernel<BK, NT, WIN>)
                           : reinterpret_cast<const void*>(conv_tc_kernel<BK, NT, WIN>);
  if (int rc = ensure_dyn_smem(kernel, 220 * 1024, "cudaFuncSetAttribute(conv_tc)")) return rc;
  const cudaError_t e = up2 ? launch_kernel(conv_tc_up2_kernel<BK, NT, WIN>, grid, dim3(kThreads), smem_bytes, stream, q)
                            : launch_kernel(conv_tc_kernel<BK, NT, WIN>, grid, dim3(kThreads), smem_bytes, stream, q.p);
  return e == cudaSuccess ? FSB_OK : set_cuda_error(e, "conv_tc launch");
}

template <int BK, bool WIN>
static int conv_tc_run_nt(int n_tile, dim3 grid, size_t smem_bytes, cudaStream_t stream, const ConvTcUp2Params& q) {
  switch (n_tile) {
    case 16: return conv_tc_run<BK, 16, WIN>(grid, smem_bytes, stream, q);
    case 32: return conv_tc_run<BK, 32, WIN>(grid, smem_bytes, stream, q);
    case 48: return conv_tc_run<BK, 48, WIN>(grid, smem_bytes, stream, q);
    case 64: return conv_tc_run<BK, 64, WIN>(grid, smem_bytes, stream, q);
    case 96: return conv_tc_run<BK, 96, WIN>(grid, smem_bytes, stream, q);
    default: return conv_tc_run<BK, 128, WIN>(grid, smem_bytes, stream, q);
  }
}

int conv_tc_launch(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                   void* y, float* stats, cudaStream_t stream, const ConvTcCustom* cu, bool window_ok) {
  const ConvGeom g = conv_geom(d);
  if (cu && (d->stride != 1 || (d->flags & (FSB_CONV_OUT_F32 | FSB_CONV_STATS))))
    return set_error(FSB_ERR_INVALID, "conv_tc: custom tap tables need a stride-1 fp16 problem");
  if (cu && (d->flags & (FSB_CONV_X_DOWN2 | FSB_CONV_Y_UP2)))
    return set_error(FSB_ERR_UNSUPPORTED, "conv_tc: FSB_CONV_X_DOWN2 / FSB_CONV_Y_UP2 cannot be combined with a custom output lattice");
  if ((d->flags & FSB_CONV_X_DOWN2) && d->stride != 1)
    return set_error(FSB_ERR_UNSUPPORTED, "conv_tc: FSB_CONV_X_DOWN2 needs a stride-1 conv");
  if ((d->flags & FSB_CONV_Y_UP2) && (d->flags & (FSB_CONV_STATS | FSB_CONV_OUT_F32)))
    return set_error(FSB_ERR_UNSUPPORTED, "conv_tc: FSB_CONV_Y_UP2 cannot be combined with FSB_CONV_STATS or FSB_CONV_OUT_F32");
  if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(wpacked) & 15))
    return set_error(FSB_ERR_INVALID, "conv_tc: x / wpacked must be 16-byte aligned");
  ConvTcUp2Params q;
  memset(&q, 0, sizeof(q));
  ConvTcParams& p = q.p;
  const ConvTcMode mode = cu ? kPerTap : conv_tc_mode(d);
  const bool strip = mode == kStrip;
  p.taps = cu ? cu->ntaps : g.taps;
  p.Ho = cu ? cu->Ho : d->Ho;
  p.Wo = cu ? cu->Wo : d->Wo;
  p.tw = strip ? kTileM : (p.Wo >= 16 ? 16 : 8);
  p.th = kTileM / p.tw;
  p.tiles_w = (p.Wo + p.tw - 1) / p.tw;
  p.tiles_h = (p.Ho + p.th - 1) / p.th;
  for (int i = 0; i < 9; ++i) p.tap_widx[i] = i;
  p.Cout = d->Cout;
  // Output-channel tiling: N tiles of 16, 32, 48, 64, 96 or 128 channels (the wgmma N of the kernel instance; B boxes past npad
  // rows are zero-filled by TMA and the epilogue stores only channels < Cout): the fewest tiles of <= 128, each the smallest
  // instance that covers its share.  When the spatial tiling alone cannot fill the machine (small maps at 1/16, 1/32
  // resolution), split N further so that more SMs pull operands from L2 in parallel.
  static const int kNt[] = {16, 32, 48, 64, 96, 128};
  const int m_tiles = p.tiles_w * p.tiles_h * d->N;
  int n_tiles = (g.npad + 127) / 128;
  int ni = 0;
  while (kNt[ni] * n_tiles < g.npad) ++ni;
  int n_tile = kNt[ni];
  n_tiles = (g.npad + n_tile - 1) / n_tile;
  const int sms = sm_count();
  // FSB_CONV_NTILE_MIN: smallest N tile the split may produce (default 32).  Splitting N does not shorten a CTA's main loop
  // (every tap and channel chunk is still walked); it spreads the weight loads and the epilogue over more SMs.
  const int nt_min = opt(OPT_CONV_NTILE_MIN) >= 16 ? opt(OPT_CONV_NTILE_MIN) : 32;
  while (m_tiles * n_tiles < sms && ni > 0 && kNt[ni - 1] >= nt_min) {
    n_tile = kNt[--ni];
    n_tiles = (g.npad + n_tile - 1) / n_tile;
  }
  // A grid of at most one CTA per SM is bound by each CTA's latency, not by L2 -> SM traffic; there the window mode's wait for
  // a whole window before the first MMA makes it slower (by 7-19 % on the student's 1/16 and 1/32 maps), so it runs only on
  // larger grids unless FSB_CONV_TC2=1 forces it.  The training convs (BN-train statistics, and the data gradient, whose
  // caller passes window_ok = false) stay per-tap: with them in window mode the distillation step measured slower.
  const bool win = strip || (mode == kWindow && ((window_ok && m_tiles * n_tiles > sms && !(d->flags & FSB_CONV_STATS)) ||
                                                 opt(OPT_CONV_TC2) == 1));
  // window mode: 64-channel chunks for every Cin; a ragged last chunk is zero-filled by TMA on both operands (the input map
  // ends at Cin, the weight map at kpad)
  const int bk = win ? 64 : g.bk;
  p.k_chunks = (g.kpad + bk - 1) / bk;
  if (win) {
    p.win_pitch = p.tw + 2;
    p.win_rows = p.th + 2;
    p.win_stride = (p.win_rows * p.win_pitch * 128 + 1023) / 1024 * 1024;
    p.m_half = 64;
    p.m_grp = 8;
    if (strip) {
      p.win_sbo = 8 * 128;
      p.win_half = 64;
    } else if (p.tw == 16) {
      p.win_sbo = p.win_pitch * 128;
      p.win_half = 8;
      p.m_half = 8;
      p.m_grp = 16;
    } else {
      p.win_sbo = p.win_pitch * 128;
      p.win_half = 8 * p.win_pitch;
    }
  }
  p.y_cstride = d->y_cstride;
  p.flags = d->flags;
  p.scale = scale;
  p.shift = shift;
  p.y = static_cast<__half*>(y);
  p.stats = stats;
  p.stats_C = d->stats_C > 0 ? d->stats_C : d->Cout;
  p.stats_off = d->stats_off;
  if ((d->flags & FSB_CONV_STATS) && stats && (d->stats_off < 0 || d->stats_off + d->Cout > p.stats_C))
    return set_error(FSB_ERR_INVALID, "conv_tc: stats_off + Cout exceeds stats_C");

  const size_t stage_bytes = (win ? 0 : static_cast<size_t>(kTileM) * bk * 2) + static_cast<size_t>(n_tile) * bk * 2;
  const int k_iters = p.taps * p.k_chunks;
  // 128-channel tiles hold 128 accumulator registers per thread: one CTA per SM, give the pipeline (almost) the whole shared
  // memory; the same when the grid has at most one CTA per SM anyway (and for the row strip, whose windows alone take 100 KB).
  // Otherwise keep two CTAs per SM resident.
  const size_t smem_budget = (n_tile == 128 || m_tiles * n_tiles <= sms || strip) ? 200 * 1024 : 100 * 1024;
  const size_t win_bytes = win ? 2 * static_cast<size_t>(p.win_stride) : 0;   // two input windows ahead of the weight ring
  int stages = static_cast<int>((smem_budget - win_bytes) / stage_bytes);
  if (stages < 2) stages = 2;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > k_iters) stages = k_iters;
  p.stages = stages;
  const size_t epi_bytes = n_tile == 16 ? conv_tc_epilogue_bytes<16>() : n_tile == 32 ? conv_tc_epilogue_bytes<32>()
                           : n_tile == 48 ? conv_tc_epilogue_bytes<48>() : n_tile == 64 ? conv_tc_epilogue_bytes<64>()
                           : n_tile == 96 ? conv_tc_epilogue_bytes<96>() : conv_tc_epilogue_bytes<128>();
  size_t smem_bytes = (win_bytes + stage_bytes * stages > epi_bytes ? win_bytes + stage_bytes * stages : epi_bytes) + 1024;
  // ---- TMA-store epilogue: fp16 output whose pixels start on 16 B and whose channel count is a multiple of 8 ----
  // FSB_CONV_Y_UP2: y is the 2Ho x 2Wo map and every output pixel goes to its 2x2 block (nearest x2 folded into the store):
  // four lattice maps, one per (row, column) parity, each with the pixel steps of the full map doubled; the epilogue stores
  // every staged slab to each of them.
  const bool up2 = (d->flags & FSB_CONV_Y_UP2) != 0;
  p.tma_store = 0;
  q.y_reps = 1;
  if (!(d->flags & (FSB_CONV_OUT_F32 | FSB_CONV_STATS)) && d->Cout % 8 == 0 && d->y_cstride % 8 == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0 &&
      n_tile % 8 == 0 && (cu || up2 || opt(OPT_NO_TMA_STORE) <= 0)) {
    const uint64_t ycs = static_cast<uint64_t>(d->y_cstride) * 2;
    uint64_t dims[4] = {static_cast<uint64_t>(d->Cout), static_cast<uint64_t>(d->Wo), static_cast<uint64_t>(d->Ho),
                        static_cast<uint64_t>(d->N)};
    uint64_t str[3] = {ycs, ycs * d->Wo, ycs * d->Wo * d->Ho};
    const uint8_t* ybase[4] = {static_cast<const uint8_t*>(y), nullptr, nullptr, nullptr};
    if (cu) {  // output = a strided sub-lattice (parity plane) of the destination tensor
      ybase[0] = static_cast<const uint8_t*>(cu->y_base);
      for (int i = 0; i < 4; ++i) dims[i] = cu->y_dims[i];
      for (int i = 0; i < 3; ++i) str[i] = cu->y_strides[i];
    }
    if (up2) {
      q.y_reps = 4;
      const uint64_t row = ycs * 2 * d->Wo;  // one row of the 2Ho x 2Wo map
      str[0] = 2 * ycs;
      str[1] = 2 * row;
      str[2] = row * 2 * d->Ho;
      for (int l = 0; l < 4; ++l) ybase[l] = static_cast<const uint8_t*>(y) + (l >> 1) * row + (l & 1) * ycs;
    }
    const uint32_t box64[4] = {64u, static_cast<uint32_t>(p.tw), static_cast<uint32_t>(p.th), 1u};
    p.tail_w = n_tile % 64;
    const uint32_t boxt[4] = {static_cast<uint32_t>(p.tail_w), static_cast<uint32_t>(p.tw), static_cast<uint32_t>(p.th), 1u};
    for (int l = 0; l < q.y_reps; ++l) {
      CUtensorMap* maps = l == 0 ? p.tmap_y : q.tmap_up + 2 * (l - 1);
      int rc = 0;
      if (n_tile >= 64) rc = encode_tiled(&maps[0], ybase[l], 4, dims, str, box64, 128);
      if (!rc && p.tail_w) rc = encode_tiled(&maps[1], ybase[l], 4, dims, str, boxt, 0);
      if (rc) return rc;
      if (n_tile < 64) maps[0] = maps[1];
    }
    p.tma_store = 1;
  }
  if (cu && !p.tma_store) return set_error(FSB_ERR_UNSUPPORTED, "conv_tc: custom output lattice needs the TMA-store epilogue");
  if (up2 && !p.tma_store)
    return set_error(FSB_ERR_UNSUPPORTED, "conv_tc: FSB_CONV_Y_UP2 needs the TMA-store epilogue (fp16 output, Cout and y_cstride "
                                          "multiples of 8, 16-byte aligned y)");

  // ---- A tensor maps ----
  const __half* xb = static_cast<const __half*>(x);
  const uint64_t cs = static_cast<uint64_t>(d->x_cstride) * 2;  // bytes per pixel step
  const uint32_t boxA[4] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(win ? p.win_pitch : p.tw),
                            static_cast<uint32_t>(win ? p.win_rows : p.th), 1u};
  if (d->stride == 1) {
    const uint64_t dims[4] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(d->W), static_cast<uint64_t>(d->H),
                              static_cast<uint64_t>(d->N)};
    // FSB_CONV_X_DOWN2: x is the 2H x 2W map and the conv reads its even rows and columns (nearest /2 folded into the load)
    const bool down2 = (d->flags & FSB_CONV_X_DOWN2) != 0;
    const uint64_t str[3] = {down2 ? 2 * cs : cs, down2 ? 4 * cs * d->W : cs * d->W, down2 ? 4 * cs * d->W * d->H : cs * d->W * d->H};
    int rc = encode_tiled(&p.tmap_a[0], xb, 4, dims, str, boxA, bk * 2);
    if (rc) return rc;
    for (int r = 0; r < d->ksize; ++r)
      for (int s = 0; s < d->ksize; ++s) {
        const int tp = r * d->ksize + s;
        p.tap_map[tp] = 0;
        p.tap_dh[tp] = r * d->dil - d->pad + d->off_h;
        p.tap_dw[tp] = s * d->dil - d->pad + d->off_w;
      }
    if (cu)
      for (int i = 0; i < cu->ntaps; ++i) {
        p.tap_map[i] = 0;
        p.tap_dh[i] = cu->dh[i];
        p.tap_dw[i] = cu->dw[i];
        p.tap_widx[i] = cu->widx[i];
      }
  } else {
    bool used[4] = {false, false, false, false};
    for (int r = 0; r < d->ksize; ++r)
      for (int s = 0; s < d->ksize; ++s) {
        const int tp = r * d->ksize + s;
        const int qh = r * d->dil - d->pad + d->off_h;
        const int qw = s * d->dil - d->pad + d->off_w;
        const int ph = ((qh % 2) + 2) % 2, pw = ((qw % 2) + 2) % 2;
        p.tap_map[tp] = ph * 2 + pw;
        p.tap_dh[tp] = floordiv(qh, 2);
        p.tap_dw[tp] = floordiv(qw, 2);
        used[ph * 2 + pw] = true;
      }
    for (int ph = 0; ph < 2; ++ph)
      for (int pw = 0; pw < 2; ++pw) {
        if (!used[ph * 2 + pw]) continue;
        const int Hp = (d->H - ph + 1) / 2, Wp = (d->W - pw + 1) / 2;
        if (Hp <= 0 || Wp <= 0) return set_error(FSB_ERR_INVALID, "conv_tc: empty parity plane");
        const uint64_t dims[4] = {static_cast<uint64_t>(d->Cin), static_cast<uint64_t>(Wp), static_cast<uint64_t>(Hp),
                                  static_cast<uint64_t>(d->N)};
        const uint64_t str[3] = {2 * cs, 2 * cs * d->W, cs * d->W * d->H};
        const __half* base = xb + (static_cast<size_t>(ph) * d->W + pw) * d->x_cstride;
        int rc = encode_tiled(&p.tmap_a[ph * 2 + pw], base, 4, dims, str, boxA, g.bk * 2);
        if (rc) return rc;
      }
    // prefetch target must be a valid map
    if (!used[0]) p.tmap_a[0] = p.tmap_a[p.tap_map[0]];
  }
  // ---- B tensor map ----
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(g.kpad), static_cast<uint64_t>(g.npad), static_cast<uint64_t>(g.taps)};
    const uint64_t str[2] = {static_cast<uint64_t>(g.kpad) * 2, static_cast<uint64_t>(g.kpad) * g.npad * 2};
    const uint32_t boxB[3] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(n_tile), 1u};
    int rc = encode_tiled(&p.tmap_b, wpacked, 3, dims, str, boxB, bk * 2);
    if (rc) return rc;
  }
  const dim3 grid(static_cast<unsigned>(m_tiles), static_cast<unsigned>(n_tiles));
  if (win) return conv_tc_run_nt<64, true>(n_tile, grid, smem_bytes, stream, q);
  if (g.bk == 64) return conv_tc_run_nt<64, false>(n_tile, grid, smem_bytes, stream, q);
  return conv_tc_run_nt<32, false>(n_tile, grid, smem_bytes, stream, q);
}

}  // namespace fsb
