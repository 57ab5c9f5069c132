// fsb_internal.h -- declarations shared between the translation units of libfsb200.so (not part of the ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/fsb200.h"

namespace fsb {

int set_error(int code, const char* msg);
int set_cuda_error(cudaError_t e, const char* where);

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();
// cuTensorMapEncodeTiled of an fp16 tensor (rank <= 5, dims / strides innermost first, strides in bytes) with a 128/64/32-byte or
// no swizzle; errors land in fsb_last_error_string
int encode_tiled(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes);

// derived geometry shared by the packer and the kernels
struct ConvGeom {
  int taps;     // ksize^2
  int bk;       // K chunk (channels per TMA box / smem row): 64 if Cin % 64 == 0 else 32
  int kpad;     // Cin rounded up to bk
  int npad;     // Cout rounded up to 16 (rows of the packed weight matrix per tap)
};
ConvGeom conv_geom(const fsb_conv_desc* d);

bool pdl_enabled();
int sm_count();
int stat_rows(int64_t pixels);  // partial statistic rows of the CUDA-core kernels (bn.cu)

// Tuning / validation switches.  Read from the environment ONCE (first use) and settable through fsb_set_option(); never a
// getenv() on the launch path.  -1 = unset.
enum Opt {
  OPT_CONV_TC2 = 0,      // FSB_CONV_TC2: mode of conv_tc for 3x3 stride-1 convs: 0 = per-tap, 1 = window
                         // (default: window on inference convs with more CTAs than SMs, else per-tap)
  OPT_DGRAD_S2_DIRECT,   // FSB_DGRAD_S2_DIRECT
  OPT_WGRAD_TC,          // FSB_WGRAD_TC: 0 = CUDA-core weight gradient
  OPT_UPSAMPLE_V2,       // FSB_UPSAMPLE_V2
  OPT_DETERMINISTIC,     // FSB_DETERMINISTIC: 1 = weight gradients without split-K atomics (bit-reproducible steps)
  OPT_COUNT
};
int opt(Opt o);

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute: remember it per (kernel, device), not per process
int ensure_dyn_smem(const void* kernel, int bytes, const char* what);

// Launch with (optionally) the programmatic-dependent-launch attribute; every kernel of this library calls
// pdl_launch_dependents() at entry and pdl_wait() before its first dependent global access.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// launch + remember the error in a thread-local that the following cudaGetLastError()-style check picks up
extern thread_local cudaError_t g_launch_err;
#define FSB_LAUNCH(kernel, grid, block, smem, stream, ...) \
  (::fsb::g_launch_err = ::fsb::launch_kernel(kernel, grid, block, smem, stream, __VA_ARGS__))
inline cudaError_t last_launch_error() {
  cudaError_t e = g_launch_err;
  g_launch_err = cudaSuccess;
  if (e == cudaSuccess) e = cudaGetLastError();
  return e;
}

// Generalised launch of the per-tap kernel: arbitrary tap subset / offsets / weight-slice indices and an output written
// to a strided sub-lattice of the destination through the TMA-store tensor map (used by the stride-2 data gradient).
struct ConvTcCustom {
  int ntaps;
  int dh[9], dw[9], widx[9];
  int Ho, Wo;             // extent of the output lattice (tiling)
  const void* y_base;     // address of lattice point (n=0, 0, 0, c=0)
  uint64_t y_dims[4];     // {C, Wl, Hl, N}
  uint64_t y_strides[3];  // bytes: lattice step in W, in H, image
};
int conv_tc_supported(const fsb_conv_desc* d);

// Every decision of one conv launch, taken from the descriptor alone (conv_plan reads no data pointer and makes no CUDA call
// but sm_count()).  The launch, the statistics-row, kernel-id and residency queries and the fused BN-train forward all read it.
struct ConvPlan {
  int rc;                  // FSB_OK, or the error a launch of this descriptor returns; the fields below are filled either way
  bool direct;             // CUDA-core direct kernel (FSB_CONV_FORCE_DIRECT, or a problem conv_tc cannot run); the rest is conv_tc's
  int stat_rows;           // partial statistic rows written with FSB_CONV_STATS: stat_rows(N * Ho * Wo) direct, m_tiles on conv_tc
  bool win;                // window mode (one halo window per 64-channel chunk) instead of per-tap
  bool up2;                // FSB_CONV_Y_UP2: the instance that also stores the other three 2x2 lattices
  int taps, Ho, Wo;        // taps and output extent of the tiling (a custom lattice's own)
  int tw, th;              // 128-pixel tile: 16 x 8, or 8 x 16 when Wo < 16
  int tiles_w, tiles_h, m_tiles;
  int n_tile, n_tiles;     // output channels per CTA (the instance's NT) and CTAs along N
  int bk, k_chunks;        // channels per K chunk (the instance's BK) and chunks per tap
  int win_pitch, win_rows, win_sbo, win_half, win_stride, m_half, m_grp;  // window geometry, see ConvTcParams (conv_tc.cu)
  int res, stages;         // CTAs per SM the shared memory is sized for, depth of the stage ring
  size_t smem;             // dynamic shared memory of the launch
};
// window_ok = false keeps a 3x3 stride-1 problem on the per-tap mode unless FSB_CONV_TC2 forces the window mode; cu (custom tap
// tables) always runs per-tap
ConvPlan conv_plan(const fsb_conv_desc* d, const ConvTcCustom* cu = nullptr, bool window_ok = true);
// Largest output extent (rows or columns) at which a bilinear /2 of it is local to 2x2 blocks and an exact x2 upsample of
// half of it reads at most 3 x 3 source pixels per 2x2 output block: checked for every even extent up to here with the fp32
// index rule of src_index (fsb_common.cuh, tests/test_resize_fusion_cpu.py).  At 4164 the fp32 rounding of src already moves a
// /2 footprint out of its block.
constexpr int kBilinearLocalMax = 4096;

// second output of fsb_conv_fwd_half: bilinear(y, (Ho / 2, Wo / 2), align_corners=True), NHWC fp16 with pixel stride cstride
struct ConvHalfOut {
  void* y;
  int cstride;
};
// launch conv_tc as planned (plan = conv_plan(d, cu, ...), not direct); half: also store the /2 output (even Ho, Wo)
int conv_tc_launch(const ConvPlan& plan, const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale,
                   const float* shift, void* y, float* stats, cudaStream_t stream, const ConvTcCustom* cu = nullptr,
                   const ConvHalfOut* half = nullptr);
// CTAs per SM of the planned conv_tc launch, from the CUDA occupancy calculator; launches nothing
int conv_tc_occupancy(const ConvPlan& plan);
int conv_wgrad_tc_supported(const fsb_conv_desc* d, int dy_cstride);
int conv_wgrad_tc_launch(const fsb_conv_desc* d, const void* x, const void* dy, int dcs, float* dw, int64_t so, int64_t si,
                         int accumulate, float gscale, cudaStream_t stream);
int zero_wgrad_launch(const fsb_conv_desc* d, float* dw, int64_t so, int64_t si, cudaStream_t stream);
int conv_direct_launch(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                       void* y, float* stats, cudaStream_t stream);

}  // namespace fsb
