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

// Tuning / validation switches.  Read from the environment ONCE (first use) and settable through fsb_set_option(); never a
// getenv() on the launch path.  -1 = unset.  The switches marked "no effect" selected conv kernel variants that this sm_90a
// library does not have; their names stay accepted so that existing settings keep working.
enum Opt {
  OPT_CONV_TC2 = 0,      // FSB_CONV_TC2: mode of conv_tc for 3x3 stride-1 convs: 0 = per-tap, 1 = window, 2 = row strip
                         // (default: window on inference convs with more CTAs than SMs, else per-tap)
  OPT_TC2_R,             // FSB_TC2_R: no effect
  OPT_TC2_ASTAGES,       // FSB_TC2_ASTAGES: no effect
  OPT_NO_TMA_STORE,      // FSB_NO_TMA_STORE
  OPT_DGRAD_S2_DIRECT,   // FSB_DGRAD_S2_DIRECT
  OPT_WGRAD_TC,          // FSB_WGRAD_TC: 0 = CUDA-core weight gradient
  OPT_CONV_PERSIST,      // FSB_CONV_PERSIST: no effect
  OPT_PERSIST_OCC,       // FSB_PERSIST_OCC: no effect
  OPT_PERSIST_STAGES,    // FSB_PERSIST_STAGES: no effect
  OPT_UPSAMPLE_V2,       // FSB_UPSAMPLE_V2
  OPT_DETERMINISTIC,     // FSB_DETERMINISTIC: 1 = weight gradients without split-K atomics (bit-reproducible steps)
  OPT_CONV_TC3,          // FSB_CONV_TC3: no effect
  OPT_CONV_TC4,          // FSB_CONV_TC4: no effect
  OPT_CONV_TC5,          // FSB_CONV_TC5: no effect
  OPT_CONV_KSPLIT,       // FSB_CONV_KSPLIT: no effect
  OPT_CONV_NTILE_MIN,    // FSB_CONV_NTILE_MIN: lower bound of the output-channel tile when conv_tc splits N to occupy more SMs (default 32)
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
bool conv_tc_strip(const fsb_conv_desc* d);  // conv_tc runs d in row-strip mode
// window_ok = false keeps a 3x3 stride-1 problem on the per-tap mode unless FSB_CONV_TC2 forces the window mode;
// residency != nullptr launches nothing and stores the CTAs per SM of the instance and shared memory the call would launch with
int conv_tc_launch(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                   void* y, float* stats, cudaStream_t stream, const ConvTcCustom* cu = nullptr, bool window_ok = true,
                   int* residency = nullptr);
int conv_wgrad_tc_supported(const fsb_conv_desc* d, int dy_cstride);
int conv_wgrad_tc_launch(const fsb_conv_desc* d, const void* x, const void* dy, int dcs, float* dw, int64_t so, int64_t si,
                         float gscale, cudaStream_t stream);
int conv_direct_launch(const fsb_conv_desc* d, const void* x, const void* wpacked, const float* scale, const float* shift,
                       void* y, float* stats, cudaStream_t stream);

}  // namespace fsb
