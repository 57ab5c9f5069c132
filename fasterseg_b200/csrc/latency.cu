// latency.cu -- K14: the supernet's expected latency (search/model_search.py:361-475) and its gradient, one launch each.
//
// The plan (built and documented in fasterseg_b200/supernet_latency.py) is an int32 buffer: a 32-slot header, the constants,
// one int4 per MixedOp term {alpha row, in ratio row | -1, out ratio row | -1, offset of its [5][n_w][n_w] latency slice},
// one int4 per instruction {ADD | MUL, operand register, operand register, 0} (instruction i writes register reg_instr + i),
// the latency slices, and two CSR lists: alpha row -> terms, ratio row -> 2 * term + side.
// Registers: constants | beta softmax values (2 per row) | term values | instruction results.
// One CTA: softmaxes and gumbel samples one thread per row, terms one thread each, the program in thread 0 (a few hundred
// dependent scalar ops).  Every sum runs in a fixed order: the result is deterministic.
#include "fsb_internal.h"

namespace fsb {
namespace {

constexpr int kOps = 5;
constexpr int kThreads = 256;
constexpr int kMaxWidths = 16;
enum {
  H_VERSION = 0, H_NW = 1, H_AROWS = 2, H_BROWS = 5, H_RROWS = 7, H_FLAGS = 10, H_TERMS = 11, H_REGS = 12, H_INSTRS = 13, H_OUT = 14,
  H_CONSTS = 15, H_OFF_CONST = 16, H_OFF_TERMS = 17, H_OFF_INSTR = 18, H_OFF_LAT = 19, H_OFF_APTR = 20, H_OFF_AIDX = 21,
  H_OFF_RPTR = 22, H_OFF_RIDX = 23, H_REG_BETA = 24, H_REG_TERM = 25, H_REG_INSTR = 26, H_LEN = 27
};
constexpr int kPlanVersion = 1;
constexpr int F_ALPHA = 1, F_BETA = 2, F_SAMPLED = 4;

struct Arch {
  const float* a[3];
  const float* b[2];
  const float* r[3];
};
struct ArchGrad {
  float* a[3];
  float* b[2];
  float* r[3];
};

// workspace (floats): registers | alpha softmax [RA][5] | soft [RR][n_w] | pi [RR][n_w] | score [RR] | winner [RR] (int)
struct Ws {
  float *reg, *A, *soft, *pi, *score;
  int* win;
};
__host__ __device__ inline int rows_sum(const int* h, int f, int n) {
  int s = 0;
  for (int i = 0; i < n; ++i) s += h[f + i];
  return s;
}
__host__ __device__ inline Ws ws_layout(const int* h, float* base) {
  const int RA = rows_sum(h, H_AROWS, 3), RR = rows_sum(h, H_RROWS, 3), nw = h[H_NW];
  Ws w;
  w.reg = base;
  w.A = w.reg + h[H_REGS];
  w.soft = w.A + RA * kOps;
  w.pi = w.soft + RR * nw;
  w.score = w.pi + RR * nw;
  w.win = reinterpret_cast<int*>(w.score + RR);
  return w;
}
size_t ws_floats(const int* h) {
  return (size_t)h[H_REGS] + (size_t)rows_sum(h, H_AROWS, 3) * kOps + (size_t)rows_sum(h, H_RROWS, 3) * (2 * h[H_NW] + 2);
}

// global row -> (tensor, local row) over `n` tensors with row counts h[f..f+n)
__device__ inline void locate(const int* h, int f, int n, int row, int& t, int& local) {
  t = 0;
  local = row;
  while (t < n - 1 && local >= h[f + t]) local -= h[f + t++];
}

__device__ inline float term_lat(const int* plan, const int4 tm, int k, const int* win, int nw) {
  const int i = tm.y >= 0 ? win[tm.y] : 0, j = tm.z >= 0 ? win[tm.z] : 0;
  return __int_as_float(plan[plan[H_OFF_LAT] + tm.w + (k * nw + i) * nw + j]);
}

__global__ void __launch_bounds__(kThreads)
supernet_latency_fwd_kernel(const int* __restrict__ plan, Arch arch, const float* __restrict__ noise, float* __restrict__ wsbase,
                            float* __restrict__ out) {
  extern __shared__ float sm[];
  const int* h = plan;
  const int nw = h[H_NW], flags = h[H_FLAGS], NR = h[H_REGS], NI = h[H_INSTRS], M = h[H_TERMS];
  const int RA = rows_sum(h, H_AROWS, 3), RB = rows_sum(h, H_BROWS, 2), RR = rows_sum(h, H_RROWS, 3);
  Ws ws = ws_layout(h, wsbase);
  float* reg = sm;
  int4* ins = reinterpret_cast<int4*>(sm + ((NR + 3) & ~3));
  const int tid = threadIdx.x;

  for (int r = tid; r < RA; r += blockDim.x) {      // alphas: softmax per row, or the uniform 1/5 stand-in
    float* A = ws.A + r * kOps;
    if (flags & F_ALPHA) {
      int t, lr;
      locate(h, H_AROWS, 3, r, t, lr);
      const float* p = arch.a[t] + lr * kOps;
      float mx = p[0];
      for (int k = 1; k < kOps; ++k) mx = fmaxf(mx, p[k]);
      float e[kOps], s = 0.f;
      for (int k = 0; k < kOps; ++k) s += (e[k] = expf(p[k] - mx));
      for (int k = 0; k < kOps; ++k) A[k] = e[k] / s;
    } else {
      for (int k = 0; k < kOps; ++k) A[k] = 1.f * (1.f / kOps);
    }
  }
  for (int r = tid; r < RB; r += blockDim.x) {      // betas: 2-way softmax per row, or 1/2
    float* b = reg + h[H_REG_BETA] + 2 * r;
    if (flags & F_BETA) {
      int t, lr;
      locate(h, H_BROWS, 2, r, t, lr);
      const float* p = arch.b[t] + 2 * lr;
      const float mx = fmaxf(p[0], p[1]), e0 = expf(p[0] - mx), e1 = expf(p[1] - mx), s = e0 + e1;
      b[0] = e0 / s;
      b[1] = e1 / s;
    } else {
      b[0] = b[1] = 0.5f;
    }
  }
  for (int r = tid; r < RR; r += blockDim.x) {      // widths: straight-through gumbel sample, or a forced index with score 1
    if (flags & F_SAMPLED) {
      int t, lr;
      locate(h, H_RROWS, 3, r, t, lr);
      const float* p = arch.r[t] + lr * nw;
      const float* u = noise + r * nw;
      float mx = p[0];
      for (int k = 1; k < nw; ++k) mx = fmaxf(mx, p[k]);
      float s = 0.f;
      for (int k = 0; k < nw; ++k) s += expf(p[k] - mx);
      const float lse = logf(s);
      float z[kMaxWidths], zmax = -INFINITY;
      for (int k = 0; k < nw; ++k) {
        ws.pi[r * nw + k] = expf(p[k] - mx) / s;
        const float g = -logf(1e-20f - logf(u[k] + 1e-20f));
        z[k] = (p[k] - mx - lse) + g;                 // log_softmax(p) + gumbel
        zmax = fmaxf(zmax, z[k]);
      }
      float zs = 0.f;
      for (int k = 0; k < nw; ++k) zs += (z[k] = expf(z[k] - zmax));
      int best = 0;
      float bv = -1.f;
      for (int k = 0; k < nw; ++k) {
        const float v = z[k] / zs;
        ws.soft[r * nw + k] = v;
        if (v > bv) bv = v, best = k;                 // first maximum, like torch.max
      }
      ws.win[r] = best;
      ws.score[r] = (1.f - bv) + bv;                 // (one_hot - soft).detach() + soft at the winner
    } else {
      ws.win[r] = static_cast<int>(noise[r]);
      ws.score[r] = 1.f;
    }
  }
  for (int c = tid; c < h[H_CONSTS]; c += blockDim.x) reg[c] = __int_as_float(plan[h[H_OFF_CONST] + c]);
  const int4* gins = reinterpret_cast<const int4*>(plan + h[H_OFF_INSTR]);
  for (int i = tid; i < NI; i += blockDim.x) ins[i] = gins[i];
  __syncthreads();

  const int4* terms = reinterpret_cast<const int4*>(plan + h[H_OFF_TERMS]);
  for (int m = tid; m < M; m += blockDim.x) {       // MixedOp terms: sum_k lat_k * (a_k * s_in * s_out), in the walk's order
    const int4 tm = terms[m];
    const float si = tm.y >= 0 ? ws.score[tm.y] : 1.f, so = tm.z >= 0 ? ws.score[tm.z] : 1.f;
    const float* A = ws.A + tm.x * kOps;
    float acc = 0.f;
    for (int k = 0; k < kOps; ++k) acc = __fadd_rn(acc, __fmul_rn(term_lat(plan, tm, k, ws.win, nw), __fmul_rn(__fmul_rn(A[k], si), so)));
    reg[h[H_REG_TERM] + m] = acc;
  }
  __syncthreads();

  if (tid == 0) {                                   // the recurrence: straight-line program
    float* dst = reg + h[H_REG_INSTR];
    for (int i = 0; i < NI; ++i) {
      const int4 q = ins[i];
      dst[i] = q.x == 0 ? __fadd_rn(reg[q.y], reg[q.z]) : __fmul_rn(reg[q.y], reg[q.z]);
    }
    out[0] = reg[h[H_OUT]];
  }
  __syncthreads();
  for (int i = tid; i < NR; i += blockDim.x) ws.reg[i] = reg[i];
}

__global__ void __launch_bounds__(kThreads)
supernet_latency_bwd_kernel(const int* __restrict__ plan, const float* __restrict__ gout, const float* __restrict__ wsbase, ArchGrad g) {
  extern __shared__ float sm[];
  const int* h = plan;
  const int nw = h[H_NW], flags = h[H_FLAGS], NR = h[H_REGS], NI = h[H_INSTRS];
  const int RA = rows_sum(h, H_AROWS, 3), RB = rows_sum(h, H_BROWS, 2), RR = rows_sum(h, H_RROWS, 3);
  const Ws ws = ws_layout(h, const_cast<float*>(wsbase));
  const int npad = (NR + 3) & ~3;
  float* val = sm;
  float* adj = sm + npad;
  int4* ins = reinterpret_cast<int4*>(sm + 2 * npad);
  const int tid = threadIdx.x;

  for (int i = tid; i < NR; i += blockDim.x) {
    val[i] = ws.reg[i];
    adj[i] = 0.f;
  }
  const int4* gins = reinterpret_cast<const int4*>(plan + h[H_OFF_INSTR]);
  for (int i = tid; i < NI; i += blockDim.x) ins[i] = gins[i];
  __syncthreads();
  if (tid == 0) {                                   // reverse sweep of the program
    adj[h[H_OUT]] = gout[0];
    const int base = h[H_REG_INSTR];
    for (int i = NI - 1; i >= 0; --i) {
      const float d = adj[base + i];
      const int4 q = ins[i];
      if (q.x == 0) {
        adj[q.y] += d;
        adj[q.z] += d;
      } else {
        const float vy = val[q.y], vz = val[q.z];
        adj[q.y] += d * vz;
        adj[q.z] += d * vy;
      }
    }
  }
  __syncthreads();

  if (flags & F_BETA) {
    for (int r = tid; r < RB; r += blockDim.x) {    // 2-way softmax backward, b_0 b_1 (g_0 - g_1): exactly 0 when g_0 == g_1
      int t, lr;
      locate(h, H_BROWS, 2, r, t, lr);
      const int b = h[H_REG_BETA] + 2 * r;
      const float d = val[b] * val[b + 1] * (adj[b] - adj[b + 1]);
      g.b[t][2 * lr] = d;
      g.b[t][2 * lr + 1] = -d;
    }
  }
  const int4* terms = reinterpret_cast<const int4*>(plan + h[H_OFF_TERMS]);
  const int treg = h[H_REG_TERM];
  if (flags & F_ALPHA) {
    const int* ptr = plan + h[H_OFF_APTR];
    const int* idx = plan + h[H_OFF_AIDX];
    for (int r = tid; r < RA; r += blockDim.x) {    // d softmax(alpha row) from every term that uses it, then softmax backward
      float dA[kOps] = {0.f, 0.f, 0.f, 0.f, 0.f};
      for (int e = ptr[r]; e < ptr[r + 1]; ++e) {
        const int m = idx[e];
        const int4 tm = terms[m];
        const float si = tm.y >= 0 ? ws.score[tm.y] : 1.f, so = tm.z >= 0 ? ws.score[tm.z] : 1.f;
        for (int k = 0; k < kOps; ++k) dA[k] += adj[treg + m] * term_lat(plan, tm, k, ws.win, nw) * so * si;
      }
      const float* A = ws.A + r * kOps;
      float dot = 0.f;
      for (int k = 0; k < kOps; ++k) dot += A[k] * dA[k];
      int t, lr;
      locate(h, H_AROWS, 3, r, t, lr);
      for (int k = 0; k < kOps; ++k) g.a[t][lr * kOps + k] = A[k] * (dA[k] - dot);
    }
  }
  if (flags & F_SAMPLED) {
    const int* ptr = plan + h[H_OFF_RPTR];
    const int* idx = plan + h[H_OFF_RIDX];
    for (int r = tid; r < RR; r += blockDim.x) {    // d score from every term side that uses the row, then through the sample
      float dS = 0.f;
      for (int e = ptr[r]; e < ptr[r + 1]; ++e) {
        const int m = idx[e] >> 1, side = idx[e] & 1;
        const int4 tm = terms[m];
        const int other = side ? tm.y : tm.z;
        const float so = other >= 0 ? ws.score[other] : 1.f;
        const float* A = ws.A + tm.x * kOps;
        float s = 0.f;
        for (int k = 0; k < kOps; ++k) s += term_lat(plan, tm, k, ws.win, nw) * A[k];
        dS += adj[treg + m] * s * so;
      }
      // straight-through: d soft = dS at the winner; soft = softmax(z): dz_j = soft_j (dsoft_j - soft_w dS);
      // z = log_softmax(p) + g: dp_l = dz_l - pi_l * sum_j dz_j
      const float* soft = ws.soft + r * nw;
      const float* pi = ws.pi + r * nw;
      const int w = ws.win[r];
      float dz[kMaxWidths], sdz = 0.f;
      for (int k = 0; k < nw; ++k) {
        dz[k] = soft[k] * ((k == w ? dS : 0.f) - soft[w] * dS);
        sdz += dz[k];
      }
      int t, lr;
      locate(h, H_RROWS, 3, r, t, lr);
      for (int k = 0; k < nw; ++k) g.r[t][lr * nw + k] = dz[k] - pi[k] * sdz;
    }
  }
}

int check_plan(const int* h) {
  if (!h) return set_error(FSB_ERR_INVALID, "supernet latency: null plan");
  if (h[H_VERSION] != kPlanVersion) return set_error(FSB_ERR_INVALID, "supernet latency: plan version mismatch");
  if (h[H_NW] < 1 || h[H_NW] > kMaxWidths) return set_error(FSB_ERR_UNSUPPORTED, "supernet latency: 1..16 widths");
  if (h[H_REGS] <= 0 || h[H_INSTRS] < 0 || h[H_OUT] < 0 || h[H_OUT] >= h[H_REGS])
    return set_error(FSB_ERR_INVALID, "supernet latency: bad plan header");
  return FSB_OK;
}

size_t fwd_smem(const int* h) { return (size_t)((h[H_REGS] + 3) & ~3) * 4 + (size_t)h[H_INSTRS] * 16; }
size_t bwd_smem(const int* h) { return (size_t)((h[H_REGS] + 3) & ~3) * 8 + (size_t)h[H_INSTRS] * 16; }

}  // namespace
}  // namespace fsb

using namespace fsb;

extern "C" {

size_t fsb_supernet_latency_workspace_bytes(const int32_t* plan) {
  if (check_plan(plan)) return 0;
  return ws_floats(plan) * sizeof(float);
}

int fsb_supernet_latency_fwd(const int32_t* plan_host, const int32_t* plan, const float* alpha0, const float* alpha1,
                             const float* alpha2, const float* beta1, const float* beta2, const float* ratio0, const float* ratio1,
                             const float* ratio2, const float* noise, float* workspace, float* out, void* stream) {
  if (int rc = check_plan(plan_host)) return rc;
  const int flags = plan_host[H_FLAGS];
  if (!plan || !noise || !workspace || !out) return set_error(FSB_ERR_INVALID, "fsb_supernet_latency_fwd: null pointer");
  if (((flags & F_ALPHA) && !(alpha0 && alpha1 && alpha2)) || ((flags & F_BETA) && !(beta1 && beta2)) ||
      ((flags & F_SAMPLED) && !(ratio0 && ratio1 && ratio2)))
    return set_error(FSB_ERR_INVALID, "fsb_supernet_latency_fwd: null arch parameter");
  const size_t smem = fwd_smem(plan_host);
  if (smem > 48 * 1024) {
    if (smem > 200 * 1024) return set_error(FSB_ERR_UNSUPPORTED, "fsb_supernet_latency_fwd: plan too large");
    if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(supernet_latency_fwd_kernel), (int)smem, "fsb_supernet_latency_fwd")) return rc;
  }
  Arch a{{alpha0, alpha1, alpha2}, {beta1, beta2}, {ratio0, ratio1, ratio2}};
  supernet_latency_fwd_kernel<<<1, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(plan, a, noise, workspace, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, "fsb_supernet_latency_fwd launch");
  return FSB_OK;
}

int fsb_supernet_latency_bwd(const int32_t* plan_host, const int32_t* plan, const float* gout, const float* workspace, float* dalpha0,
                             float* dalpha1, float* dalpha2, float* dbeta1, float* dbeta2, float* dratio0, float* dratio1, float* dratio2,
                             void* stream) {
  if (int rc = check_plan(plan_host)) return rc;
  const int flags = plan_host[H_FLAGS];
  if (!plan || !gout || !workspace) return set_error(FSB_ERR_INVALID, "fsb_supernet_latency_bwd: null pointer");
  if (((flags & F_ALPHA) && !(dalpha0 && dalpha1 && dalpha2)) || ((flags & F_BETA) && !(dbeta1 && dbeta2)) ||
      ((flags & F_SAMPLED) && !(dratio0 && dratio1 && dratio2)))
    return set_error(FSB_ERR_INVALID, "fsb_supernet_latency_bwd: null gradient");
  const size_t smem = bwd_smem(plan_host);
  if (smem > 48 * 1024) {
    if (smem > 200 * 1024) return set_error(FSB_ERR_UNSUPPORTED, "fsb_supernet_latency_bwd: plan too large");
    if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(supernet_latency_bwd_kernel), (int)smem, "fsb_supernet_latency_bwd")) return rc;
  }
  ArchGrad g{{dalpha0, dalpha1, dalpha2}, {dbeta1, dbeta2}, {dratio0, dratio1, dratio2}};
  supernet_latency_bwd_kernel<<<1, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(plan, gout, workspace, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, "fsb_supernet_latency_bwd launch");
  return FSB_OK;
}

}  // extern "C"
