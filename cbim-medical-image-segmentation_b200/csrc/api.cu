// api.cu — C-ABI entry points that dispatch between the CUDA-core and tensor-core (wgmma) conv paths, plus
// version / error plumbing.  No CPU fallback exists anywhere in this library: an unsupported
// shape or a non-sm_90 device is a hard error (SURVEY.md §8b "Errors").
#include "common.cuh"
#include "conv_args.h"
#include <stdio.h>
#include <string.h>

thread_local char g_b200seg_cuda_err[256] = "";

int b200seg_record_cuda(cudaError_t e, const char* what) {
  snprintf(g_b200seg_cuda_err, sizeof(g_b200seg_cuda_err), "%s: %s", what, cudaGetErrorString(e));
  return B200SEG_ECUDA;
}

extern "C" int b200seg_version(void) { return B200SEG_VERSION; }

extern "C" const char* b200seg_strerror(int code) {
  switch (code) {
    case B200SEG_OK: return "ok";
    case B200SEG_EINVAL: return "invalid argument";
    case B200SEG_EUNSUPPORTED: return "shape/dtype not supported by the requested algorithm";
    case B200SEG_ECUDA: return "CUDA runtime error";
    case B200SEG_ENODEVICE: return "device is not sm_90 (H100); this library has no fallback path";
    default: return "unknown error";
  }
}

extern "C" const char* b200seg_last_cuda_error(void) { return g_b200seg_cuda_err; }

extern "C" int b200seg_check_device(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { b200seg_record_cuda(e, "cudaGetDevice"); return B200SEG_ENODEVICE; }
  int major = 0, minor = 0;
  e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (e != cudaSuccess) { b200seg_record_cuda(e, "cudaDeviceGetAttribute"); return B200SEG_ENODEVICE; }
  return (major == 9 && minor == 0) ? B200SEG_OK : B200SEG_ENODEVICE;      // the library holds sm_90a code only
}

extern "C" int b200seg_conv3d_algo(int Cin, int Cout, int kd, int kh, int kw, int dtype, int B) {
  // the same batch limits as conv3d_fwd_tc_supported, so every shape routed here runs on the tensor cores with or
  // without fused statistics / dgrad mode
  if (dtype == B200SEG_F16 && conv3d_tc_shape_ok(Cin, Cout, kd, kh, kw, dtype) && B * Cin <= 4096 && B * Cout <= 8192)
    return B200SEG_ALGO_TC;
  return B200SEG_ALGO_DIRECT;
}

// The fp32 shapes the tensor-core kernel runs on TF32 operands: the kernel-size and batch limits of the fp16 rule, with
// the TF32 channel table (Cin a multiple of 8, Cout of 16).  The caller decides whether TF32 is wanted at all.
extern "C" int b200seg_conv3d_algo_tf32(int Cin, int Cout, int kd, int kh, int kw, int B) {
  if (conv3d_tc_shape_ok(Cin, Cout, kd, kh, kw, B200SEG_F32) && B * Cin <= 4096 && B * Cout <= 8192) return B200SEG_ALGO_TC_TF32;
  return B200SEG_ALGO_DIRECT;
}

// TC runs fp16 operands and TC_TF32 fp32 storage on TF32 operands; any other pairing is a caller error
static int fwd_tc(const ConvArgs& a, int dtype, int algo, cudaStream_t st) {
  if ((algo == B200SEG_ALGO_TC) != (dtype == B200SEG_F16)) return B200SEG_EUNSUPPORTED;
  return conv3d_fwd_tc(a, dtype, st);
}

extern "C" int b200seg_conv3d_fwd(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                                  const void* w_packed, const float* bias, const void* residual, int r_ld,
                                  int r_coff, void* y, int y_ld, int y_coff, double* y_stats,
                                  const void* dgrad_x, int dx_ld, int dx_coff, const double* dgrad_stats,
                                  float dgrad_eps, int dgrad_act, int B, int D, int H, int W, int Cin, int Cout,
                                  int kd, int kh, int kw, int dtype, int algo, void* stream) {
  if (!x || !w_packed || !y || B <= 0 || D <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return B200SEG_EINVAL;
  if (kd <= 0 || kh <= 0 || kw <= 0 || !(kd & 1) || !(kh & 1) || !(kw & 1)) return B200SEG_EUNSUPPORTED;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  if (dgrad_x && !dgrad_stats) return B200SEG_EINVAL;
  if (dgrad_x && (residual || bias)) return B200SEG_EINVAL;
  ConvArgs a{x, x_ld, x_coff, x_stats, eps, act, w_packed, bias, residual, r_ld, r_coff, y, y_ld, y_coff, y_stats,
             dgrad_x, dx_ld, dx_coff, dgrad_stats, dgrad_eps, dgrad_act, B, D, H, W, Cin, Cout, kd, kh, kw};
  cudaStream_t st = as_stream(stream);
  // the packed-weight layout differs per algorithm, so the caller must name one (b200seg_conv3d_algo)
  if (algo == B200SEG_ALGO_TC || algo == B200SEG_ALGO_TC_TF32) return fwd_tc(a, dtype, algo, st);
  if (algo != B200SEG_ALGO_DIRECT) return B200SEG_EINVAL;
  {
    const int rc = conv3d_fwd_small(a, dtype, st);      // HBM-bound special cases (stem, classifier head)
    if (rc != B200SEG_EUNSUPPORTED) return rc;
  }
  return conv3d_fwd_direct(a, dtype, st);
}

// Per-channel (BatchNorm) mode: x enters as act(x*s[c] + t[c]) from the [Cin][2] table x_affine (nullptr: act(x)).  The
// table is one row for the whole batch, so the tensor-core limits are those of B = 1 (b200seg_conv3d_algo(..., 1)).
extern "C" int b200seg_conv3d_fwd_pc(const void* x, int x_ld, int x_coff, const float* x_affine, int act,
                                     const void* w_packed, const float* bias, const void* residual, int r_ld, int r_coff,
                                     void* y, int y_ld, int y_coff, double* y_stats, int B, int D, int H, int W,
                                     int Cin, int Cout, int kd, int kh, int kw, int dtype, int algo, void* stream) {
  if (!x || !w_packed || !y || B <= 0 || D <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return B200SEG_EINVAL;
  if (kd <= 0 || kh <= 0 || kw <= 0 || !(kd & 1) || !(kh & 1) || !(kw & 1)) return B200SEG_EUNSUPPORTED;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  ConvArgs a{x, x_ld, x_coff, nullptr, 0.f, act, w_packed, bias, residual, r_ld, r_coff, y, y_ld, y_coff, y_stats,
             nullptr, 0, 0, nullptr, 0.f, 0, B, D, H, W, Cin, Cout, kd, kh, kw, x_affine, 1};
  cudaStream_t st = as_stream(stream);
  if (algo == B200SEG_ALGO_TC || algo == B200SEG_ALGO_TC_TF32) return fwd_tc(a, dtype, algo, st);
  if (algo != B200SEG_ALGO_DIRECT) return B200SEG_EINVAL;
  {
    const int rc = conv3d_fwd_small(a, dtype, st);
    if (rc != B200SEG_EUNSUPPORTED) return rc;
  }
  return conv3d_fwd_direct(a, dtype, st);
}


// ---- bias gradient db[c] += sum_v dy[v][c] as its own column-sum pass, so that convolutions / Linears WITH a bias
// (every nn.Linear of SwinUNETR: qkv, proj, fc1, fc2 — 32 per step) can take the tensor-core weight-gradient kernel, which has
// no bias path.  HBM-bound: dy is read once (16-byte loads), block partials in shared memory, one slice of partials per
// block column, summed over the blocks in a fixed order (add_slices).
namespace {
constexpr int kBgThreads = 256, kBgChan = 512;      // channels per block column (grid.y)
template <typename T>
__global__ void __launch_bounds__(kBgThreads) bias_grad_kernel(const T* __restrict__ dy, int ld, int coff, float* __restrict__ part,
                                                               int64_t nvox, int C, int64_t vpb) {
  __shared__ float sm[kBgThreads * 8];
  const int c0 = blockIdx.y * kBgChan, cn = (C - c0 < kBgChan) ? C - c0 : kBgChan;
  const int cpv = cn / 8, vpp = kBgThreads / cpv, cchunk = threadIdx.x % cpv, vloc = threadIdx.x / cpv;
  const bool active = vloc < vpp;
  const int64_t v0 = (int64_t)blockIdx.x * vpb, v1 = (v0 + vpb < nvox) ? v0 + vpb : nvox;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (active) {
    const T* p = dy + coff + c0 + cchunk * 8;
    for (int64_t v = v0 + vloc; v < v1; v += vpp) {
      float a[8];
      ld8<T>(p + v * ld, a);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += a[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm[threadIdx.x * 8 + i] = active ? acc[i] : 0.f;
  __syncthreads();
  for (int o = threadIdx.x; o < cn; o += kBgThreads) {
    float s = 0.f;
    for (int vl = 0; vl < vpp; ++vl) s += sm[(vl * cpv + o / 8) * 8 + (o & 7)];
    part[(int64_t)blockIdx.x * C + c0 + o] = s;
  }
}

dim3 bias_grad_grid(const WgradArgs& a, int64_t& vpb) {
  const int64_t nvox = (int64_t)a.B * a.D * a.H * a.W;
  int64_t blocks = (B200SEG_NUM_SMS * 4) / ((a.Cout + kBgChan - 1) / kBgChan);
  if (blocks < 1) blocks = 1;
  vpb = (nvox + blocks - 1) / blocks;
  if (vpb < 64) vpb = 64;
  return dim3(ceil_div(nvox, vpb), (a.Cout + kBgChan - 1) / kBgChan);
}

size_t bias_grad_workspace(const WgradArgs& a) {
  int64_t vpb;
  return (size_t)bias_grad_grid(a, vpb).x * a.Cout * sizeof(float);
}

// part: bias_grad_workspace(a) bytes
int launch_bias_grad(const WgradArgs& a, int dtype, float* part, cudaStream_t st) {
  const int64_t nvox = (int64_t)a.B * a.D * a.H * a.W;
  int64_t vpb;
  const dim3 grid = bias_grad_grid(a, vpb);
  if (dtype == B200SEG_F16) bias_grad_kernel<__half><<<grid, kBgThreads, 0, st>>>((const __half*)a.dy, a.dy_ld, a.dy_coff, part, nvox, a.Cout, vpb);
  else bias_grad_kernel<float><<<grid, kBgThreads, 0, st>>>((const float*)a.dy, a.dy_ld, a.dy_coff, part, nvox, a.Cout, vpb);
  B200_CHECK_LAUNCH("bias_grad_kernel");
  return add_slices(part, a.Cout, (int)grid.x, a.dbias, a.Cout, st);
}

size_t align16(size_t n) { return (n + 15) / 16 * 16; }
}  // namespace

static int wgrad_args(WgradArgs& a, const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                      const void* dy, int dy_ld, int dy_coff, float* dw, float* dbias, int B, int D, int H, int W,
                      int Cin, int Cout, int kd, int kh, int kw, int dtype) {
  if (B <= 0 || D <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return B200SEG_EINVAL;
  if (kd <= 0 || kh <= 0 || kw <= 0 || !(kd & 1) || !(kh & 1) || !(kw & 1)) return B200SEG_EUNSUPPORTED;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  a = WgradArgs{x, x_ld, x_coff, x_stats, eps, act, dy, dy_ld, dy_coff, dw, dbias, B, D, H, W, Cin, Cout, kd, kh, kw, 0};
  return B200SEG_OK;
}

static size_t wgrad_workspace(const WgradArgs& a, int dtype, int algo) {
  // covers every path b200seg_conv3d_wgrad can take for this shape: the real tensors' alignment (the placeholders of
  // the callers are aligned) can only rule the tensor-core path out, and then the special kernel or the CUDA-core path runs
  if (algo == B200SEG_ALGO_DIRECT) return 0;
  if (algo == B200SEG_ALGO_TC) return conv3d_wgrad_tc_supported(a, dtype) ? conv3d_wgrad_tc_workspace(a) : 0;
  size_t ws = conv3d_wgrad_small_workspace(a), tc = 0;
  if (conv3d_wgrad_tc_supported(a, dtype)) tc = conv3d_wgrad_tc_workspace(a);
  else if (a.dbias && a.Cout % 8 == 0) {
    WgradArgs nb = a;
    nb.dbias = nullptr;
    if (conv3d_wgrad_tc_supported(nb, dtype)) tc = align16(conv3d_wgrad_tc_workspace(nb)) + bias_grad_workspace(a);
  }
  return tc > ws ? tc : ws;
}

extern "C" size_t b200seg_conv3d_wgrad_workspace(int x_ld, int x_coff, int normalised, int dy_ld, int dy_coff,
                                                 int want_bias, int B, int D, int H, int W, int Cin, int Cout,
                                                 int kd, int kh, int kw, int dtype, int algo) {
  WgradArgs a;
  static const double dummy_stats = 0.0;
  static float dummy_bias = 0.f;
  // 16-byte aligned placeholders stand in for the tensors (only shapes/strides decide)
  if (wgrad_args(a, (const void*)16, x_ld, x_coff, normalised ? &dummy_stats : nullptr, 1e-4f, normalised ? 1 : 0,
                 (const void*)16, dy_ld, dy_coff, (float*)16, want_bias ? &dummy_bias : nullptr, B, D, H, W, Cin, Cout,
                 kd, kh, kw, dtype)) return 0;
  return wgrad_workspace(a, dtype, algo);
}

extern "C" size_t b200seg_conv3d_wgrad_pc_workspace(int x_ld, int x_coff, int transformed, int dy_ld, int dy_coff,
                                                    int want_bias, int B, int D, int H, int W, int Cin, int Cout,
                                                    int kd, int kh, int kw, int dtype, int algo) {
  WgradArgs a;
  static const float dummy_affine[2] = {1.f, 0.f};
  static float dummy_bias = 0.f;
  if (wgrad_args(a, (const void*)16, x_ld, x_coff, nullptr, 0.f, transformed ? 1 : 0, (const void*)16, dy_ld, dy_coff,
                 (float*)16, want_bias ? &dummy_bias : nullptr, B, D, H, W, Cin, Cout, kd, kh, kw, dtype)) return 0;
  a.x_affine = transformed ? dummy_affine : nullptr;
  a.per_channel = 1;
  return wgrad_workspace(a, dtype, algo);
}

static int wgrad_dispatch(WgradArgs& a, int dtype, int algo, void* workspace, size_t ws_bytes, cudaStream_t st) {
  int rc;
  if (algo == B200SEG_ALGO_TC) return conv3d_wgrad_tc(a, dtype, workspace, ws_bytes, st);
  if (algo == B200SEG_ALGO_AUTO && conv3d_wgrad_tc_supported(a, dtype))
    return conv3d_wgrad_tc(a, dtype, workspace, ws_bytes, st);
  if (algo != B200SEG_ALGO_AUTO && algo != B200SEG_ALGO_DIRECT) return B200SEG_EINVAL;
  if (algo == B200SEG_ALGO_AUTO && a.dbias && a.Cout % 8 == 0) {
    // the tensor-core kernel has no bias path: take the bias gradient in its own pass and let it do the weight gradient.
    // Ahead of the special kernels on purpose (tools/head_wgrad_ab.py compares the two for the 8- / 16-class 1x1x1
    // heads); Cout = 4 and the Cin = 1 stems do not qualify
    WgradArgs nb = a;
    nb.dbias = nullptr;
    if (conv3d_wgrad_tc_supported(nb, dtype)) {
      const size_t tc_ws = align16(conv3d_wgrad_tc_workspace(nb)), need = tc_ws + bias_grad_workspace(a);
      if (!workspace || ws_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15)) return B200SEG_EINVAL;
      rc = launch_bias_grad(a, dtype, reinterpret_cast<float*>(static_cast<char*>(workspace) + tc_ws), st);
      if (rc) return rc;
      return conv3d_wgrad_tc(nb, dtype, tc_ws ? workspace : nullptr, tc_ws, st);
    }
  }
  if (algo == B200SEG_ALGO_AUTO) {
    if (ws_bytes < conv3d_wgrad_small_workspace(a)) return B200SEG_EINVAL;
    a.part = reinterpret_cast<float*>(workspace);
    rc = conv3d_wgrad_small(a, dtype, st);
    if (rc != B200SEG_EUNSUPPORTED) return rc;
  }
  return conv3d_wgrad_direct(a, dtype, st);
}

extern "C" int b200seg_conv3d_wgrad(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                                    const void* dy, int dy_ld, int dy_coff, float* dw, float* dbias, int B, int D,
                                    int H, int W, int Cin, int Cout, int kd, int kh, int kw, int dtype, int algo,
                                    void* workspace, size_t ws_bytes, void* stream) {
  if (!x || !dy || !dw) return B200SEG_EINVAL;
  WgradArgs a;
  int rc = wgrad_args(a, x, x_ld, x_coff, x_stats, eps, act, dy, dy_ld, dy_coff, dw, dbias, B, D, H, W, Cin, Cout, kd, kh, kw, dtype);
  if (rc) return rc;
  return wgrad_dispatch(a, dtype, algo, workspace, ws_bytes, as_stream(stream));
}

// Per-channel (BatchNorm) mode of the weight gradient: x enters as act(x*s[c] + t[c]) (see b200seg_conv3d_fwd_pc).
extern "C" int b200seg_conv3d_wgrad_pc(const void* x, int x_ld, int x_coff, const float* x_affine, int act,
                                       const void* dy, int dy_ld, int dy_coff, float* dw, float* dbias, int B, int D,
                                       int H, int W, int Cin, int Cout, int kd, int kh, int kw, int dtype, int algo,
                                       void* workspace, size_t ws_bytes, void* stream) {
  if (!x || !dy || !dw) return B200SEG_EINVAL;
  WgradArgs a;
  int rc = wgrad_args(a, x, x_ld, x_coff, nullptr, 0.f, act, dy, dy_ld, dy_coff, dw, dbias, B, D, H, W, Cin, Cout, kd, kh, kw, dtype);
  if (rc) return rc;
  a.x_affine = x_affine;
  a.per_channel = 1;
  return wgrad_dispatch(a, dtype, algo, workspace, ws_bytes, as_stream(stream));
}
