// conv_args.h — argument blocks shared by the direct and tensor-core (wgmma) conv implementations.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

struct ConvArgs {
  const void* x; int x_ld, x_coff;
  const double* x_stats; float eps; int act;
  const void* w; const float* bias;
  const void* res; int r_ld, r_coff;
  void* y; int y_ld, y_coff; double* y_stats;
  const void* gx; int gx_ld, gx_coff; const double* g_stats; float g_eps; int g_act;
  int B, D, H, W, Cin, Cout, kd, kh, kw;
  // Per-channel input transform (BatchNorm): x is replaced by act(x*s[c] + t[c]) from the [Cin][2] {s, t} table
  // x_affine (nullptr: act(x) only).  In this mode x_stats and the data-gradient mask are not used, and the shared
  // table is [Cin] for any batch size.
  const float* x_affine; int per_channel;
};

struct WgradArgs {
  const void* x; int x_ld, x_coff; const double* x_stats; float eps; int act;
  const void* dy; int dy_ld, dy_coff;
  float* dw; float* dbias;
  int B, D, H, W, Cin, Cout, kd, kh, kw;
  int vox_per_block;
  float* part;         // per-block partial slices (conv3d_wgrad_small_workspace bytes), summed in block order
  const float* x_affine; int per_channel;     // as in ConvArgs
};

int conv3d_fwd_direct(const ConvArgs& a, int dtype, cudaStream_t st);
int conv3d_wgrad_direct(const WgradArgs& a, int dtype, cudaStream_t st);
// HBM-bound special cases (Cin=1 stem, 1x1x1 head); EUNSUPPORTED when the shape is not one of them
int conv3d_wgrad_small(const WgradArgs& a, int dtype, cudaStream_t st);
size_t conv3d_wgrad_small_workspace(const WgradArgs& a);      // 0 when the shape is not a special case
// dst[i] += sum over s = 0 .. S-1 of part[s * stride + i] (i < n), in that order: the fixed-order end of every
// weight-gradient reduction that is split over blocks, so the result is the same on every run
int add_slices(const float* part, int64_t stride, int S, float* dst, int64_t n, cudaStream_t st);
int conv3d_fwd_small(const ConvArgs& a, int dtype, cudaStream_t st);
// tensor-core paths (conv_tc.cu / wgrad_tc.cu); return B200SEG_EUNSUPPORTED when the shape does not qualify
int conv3d_fwd_tc(const ConvArgs& a, int dtype, cudaStream_t st);
int conv3d_wgrad_tc(const WgradArgs& a, int dtype, void* workspace, size_t ws_bytes, cudaStream_t st);
size_t conv3d_wgrad_tc_workspace(const WgradArgs& a);
bool conv3d_fwd_tc_supported(const ConvArgs& a, int dtype);
bool conv3d_wgrad_tc_supported(const WgradArgs& a, int dtype);

// ---- tensor-core tiling choices shared by the packer and the kernels
// N tile (output channels per CTA tile): whole Cout when <=128, else the largest even split.  128 columns = 64 fp32
// accumulator registers per thread of each wgmma warpgroup.
__host__ __device__ static inline int tc_pick_nt(int Cout) {
  if (Cout % 16) return 0;
  if (Cout <= 128) return Cout;
  for (int t = (Cout + 127) / 128; t <= 32; ++t)
    if (Cout % t == 0 && (Cout / t) % 16 == 0 && Cout / t <= 128) return Cout / t;
  return 0;
}
// K chunk (input channels per staged halo tile): largest multiple of 16 dividing Cin, <= 64.
__host__ __device__ static inline int tc_pick_kc(int Cin) {
  if (Cin % 16) return 0;
  for (int kc = 64; kc >= 16; kc -= 16)
    if (Cin % kc == 0) return kc;
  return 0;
}
bool conv3d_tc_shape_ok(int Cin, int Cout, int kd, int kh, int kw, int dtype);
