// batchnorm.cu — BatchNorm2d (model/dim2/conv_layers.py:21-94) around the per-channel mode of the convolutions.
//
// The convolutions never see a BatchNorm tensor: the producing kernel's epilogue writes fp64 {sum x, sum x^2} per
// (sample, channel), the forward fold turns those sums into one {s, t} table per channel (and updates the running
// statistics), and the consuming convolution's loader applies act(x*s + t) (b200seg_conv3d_fwd_pc).  The backward runs
// on the raw data gradient: one reduction pass for sum dz and sum dz*xhat per channel, a fold to dgamma / dbeta and
// per-channel coefficients, and one elementwise pass for dx.
//
// Tables (all fp32, channel-major):
//   table      [C][2]  {s, t}            act(x*s + t) is the activation the next layer reads
//   mean_rstd  [C][2]  {mean, rstd}      the statistics the table was made from (batch or running)
//   coef       [C][4]  {a, b, mean, k}   dx = a*dz + b*(x - mean) + k
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

__global__ void bn_fwd_fold_kernel(const double* __restrict__ sums, int nb, int C, double count,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* running_mean, float* running_var, int64_t* num_batches_tracked,
                                   float momentum, float eps, int training, float* __restrict__ table,
                                   float* __restrict__ mean_rstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (training && c == 0 && num_batches_tracked) *num_batches_tracked += 1;
  if (c >= C) return;
  double mean, var;
  if (training) {
    double s = 0.0, q = 0.0;
    for (int b = 0; b < nb; ++b) { s += sums[((int64_t)b * C + c) * 2]; q += sums[((int64_t)b * C + c) * 2 + 1]; }
    mean = s / count;
    var = q / count - mean * mean;
    if (var < 0.0) var = 0.0;
    // torch updates the running variance with the unbiased estimate
    running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + momentum * mean);
    running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + momentum * var * count / (count - 1.0));
  } else {
    mean = running_mean[c];
    var = running_var[c];
  }
  const double rstd = 1.0 / sqrt(var + (double)eps);
  const double s = (double)gamma[c] * rstd;
  table[2 * c] = (float)s;
  table[2 * c + 1] = (float)((double)beta[c] - mean * s);
  mean_rstd[2 * c] = (float)mean;
  mean_rstd[2 * c + 1] = (float)rstd;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bn_apply_kernel(const T* __restrict__ x, int x_ld, int x_coff,
                                                            const float* __restrict__ table, int act, T* __restrict__ y,
                                                            int y_ld, int y_coff, int64_t nvox, int C) {
  const int cpv = C / 8;
  const int64_t n = nvox * cpv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / cpv;
    const int c0 = (int)(i % cpv) * 8;
    float xv[8];
    ld8<T>(x + v * x_ld + x_coff + c0, xv);
#pragma unroll
    for (int j = 0; j < 8; ++j) xv[j] = act_apply(fmaf(xv[j], table[2 * (c0 + j)], table[2 * (c0 + j) + 1]), act);
    st8<T>(y + v * y_ld + y_coff + c0, xv);
  }
}

// Per-channel {sum dz, sum dz*xhat}: each thread keeps fp32 partials of its 8 channels over a strided set of voxels, the
// block adds them per channel in a fixed order in fp64 and adds that to `sums` with one fp64 atomic per value.  The
// order of those atomics across blocks is not fixed, so the fp64 sums can differ in their last bits from run to run;
// every consumer rounds them to fp32 (dgamma, dbeta, coef), where such differences almost never survive.
template <typename T>
__global__ void __launch_bounds__(kThreads) bn_bwd_reduce_kernel(const T* __restrict__ g, int g_ld, int g_coff,
                                                                 const T* __restrict__ x, int x_ld, int x_coff,
                                                                 const float* __restrict__ table, int act,
                                                                 const float* __restrict__ mean_rstd, int64_t nvox,
                                                                 int C, double* __restrict__ sums) {
  __shared__ float red[kThreads * 16];
  const int cpv = C / 8, vpp = kThreads / cpv;
  const int c8 = threadIdx.x % cpv, vl = threadIdx.x / cpv;
  const bool active = vl < vpp;
  const bool mask = table != nullptr && act != B200SEG_ACT_NONE;
  float s1[8], s2[8], sc[8], sf[8], mu[8], rs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s1[j] = 0.f; s2[j] = 0.f;
    const int c = c8 * 8 + j;
    sc[j] = mask ? table[2 * c] : 1.f; sf[j] = mask ? table[2 * c + 1] : 0.f;
    mu[j] = mean_rstd[2 * c]; rs[j] = mean_rstd[2 * c + 1];
  }
  if (active) {
    for (int64_t v = (int64_t)blockIdx.x * vpp + vl; v < nvox; v += (int64_t)gridDim.x * vpp) {
      float gv[8], xv[8];
      ld8<T>(g + v * g_ld + g_coff + c8 * 8, gv);
      ld8<T>(x + v * x_ld + x_coff + c8 * 8, xv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dz = mask ? gv[j] * act_grad(fmaf(xv[j], sc[j], sf[j]), act) : gv[j];
        s1[j] += dz;
        s2[j] = fmaf(dz, (xv[j] - mu[j]) * rs[j], s2[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { red[threadIdx.x * 16 + j] = s1[j]; red[threadIdx.x * 16 + 8 + j] = s2[j]; }
  __syncthreads();
  for (int o = threadIdx.x; o < 2 * C; o += kThreads) {
    const int c = o >> 1, k = o & 1;
    double acc = 0.0;
    for (int w = 0; w < vpp; ++w) acc += (double)red[(w * cpv + c / 8) * 16 + k * 8 + (c & 7)];
    atomicAdd(&sums[o], acc);
  }
}

__global__ void bn_bwd_fold_kernel(const double* __restrict__ sums, double count, const float* __restrict__ gamma,
                                   const float* __restrict__ mean_rstd, int training, int C, float* __restrict__ dgamma,
                                   float* __restrict__ dbeta, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double s1 = sums[2 * c], s2 = sums[2 * c + 1];
  const double mean = mean_rstd[2 * c], rstd = mean_rstd[2 * c + 1], gr = (double)gamma[c] * rstd;
  dgamma[c] = (float)s2;
  dbeta[c] = (float)s1;
  // training: dx = gamma*rstd*(dz - s1/n - xhat*s2/n); eval: the statistics are constants, dx = gamma*rstd*dz
  coef[4 * c] = (float)gr;
  coef[4 * c + 1] = training ? (float)(-gr * rstd * s2 / count) : 0.f;
  coef[4 * c + 2] = (float)mean;
  coef[4 * c + 3] = training ? (float)(-gr * s1 / count) : 0.f;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bn_bwd_apply_kernel(const T* __restrict__ g, int g_ld, int g_coff,
                                                                const T* __restrict__ x, int x_ld, int x_coff,
                                                                const float* __restrict__ table, int act,
                                                                const float* __restrict__ coef, const T* add, int add_ld,
                                                                int add_coff, T* out, int out_ld, int out_coff,
                                                                int64_t nvox, int C) {
  const int cpv = C / 8;
  const int64_t n = nvox * cpv;
  const bool mask = table != nullptr && act != B200SEG_ACT_NONE;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = i / cpv;
    const int c0 = (int)(i % cpv) * 8;
    float gv[8], xv[8], av[8];
    ld8<T>(g + v * g_ld + g_coff + c0, gv);
    ld8<T>(x + v * x_ld + x_coff + c0, xv);
    if (add) ld8<T>(add + v * add_ld + add_coff + c0, av);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      const float dz = mask ? gv[j] * act_grad(fmaf(xv[j], table[2 * c], table[2 * c + 1]), act) : gv[j];
      const float4 k = *reinterpret_cast<const float4*>(coef + 4 * c);
      float d = fmaf(k.x, dz, fmaf(k.y, xv[j] - k.z, k.w));
      if (add) d += av[j];
      gv[j] = d;
    }
    st8<T>(out + v * out_ld + out_coff + c0, gv);
  }
}

int elementwise_grid(int64_t n) {
  const int64_t want = (n + kThreads - 1) / kThreads, cap = (int64_t)B200SEG_NUM_SMS * 16;
  return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

// 8-channel vectors: channel count, leading dimensions and offsets in whole 16-byte chunks
bool vec_ok(int C, int ld, int coff) { return C > 0 && C % 8 == 0 && ld % 8 == 0 && coff % 8 == 0 && coff + C <= ld; }

}  // namespace

extern "C" int b200seg_batchnorm_fwd_fold(const double* sums, int nb, int C, double count, const float* gamma,
                                          const float* beta, float* running_mean, float* running_var,
                                          int64_t* num_batches_tracked, float momentum, float eps, int training,
                                          float* table, float* mean_rstd, void* stream) {
  if (!gamma || !beta || !running_mean || !running_var || !table || !mean_rstd || C <= 0) return B200SEG_EINVAL;
  // torch: "Expected more than 1 value per channel when training"
  if (training && (!sums || nb <= 0 || count <= 1.0)) return B200SEG_EINVAL;
  bn_fwd_fold_kernel<<<(C + kThreads - 1) / kThreads, kThreads, 0, as_stream(stream)>>>(
      sums, nb, C, count, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, training, table,
      mean_rstd);
  B200_CHECK_LAUNCH("bn_fwd_fold_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_batchnorm_apply(const void* x, int dtype, int x_ld, int x_coff, const float* table, int act,
                                       void* y, int y_ld, int y_coff, int64_t nvox, int C, void* stream) {
  if (!x || !table || !y || nvox <= 0) return B200SEG_EINVAL;
  if (!vec_ok(C, x_ld, x_coff) || !vec_ok(C, y_ld, y_coff)) return B200SEG_EUNSUPPORTED;
  const int grid = elementwise_grid(nvox * (C / 8));
  cudaStream_t st = as_stream(stream);
  if (dtype == B200SEG_F16)
    bn_apply_kernel<__half><<<grid, kThreads, 0, st>>>((const __half*)x, x_ld, x_coff, table, act, (__half*)y, y_ld, y_coff, nvox, C);
  else if (dtype == B200SEG_F32)
    bn_apply_kernel<float><<<grid, kThreads, 0, st>>>((const float*)x, x_ld, x_coff, table, act, (float*)y, y_ld, y_coff, nvox, C);
  else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("bn_apply_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_batchnorm_bwd_reduce(const void* g, int g_ld, int g_coff, const void* x, int x_ld, int x_coff,
                                            int dtype, const float* table, int act, const float* mean_rstd,
                                            int64_t nvox, int C, double* sums, void* stream) {
  if (!g || !x || !mean_rstd || !sums || nvox <= 0) return B200SEG_EINVAL;
  if (!vec_ok(C, g_ld, g_coff) || !vec_ok(C, x_ld, x_coff) || C / 8 > kThreads) return B200SEG_EUNSUPPORTED;
  const int vpp = kThreads / (C / 8);
  const int64_t want = (nvox + vpp - 1) / vpp, cap = (int64_t)B200SEG_NUM_SMS * 4;
  const int grid = (int)(want < cap ? want : cap);
  cudaStream_t st = as_stream(stream);
  if (dtype == B200SEG_F16)
    bn_bwd_reduce_kernel<__half><<<grid, kThreads, 0, st>>>((const __half*)g, g_ld, g_coff, (const __half*)x, x_ld, x_coff,
                                                            table, act, mean_rstd, nvox, C, sums);
  else if (dtype == B200SEG_F32)
    bn_bwd_reduce_kernel<float><<<grid, kThreads, 0, st>>>((const float*)g, g_ld, g_coff, (const float*)x, x_ld, x_coff,
                                                           table, act, mean_rstd, nvox, C, sums);
  else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("bn_bwd_reduce_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_batchnorm_bwd_fold(const double* sums, double count, const float* gamma, const float* mean_rstd,
                                          int training, int C, float* dgamma, float* dbeta, float* coef, void* stream) {
  if (!sums || !gamma || !mean_rstd || !dgamma || !dbeta || !coef || C <= 0 || count <= 0.0) return B200SEG_EINVAL;
  bn_bwd_fold_kernel<<<(C + kThreads - 1) / kThreads, kThreads, 0, as_stream(stream)>>>(sums, count, gamma, mean_rstd,
                                                                                         training, C, dgamma, dbeta, coef);
  B200_CHECK_LAUNCH("bn_bwd_fold_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_batchnorm_bwd_apply(const void* g, int g_ld, int g_coff, const void* x, int x_ld, int x_coff,
                                           int dtype, const float* table, int act, const float* coef, const void* add,
                                           int add_ld, int add_coff, void* out, int out_ld, int out_coff, int64_t nvox,
                                           int C, void* stream) {
  if (!g || !x || !coef || !out || nvox <= 0) return B200SEG_EINVAL;
  if (!vec_ok(C, g_ld, g_coff) || !vec_ok(C, x_ld, x_coff) || !vec_ok(C, out_ld, out_coff) ||
      (add && !vec_ok(C, add_ld, add_coff)) || (reinterpret_cast<uintptr_t>(coef) & 15)) return B200SEG_EUNSUPPORTED;
  const int grid = elementwise_grid(nvox * (C / 8));
  cudaStream_t st = as_stream(stream);
  if (dtype == B200SEG_F16)
    bn_bwd_apply_kernel<__half><<<grid, kThreads, 0, st>>>((const __half*)g, g_ld, g_coff, (const __half*)x, x_ld, x_coff,
                                                           table, act, coef, (const __half*)add, add_ld, add_coff,
                                                           (__half*)out, out_ld, out_coff, nvox, C);
  else if (dtype == B200SEG_F32)
    bn_bwd_apply_kernel<float><<<grid, kThreads, 0, st>>>((const float*)g, g_ld, g_coff, (const float*)x, x_ld, x_coff,
                                                          table, act, coef, (const float*)add, add_ld, add_coff,
                                                          (float*)out, out_ld, out_coff, nvox, C);
  else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("bn_bwd_apply_kernel");
  return B200SEG_OK;
}
