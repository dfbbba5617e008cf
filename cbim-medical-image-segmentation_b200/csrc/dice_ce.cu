// dice_ce.cu — fused softmax + adaptive-Tversky Dice + weighted CE, forward and backward.
// One HBM pass each way (reference: ~30 full-tensor ATen passes, training/losses.py:18-58
// plus nn.CrossEntropyLoss at train_ddp.py:93,189-191).
//
// Algebra (per class c, sums over batch AND space jointly, losses.py:38-44):
//   TP = sum P*M, SP = sum P, CNT = sum M  ->  FP = SP-TP, FN = CNT-TP
//   alpha = clamp(FP/(FP+FN+s), .2, .8)  (kept in the autograd graph by the reference)
//   dice  = TP / (TP + alpha FP + (1-alpha) FN + s);  Dice loss = mean_c (1 - dice)
//   CE    = sum_v w[y] (lse - x_y) / sum_v w[y]   (lse = m + log sum exp(x - m), m = max_c x)
// Algorithmic bytes: fwd B*V*(C*s + label_bytes), bwd B*V*(2*C*s + label_bytes).
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr float kSmooth = 1e-5f;

template <typename T, int C, bool CL>
__device__ __forceinline__ void load_logits(const T* __restrict__ p, int64_t stride_c, float (&x)[C]) {
  if constexpr (CL && sizeof(T) == 2 && (C % 4 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 4; ++i) {
      uint2 u = reinterpret_cast<const uint2*>(p)[i];
      float2 a = __half22float2(*reinterpret_cast<__half2*>(&u.x));
      float2 b = __half22float2(*reinterpret_cast<__half2*>(&u.y));
      x[4 * i] = a.x; x[4 * i + 1] = a.y; x[4 * i + 2] = b.x; x[4 * i + 3] = b.y;
    }
  } else if constexpr (CL && sizeof(T) == 2 && (C % 2 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 2; ++i) {
      float2 a = __half22float2(reinterpret_cast<const __half2*>(p)[i]);
      x[2 * i] = a.x; x[2 * i + 1] = a.y;
    }
  } else if constexpr (CL && sizeof(T) == 4 && (C % 4 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 4; ++i) {
      float4 a = reinterpret_cast<const float4*>(p)[i];
      x[4 * i] = a.x; x[4 * i + 1] = a.y; x[4 * i + 2] = a.z; x[4 * i + 3] = a.w;
    }
  } else {
#pragma unroll
    for (int c = 0; c < C; ++c) x[c] = Elem<T>::ld(p + c * stride_c);
  }
}

template <typename T, int C, bool CL>
__device__ __forceinline__ void store_logits(T* __restrict__ p, int64_t stride_c, const float (&x)[C]) {
  if constexpr (CL && sizeof(T) == 2 && (C % 4 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 4; ++i) {
      uint2 u;
      *reinterpret_cast<__half2*>(&u.x) = __floats2half2_rn(x[4 * i], x[4 * i + 1]);
      *reinterpret_cast<__half2*>(&u.y) = __floats2half2_rn(x[4 * i + 2], x[4 * i + 3]);
      reinterpret_cast<uint2*>(p)[i] = u;
    }
  } else if constexpr (CL && sizeof(T) == 2 && (C % 2 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 2; ++i) reinterpret_cast<__half2*>(p)[i] = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
  } else if constexpr (CL && sizeof(T) == 4 && (C % 4 == 0)) {
#pragma unroll
    for (int i = 0; i < C / 4; ++i)
      reinterpret_cast<float4*>(p)[i] = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
  } else {
#pragma unroll
    for (int c = 0; c < C; ++c) Elem<T>::st(p + c * stride_c, x[c]);
  }
}

__device__ __forceinline__ int load_label(const void* labels, int label_bytes, int64_t i) {
  if (label_bytes == 8) return (int)reinterpret_cast<const long long*>(labels)[i];
  return (int)reinterpret_cast<const unsigned char*>(labels)[i];
}

// partial layout: [0,C)=TP, [C,2C)=SP, [2C,3C)=CNT, [3C]=sum w*nll, [3C+1]=sum w
template <typename T, int C, bool CL>
__global__ void __launch_bounds__(kThreads)
dice_ce_fwd_kernel(const T* __restrict__ logits, int64_t stride_b, int64_t stride_v, int64_t stride_c,
                   const void* __restrict__ labels, int label_bytes, const float* __restrict__ ce_w,
                   int64_t V, int64_t total, double* __restrict__ partial) {
  float tp[C], sp[C], cnt[C];
#pragma unroll
  for (int c = 0; c < C; ++c) { tp[c] = 0.f; sp[c] = 0.f; cnt[c] = 0.f; }
  float nll = 0.f, wsum = 0.f;

  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += (int64_t)gridDim.x * kThreads) {
    int64_t b = i / V, v = i - b * V;
    float x[C];
    load_logits<T, C, CL>(logits + b * stride_b + v * stride_v, stride_c, x);
    int y = load_label(labels, label_bytes, i);
    float m = x[0], xy = 0.f;
#pragma unroll
    for (int c = 1; c < C; ++c) m = fmaxf(m, x[c]);
#pragma unroll
    for (int c = 0; c < C; ++c) if (c == y) xy = x[c];
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) { x[c] = __expf(x[c] - m); s += x[c]; }
    float inv = 1.f / s;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      // rounded product, never fused into the sums: the Dice sums and with them the gradient stay bit-identical to
      // the form that also kept p_y for the CE
      float p = __fmul_rn(x[c], inv);
      sp[c] += p;
      if (c == y) { tp[c] += p; cnt[c] += 1.f; }
    }
    if (y >= 0 && y < C) {
      // lse - x_y from the logits, not -log(p_y): p_y underflows in fp32 once x_y is ~88 below the max (fp16 logits
      // reach 65504), while the CE of such a confidently wrong voxel keeps growing with the gap, as F.cross_entropy's
      float w = ce_w ? ce_w[y] : 1.f;
      nll += w * ((m - xy) + logf(s));
      wsum += w;
    }
  }

  __shared__ float red[kThreads / 32][3 * C + 2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    float a = warp_sum(tp[c]), b2 = warp_sum(sp[c]), c2 = warp_sum(cnt[c]);
    if (lane == 0) { red[wid][c] = a; red[wid][C + c] = b2; red[wid][2 * C + c] = c2; }
  }
  {
    float a = warp_sum(nll), b2 = warp_sum(wsum);
    if (lane == 0) { red[wid][3 * C] = a; red[wid][3 * C + 1] = b2; }
  }
  __syncthreads();
  if (threadIdx.x < 3 * C + 2) {
    double acc = 0.0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) acc += (double)red[w][threadIdx.x];
    atomicAdd(&partial[threadIdx.x], acc);
  }
}

__global__ void dice_ce_finalize_kernel(const double* __restrict__ partial, int C, float ce_scale,
                                        float dice_scale, float* __restrict__ out) {
  __shared__ double dsum;
  if (threadIdx.x == 0) dsum = 0.0;
  __syncthreads();
  int c = threadIdx.x;
  if (c < C) {
    const double s = (double)kSmooth;
    double TP = partial[c], SP = partial[C + c], CNT = partial[2 * C + c];
    double FP = SP - TP, FN = CNT - TP;
    double q = FP + FN + s;
    double a_raw = FP / q;
    bool inrange = (a_raw >= 0.2) && (a_raw <= 0.8);   // torch.clamp passes grad on the closed interval
    double alpha = a_raw < 0.2 ? 0.2 : (a_raw > 0.8 ? 0.8 : a_raw);
    double beta = 1.0 - alpha;
    double den = TP + alpha * FP + beta * FN;
    double ds = den + s;
    double dice = TP / ds;
    double da_dFP = inrange ? (FN + s) / (q * q) : 0.0;
    double da_dFN = inrange ? (-FP) / (q * q) : 0.0;
    double dden_dFP = alpha + (FP - FN) * da_dFP;
    double dden_dFN = beta + (FP - FN) * da_dFN;
    double ddice_dTP_direct = (ds - TP) / (ds * ds);
    double ddice_dden = -TP / (ds * ds);
    double ddice_dTP = ddice_dTP_direct - ddice_dden * (dden_dFP + dden_dFN);
    double ddice_dSP = ddice_dden * dden_dFP;
    out[4 + c] = (float)(-ddice_dTP / C);
    out[4 + C + c] = (float)(-ddice_dSP / C);
    out[4 + 2 * C + c] = (float)alpha;
    out[4 + 3 * C + c] = (float)dice;
    atomicAdd(&dsum, (1.0 - dice) / C);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double wsum = partial[3 * C + 1];
    double ce = wsum > 0.0 ? partial[3 * C] / wsum : 0.0;
    out[0] = (float)(ce_scale * ce + dice_scale * dsum);
    out[1] = (float)ce;
    out[2] = (float)dsum;
    out[3] = (float)wsum;
  }
}

template <typename T, int C, bool CL>
__global__ void __launch_bounds__(kThreads)
dice_ce_bwd_kernel(const T* __restrict__ logits, int64_t stride_b, int64_t stride_v, int64_t stride_c,
                   const void* __restrict__ labels, int label_bytes, const float* __restrict__ ce_w,
                   int64_t V, int64_t total, float ce_scale, float dice_scale,
                   const float* __restrict__ fwd_out, const float* __restrict__ grad_out,
                   T* __restrict__ dlogits) {
  __shared__ float s_gtp[C], s_gsp[C], s_w[C];
  if (threadIdx.x < C) {
    s_gtp[threadIdx.x] = fwd_out[4 + threadIdx.x] * dice_scale;
    s_gsp[threadIdx.x] = fwd_out[4 + C + threadIdx.x] * dice_scale;
    s_w[threadIdx.x] = ce_w ? ce_w[threadIdx.x] : 1.f;
  }
  __syncthreads();
  const float g = grad_out ? *grad_out : 1.f;
  const float wsum = fwd_out[3];
  const float ce_k = wsum > 0.f ? ce_scale / wsum : 0.f;

  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += (int64_t)gridDim.x * kThreads) {
    int64_t b = i / V, v = i - b * V;
    const int64_t off = b * stride_b + v * stride_v;
    float x[C];
    load_logits<T, C, CL>(logits + off, stride_c, x);
    int y = load_label(labels, label_bytes, i);
    float m = x[0];
#pragma unroll
    for (int c = 1; c < C; ++c) m = fmaxf(m, x[c]);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) { x[c] = __expf(x[c] - m); s += x[c]; }
    float inv = 1.f / s;
    float dot = 0.f;
    float dldp[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
      x[c] *= inv;
      dldp[c] = s_gsp[c] + (c == y ? s_gtp[c] : 0.f);
      dot += x[c] * dldp[c];
    }
    const float wy = (y >= 0 && y < C) ? s_w[y] * ce_k : 0.f;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float d = x[c] * (dldp[c] - dot) + wy * (x[c] - (c == y ? 1.f : 0.f));
      x[c] = d * g;
    }
    store_logits<T, C, CL>(dlogits + off, stride_c, x);
  }
}

template <typename T, int C>
int launch_fwd(const void* logits, int64_t sb, int64_t sv, int64_t sc, const void* labels, int lb,
               const float* w, int B, int64_t V, double* partial, cudaStream_t st) {
  int64_t total = (int64_t)B * V;
  int grid = (int)((total + kThreads - 1) / kThreads);
  int maxg = B200SEG_NUM_SMS * 8;
  if (grid > maxg) grid = maxg;
  bool cl = (sc == 1 && sv == C) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) && (sb % 8 == 0);
  if (cl)
    dice_ce_fwd_kernel<T, C, true><<<grid, kThreads, 0, st>>>((const T*)logits, sb, sv, sc, labels, lb, w, V, total, partial);
  else
    dice_ce_fwd_kernel<T, C, false><<<grid, kThreads, 0, st>>>((const T*)logits, sb, sv, sc, labels, lb, w, V, total, partial);
  return 0;
}

template <typename T, int C>
int launch_bwd(const void* logits, int64_t sb, int64_t sv, int64_t sc, const void* labels, int lb,
               const float* w, int B, int64_t V, float ce_scale, float dice_scale, const float* fwd_out,
               const float* grad_out, void* dlogits, cudaStream_t st) {
  int64_t total = (int64_t)B * V;
  int grid = (int)((total + kThreads - 1) / kThreads);
  int maxg = B200SEG_NUM_SMS * 16;
  if (grid > maxg) grid = maxg;
  bool cl = (sc == 1 && sv == C) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
            ((reinterpret_cast<uintptr_t>(dlogits) & 15) == 0) && (sb % 8 == 0);
  if (cl)
    dice_ce_bwd_kernel<T, C, true><<<grid, kThreads, 0, st>>>((const T*)logits, sb, sv, sc, labels, lb, w, V, total,
                                                              ce_scale, dice_scale, fwd_out, grad_out, (T*)dlogits);
  else
    dice_ce_bwd_kernel<T, C, false><<<grid, kThreads, 0, st>>>((const T*)logits, sb, sv, sc, labels, lb, w, V, total,
                                                               ce_scale, dice_scale, fwd_out, grad_out, (T*)dlogits);
  return 0;
}

}  // namespace

#define DISPATCH_C(C, FN, ...)                    \
  switch (C) {                                    \
    case 2: FN<T, 2>(__VA_ARGS__); break;         \
    case 3: FN<T, 3>(__VA_ARGS__); break;         \
    case 4: FN<T, 4>(__VA_ARGS__); break;         \
    case 5: FN<T, 5>(__VA_ARGS__); break;         \
    case 6: FN<T, 6>(__VA_ARGS__); break;         \
    case 7: FN<T, 7>(__VA_ARGS__); break;         \
    case 8: FN<T, 8>(__VA_ARGS__); break;         \
    case 9: FN<T, 9>(__VA_ARGS__); break;         \
    case 10: FN<T, 10>(__VA_ARGS__); break;       \
    case 11: FN<T, 11>(__VA_ARGS__); break;       \
    case 12: FN<T, 12>(__VA_ARGS__); break;       \
    case 13: FN<T, 13>(__VA_ARGS__); break;       \
    case 14: FN<T, 14>(__VA_ARGS__); break;       \
    case 15: FN<T, 15>(__VA_ARGS__); break;       \
    case 16: FN<T, 16>(__VA_ARGS__); break;       \
    default: return B200SEG_EUNSUPPORTED;         \
  }

template <typename T>
static int fwd_t(const void* logits, int64_t sb, int64_t sv, int64_t sc, const void* labels, int lb,
                 const float* w, int B, int64_t V, int C, double* partial, cudaStream_t st) {
  DISPATCH_C(C, launch_fwd, logits, sb, sv, sc, labels, lb, w, B, V, partial, st);
  return 0;
}
template <typename T>
static int bwd_t(const void* logits, int64_t sb, int64_t sv, int64_t sc, const void* labels, int lb,
                 const float* w, int B, int64_t V, int C, float ce_scale, float dice_scale,
                 const float* fwd_out, const float* grad_out, void* dlogits, cudaStream_t st) {
  DISPATCH_C(C, launch_bwd, logits, sb, sv, sc, labels, lb, w, B, V, ce_scale, dice_scale, fwd_out, grad_out, dlogits, st);
  return 0;
}

extern "C" int b200seg_dice_ce_fwd(const void* logits, int dtype, int64_t stride_b, int64_t stride_v,
                                   int64_t stride_c, const void* labels, int label_bytes,
                                   const float* ce_weight, int B, int64_t V, int C, float ce_scale,
                                   float dice_scale, double* partial, float* out, void* stream) {
  if (!logits || !labels || !partial || !out || B <= 0 || V <= 0 || C < 2) return B200SEG_EINVAL;
  if (label_bytes != 8 && label_bytes != 1) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  B200_CUDA(cudaMemsetAsync(partial, 0, sizeof(double) * (3 * C + 2), st));
  int rc;
  if (dtype == B200SEG_F16) rc = fwd_t<__half>(logits, stride_b, stride_v, stride_c, labels, label_bytes, ce_weight, B, V, C, partial, st);
  else if (dtype == B200SEG_F32) rc = fwd_t<float>(logits, stride_b, stride_v, stride_c, labels, label_bytes, ce_weight, B, V, C, partial, st);
  else return B200SEG_EINVAL;
  if (rc) return rc;
  B200_CHECK_LAUNCH("dice_ce_fwd_kernel");
  dice_ce_finalize_kernel<<<1, 32, 0, st>>>(partial, C, ce_scale, dice_scale, out);
  B200_CHECK_LAUNCH("dice_ce_finalize_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_dice_ce_bwd(const void* logits, int dtype, int64_t stride_b, int64_t stride_v,
                                   int64_t stride_c, const void* labels, int label_bytes,
                                   const float* ce_weight, int B, int64_t V, int C, float ce_scale,
                                   float dice_scale, const float* fwd_out, const float* grad_out,
                                   void* dlogits, void* stream) {
  if (!logits || !labels || !fwd_out || !dlogits || B <= 0 || V <= 0 || C < 2) return B200SEG_EINVAL;
  if (label_bytes != 8 && label_bytes != 1) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  int rc;
  if (dtype == B200SEG_F16) rc = bwd_t<__half>(logits, stride_b, stride_v, stride_c, labels, label_bytes, ce_weight, B, V, C, ce_scale, dice_scale, fwd_out, grad_out, dlogits, st);
  else if (dtype == B200SEG_F32) rc = bwd_t<float>(logits, stride_b, stride_v, stride_c, labels, label_bytes, ce_weight, B, V, C, ce_scale, dice_scale, fwd_out, grad_out, dlogits, st);
  else return B200SEG_EINVAL;
  if (rc) return rc;
  B200_CHECK_LAUNCH("dice_ce_bwd_kernel");
  return B200SEG_OK;
}
