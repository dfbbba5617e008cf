// swin.cu — the SwinUNETR-specific operators (reference model/dim3/swin_unetr.py), channels-last tensors.
//
//  * window attention core, WindowAttention.forward swin_unetr.py:467-490 between the qkv and proj Linears, fused with
//    the plumbing of SwinTransformerBlock.forward_part1 :554-606: zero-padding to a window multiple, the cyclic shift,
//    window_partition / window_reverse (:295-355), the shift mask of compute_mask (:737-773) and the relative-position
//    bias gather (:417-459,473-476) are all index arithmetic inside the kernel — the padded / rolled / partitioned
//    copies of the activation, the [nW,n,n] mask and the [heads,n,n] bias tensor never exist.  Scores never leave the
//    SM: one CTA per (window, head), K and V of the window in shared memory, an online softmax per query row
//    (the reference materialises [b*nW, heads, 343, 343] fp32 scores: 1.4 GB at stage 1).
//    Padding tokens: the reference pads AFTER norm1 and BEFORE the qkv Linear, so a padding token's q/k/v is the
//    qkv bias; it takes part as a key/value and its gradient lands on that bias (dqkv_bias_pad).
//    Quirk kept: relative_position_index[:n,:n] is sliced from the FULL 7x7x7 table, i.e. token t of a clamped
//    window is looked up as if it were token t of a 7^3 window (:474).
//    Backward = two recomputing passes (query-stationary for dQ and the softmax row terms, key-stationary for dK / dV),
//    d(bias table) accumulated per CTA in shared memory.
//  * PatchMerging v0.9 gather with its duplicated slices (:717-727) and its scatter-add gradient.
#include "swin_geom.cuh"
#include <math.h>

namespace {

using namespace swin;

// a padding token's q / k / v is the qkv bias as the reference's Linear returns it for a zero input: in the activation
// type, i.e. rounded to fp16 under autocast (as swin_mma.cu's load_token does)
template <typename T> __device__ __forceinline__ float pad_value(float b) { return b; }
template <> __device__ __forceinline__ float pad_value<__half>(float b) { return __half2float(__float2half_rn(b)); }

template <typename T>
__device__ __forceinline__ void load_vec(const T* p, const float* bias, bool valid, int dh, float* out) {
  for (int d = 0; d < dh; ++d) out[d] = valid ? Elem<T>::ld(p + d) : (bias ? pad_value<T>(bias[d]) : 0.f);
}

// shared layout: K[n][dh], V[n][dh] (fp32), table[T] (this head's bias column), rid[n], rc[n]
template <typename T>
__global__ void __launch_bounds__(kWinThreads)
win_attn_fwd_kernel(const T* __restrict__ qkv, const float* __restrict__ qkv_bias, const float* __restrict__ table,
                    T* __restrict__ out, float* __restrict__ lse, WinGeom g, float scale) {
  extern __shared__ float sm[];
  const int n = g.n, dh = g.dh, C = g.heads * dh, TBL = (2 * g.full[0] - 1) * (2 * g.full[1] - 1) * (2 * g.full[2] - 1);
  float* sK = sm; float* sV = sK + n * dh; float* sT = sV + n * dh;
  int* sRid = reinterpret_cast<int*>(sT + TBL); int* sRc = sRid + n;
  const int head = blockIdx.y;
  int wlin = blockIdx.x;
  const int ww = wlin % g.nw[2]; wlin /= g.nw[2];
  const int wh = wlin % g.nw[1]; wlin /= g.nw[1];
  const int wd = wlin % g.nw[0]; const int b = wlin / g.nw[0];
  const int64_t V = (int64_t)g.D * g.H * g.W;
  const int t = threadIdx.x;
  for (int i = t; i < TBL; i += kWinThreads) sT[i] = table[(int64_t)i * g.heads + head];
  float q[kMaxDh];
  TokenInfo ti; ti.valid = false; ti.vox = 0; ti.rid = 0; ti.rc = 0;
  if (t < n) {
    ti = token_info(g, wd, wh, ww, t);
    const T* base = qkv + ((int64_t)b * V + ti.vox) * (3 * C) + head * dh;
    float kv[kMaxDh];
    load_vec<T>(base, qkv_bias ? qkv_bias + head * dh : nullptr, ti.valid, dh, q);
    for (int d = 0; d < dh; ++d) q[d] *= scale;
    load_vec<T>(base + C, qkv_bias ? qkv_bias + C + head * dh : nullptr, ti.valid, dh, kv);
    for (int d = 0; d < dh; ++d) sK[t * dh + d] = kv[d];
    load_vec<T>(base + 2 * C, qkv_bias ? qkv_bias + 2 * C + head * dh : nullptr, ti.valid, dh, kv);
    for (int d = 0; d < dh; ++d) sV[t * dh + d] = kv[d];
    sRid[t] = ti.rid; sRc[t] = ti.rc;
  }
  __syncthreads();
  if (t >= n) return;
  float m = -INFINITY, l = 0.f, acc[kMaxDh];
  for (int d = 0; d < dh; ++d) acc[d] = 0.f;
  for (int j = 0; j < n; ++j) {
    float s = 0.f;
    for (int d = 0; d < dh; ++d) s = fmaf(q[d], sK[j * dh + d], s);
    s += sT[rel_index(g, ti.rc, sRc[j])];
    if (g.masked && sRid[j] != ti.rid) s -= 100.f;
    const float mn = fmaxf(m, s);
    const float corr = __expf(m - mn), pj = __expf(s - mn);
    l = l * corr + pj;
    for (int d = 0; d < dh; ++d) acc[d] = fmaf(acc[d], corr, pj * sV[j * dh + d]);
    m = mn;
  }
  const float inv = 1.f / l;
  lse[((int64_t)blockIdx.x * g.heads + head) * n + t] = m + __logf(l);
  if (ti.valid) {
    T* o = out + ((int64_t)b * V + ti.vox) * C + head * dh;
    for (int d = 0; d < dh; ++d) Elem<T>::st(o + d, acc[d] * inv);
  }
}

// pass A (query-stationary): delta_i = <dO_i, O_i>, dQ_i, d(bias table)
template <typename T>
__global__ void __launch_bounds__(kWinThreads)
win_attn_bwd_q_kernel(const T* __restrict__ qkv, const float* __restrict__ qkv_bias, const float* __restrict__ table,
                      const T* __restrict__ out, const T* __restrict__ dout, const float* __restrict__ lse,
                      float* __restrict__ delta, T* __restrict__ dqkv, float* __restrict__ dtable, WinGeom g, float scale) {
  extern __shared__ float sm[];
  const int n = g.n, dh = g.dh, C = g.heads * dh, TBL = (2 * g.full[0] - 1) * (2 * g.full[1] - 1) * (2 * g.full[2] - 1);
  float* sK = sm; float* sV = sK + n * dh; float* sT = sV + n * dh; float* sDT = sT + TBL;
  int* sRid = reinterpret_cast<int*>(sDT + TBL); int* sRc = sRid + n;
  const int head = blockIdx.y;
  int wlin = blockIdx.x;
  const int ww = wlin % g.nw[2]; wlin /= g.nw[2];
  const int wh = wlin % g.nw[1]; wlin /= g.nw[1];
  const int wd = wlin % g.nw[0]; const int b = wlin / g.nw[0];
  const int64_t V = (int64_t)g.D * g.H * g.W;
  const int t = threadIdx.x;
  for (int i = t; i < TBL; i += kWinThreads) { sT[i] = table[(int64_t)i * g.heads + head]; sDT[i] = 0.f; }
  float q[kMaxDh], dO[kMaxDh];
  TokenInfo ti; ti.valid = false; ti.vox = 0; ti.rid = 0; ti.rc = 0;
  float dlt = 0.f, ls = 0.f;
  if (t < n) {
    ti = token_info(g, wd, wh, ww, t);
    const T* base = qkv + ((int64_t)b * V + ti.vox) * (3 * C) + head * dh;
    float kv[kMaxDh];
    load_vec<T>(base, qkv_bias ? qkv_bias + head * dh : nullptr, ti.valid, dh, q);
    for (int d = 0; d < dh; ++d) q[d] *= scale;
    load_vec<T>(base + C, qkv_bias ? qkv_bias + C + head * dh : nullptr, ti.valid, dh, kv);
    for (int d = 0; d < dh; ++d) sK[t * dh + d] = kv[d];
    load_vec<T>(base + 2 * C, qkv_bias ? qkv_bias + 2 * C + head * dh : nullptr, ti.valid, dh, kv);
    for (int d = 0; d < dh; ++d) sV[t * dh + d] = kv[d];
    sRid[t] = ti.rid; sRc[t] = ti.rc;
    // a padding query's output is cropped away by the reference (:600-601): its upstream gradient is zero
    const int64_t oo = ((int64_t)b * V + ti.vox) * C + head * dh;
    for (int d = 0; d < dh; ++d) {
      dO[d] = ti.valid ? Elem<T>::ld(dout + oo + d) : 0.f;
      dlt += dO[d] * (ti.valid ? Elem<T>::ld(out + oo + d) : 0.f);
    }
    ls = lse[((int64_t)blockIdx.x * g.heads + head) * n + t];
    delta[((int64_t)blockIdx.x * g.heads + head) * n + t] = dlt;
  }
  __syncthreads();
  if (t < n) {
    float dq[kMaxDh];
    for (int d = 0; d < dh; ++d) dq[d] = 0.f;
    if (ti.valid) {
      for (int j = 0; j < n; ++j) {
        float s = 0.f, dp = 0.f;
        for (int d = 0; d < dh; ++d) { s = fmaf(q[d], sK[j * dh + d], s); dp = fmaf(dO[d], sV[j * dh + d], dp); }
        const int ri = rel_index(g, ti.rc, sRc[j]);
        s += sT[ri];
        if (g.masked && sRid[j] != ti.rid) s -= 100.f;
        const float p = __expf(s - ls);
        const float ds = p * (dp - dlt);
        for (int d = 0; d < dh; ++d) dq[d] = fmaf(ds, sK[j * dh + d], dq[d]);
        atomicAdd(&sDT[ri], ds);
      }
      T* o = dqkv + ((int64_t)b * V + ti.vox) * (3 * C) + head * dh;
      for (int d = 0; d < dh; ++d) Elem<T>::st(o + d, dq[d] * scale);
    }
  }
  __syncthreads();
  for (int i = t; i < TBL; i += kWinThreads) {
    const float v = sDT[i];
    if (v != 0.f) atomicAdd(&dtable[(int64_t)i * g.heads + head], v);
  }
}

// pass B (key-stationary): dK_j, dV_j; padding keys' gradients go to the qkv bias
template <typename T>
__global__ void __launch_bounds__(kWinThreads)
win_attn_bwd_kv_kernel(const T* __restrict__ qkv, const float* __restrict__ qkv_bias, const float* __restrict__ table,
                       const T* __restrict__ dout, const float* __restrict__ lse, const float* __restrict__ delta,
                       T* __restrict__ dqkv, float* __restrict__ dbias_pad, WinGeom g, float scale) {
  extern __shared__ float sm[];
  const int n = g.n, dh = g.dh, C = g.heads * dh, TBL = (2 * g.full[0] - 1) * (2 * g.full[1] - 1) * (2 * g.full[2] - 1);
  float* sQ = sm; float* sDO = sQ + n * dh; float* sT = sDO + n * dh; float* sL = sT + TBL; float* sD = sL + n;
  int* sRid = reinterpret_cast<int*>(sD + n); int* sRc = sRid + n; int* sVal = sRc + n;
  const int head = blockIdx.y;
  int wlin = blockIdx.x;
  const int ww = wlin % g.nw[2]; wlin /= g.nw[2];
  const int wh = wlin % g.nw[1]; wlin /= g.nw[1];
  const int wd = wlin % g.nw[0]; const int b = wlin / g.nw[0];
  const int64_t V = (int64_t)g.D * g.H * g.W;
  const int t = threadIdx.x;
  for (int i = t; i < TBL; i += kWinThreads) sT[i] = table[(int64_t)i * g.heads + head];
  float k[kMaxDh], v[kMaxDh];
  TokenInfo ti; ti.valid = false; ti.vox = 0; ti.rid = 0; ti.rc = 0;
  if (t < n) {
    ti = token_info(g, wd, wh, ww, t);
    const T* base = qkv + ((int64_t)b * V + ti.vox) * (3 * C) + head * dh;
    float tmp[kMaxDh];
    load_vec<T>(base, qkv_bias ? qkv_bias + head * dh : nullptr, ti.valid, dh, tmp);
    for (int d = 0; d < dh; ++d) sQ[t * dh + d] = tmp[d] * scale;
    load_vec<T>(base + C, qkv_bias ? qkv_bias + C + head * dh : nullptr, ti.valid, dh, k);
    load_vec<T>(base + 2 * C, qkv_bias ? qkv_bias + 2 * C + head * dh : nullptr, ti.valid, dh, v);
    const int64_t oo = ((int64_t)b * V + ti.vox) * C + head * dh;
    for (int d = 0; d < dh; ++d) sDO[t * dh + d] = ti.valid ? Elem<T>::ld(dout + oo + d) : 0.f;
    sL[t] = lse[((int64_t)blockIdx.x * g.heads + head) * n + t];
    sD[t] = delta[((int64_t)blockIdx.x * g.heads + head) * n + t];
    sRid[t] = ti.rid; sRc[t] = ti.rc; sVal[t] = ti.valid ? 1 : 0;
  }
  __syncthreads();
  if (t >= n) return;
  float dk[kMaxDh], dv[kMaxDh];
  for (int d = 0; d < dh; ++d) { dk[d] = 0.f; dv[d] = 0.f; }
  for (int i = 0; i < n; ++i) {
    if (!sVal[i]) continue;                        // padding queries carry no gradient
    float s = 0.f, dp = 0.f;
    for (int d = 0; d < dh; ++d) { s = fmaf(sQ[i * dh + d], k[d], s); dp = fmaf(sDO[i * dh + d], v[d], dp); }
    s += sT[rel_index(g, sRc[i], ti.rc)];
    if (g.masked && sRid[i] != ti.rid) s -= 100.f;
    const float p = __expf(s - sL[i]);
    const float ds = p * (dp - sD[i]);
    for (int d = 0; d < dh; ++d) { dv[d] = fmaf(p, sDO[i * dh + d], dv[d]); dk[d] = fmaf(ds, sQ[i * dh + d], dk[d]); }
  }
  if (ti.valid) {
    T* o = dqkv + ((int64_t)b * V + ti.vox) * (3 * C) + head * dh;
    for (int d = 0; d < dh; ++d) { Elem<T>::st(o + C + d, dk[d]); Elem<T>::st(o + 2 * C + d, dv[d]); }
  } else if (dbias_pad) {
    for (int d = 0; d < dh; ++d) { atomicAdd(&dbias_pad[C + head * dh + d], dk[d]); atomicAdd(&dbias_pad[2 * C + head * dh + d], dv[d]); }
  }
}

// ---- PatchMerging v0.9 (swin_unetr.py:717-727): y[.., q*C + c] = x[2d+i_q, 2h+j_q, 2w+k_q, c] with the reference's
// offset list INCLUDING its duplicates (x5 == x2, x6 == x3; the (0,1,1) and (1,1,0) sub-lattices are never read).
__constant__ int kMergeOff[8][3] = {{0, 0, 0}, {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {1, 0, 1}, {0, 1, 0}, {0, 0, 1}, {1, 1, 1}};
__constant__ int kMergeOffV2[8][3] = {{0, 0, 0}, {0, 0, 1}, {0, 1, 0}, {0, 1, 1}, {1, 0, 0}, {1, 0, 1}, {1, 1, 0}, {1, 1, 1}};

template <typename T>
__global__ void merge_gather_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int D, int H, int W, int C, int Do, int Ho,
                                    int Wo, int v2) {
  const int c8n = C / 8;
  const int64_t total = (int64_t)B * Do * Ho * Wo * 8 * c8n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % c8n); int64_t r = i / c8n;
    const int q = (int)(r % 8); r /= 8;
    const int w = (int)(r % Wo); r /= Wo; const int h = (int)(r % Ho); r /= Ho; const int d = (int)(r % Do); const int b = (int)(r / Do);
    const int* off = v2 ? kMergeOffV2[q] : kMergeOff[q];
    const int sd = 2 * d + off[0], sh = 2 * h + off[1], sw = 2 * w + off[2];
    uint4 val = make_uint4(0, 0, 0, 0);            // F.pad(x, ...) with zeros for odd extents
    float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const bool in = sd < D && sh < H && sw < W;
    T* dst = y + ((((int64_t)b * Do + d) * Ho + h) * Wo + w) * (8 * C) + q * C + c8 * 8;
    if (in) ld8<T>(x + ((((int64_t)b * D + sd) * H + sh) * W + sw) * C + c8 * 8, f);
    (void)val;
    st8<T>(dst, f);
  }
}

// gradient: dx[src voxel] = sum over the slices q that read it of dy[.., q*C + c]
template <typename T>
__global__ void merge_scatter_kernel(const T* __restrict__ dy, T* __restrict__ dx, int B, int D, int H, int W, int C, int Do, int Ho,
                                     int Wo, int v2) {
  const int c8n = C / 8;
  const int64_t total = (int64_t)B * D * H * W * c8n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % c8n); int64_t r = i / c8n;
    const int w = (int)(r % W); r /= W; const int h = (int)(r % H); r /= H; const int d = (int)(r % D); const int b = (int)(r / D);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const int pd = d & 1, ph = h & 1, pw = w & 1;
    const T* src = dy + ((((int64_t)b * Do + (d >> 1)) * Ho + (h >> 1)) * Wo + (w >> 1)) * (8 * C) + c8 * 8;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int* off = v2 ? kMergeOffV2[q] : kMergeOff[q];
      if (off[0] == pd && off[1] == ph && off[2] == pw) {
        float f[8];
        ld8<T>(src + q * C, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
      }
    }
    st8<T>(dx + i * 8, acc);
  }
}

}  // namespace

// tensor-core (mma.sync m16n8k16) path for fp16 activations, swin_mma.cu
bool b200seg_winattn_mma_applies(const void* qkv, int heads, int dh, int dtype);
int b200seg_winattn_mma_fwd(const swin::WinGeom& g, const void* qkv, const float* qkv_bias, const float* table, void* out, float* lse,
                            float scale, cudaStream_t st);
int b200seg_winattn_mma_bwd(const swin::WinGeom& g, const void* qkv, const float* qkv_bias, const float* table, const void* out,
                            const void* dout, const float* lse, float* delta, void* dqkv, float* dtable, float* dbias_pad, float scale,
                            cudaStream_t st);

extern "C" size_t b200seg_window_attn_workspace(int B, int D, int H, int W, int heads, const int* window) {
  WinGeom g;
  const int zero[3] = {0, 0, 0};
  if (fill_geom(g, B, D, H, W, heads, 1, window, zero)) return 0;
  return (size_t)B * g.nw[0] * g.nw[1] * g.nw[2] * heads * g.n * sizeof(float);       // one fp32 per (window, head, token)
}

// out[b, voxel, head*dh + d] from qkv[b, voxel, {q,k,v} x heads x dh]; lse: workspace-sized fp32 buffer kept for backward
extern "C" int b200seg_window_attn_fwd(const void* qkv, const float* qkv_bias, const float* bias_table, void* out, float* lse,
                                       int B, int D, int H, int W, int heads, int dh, const int* window, const int* shift,
                                       int dtype, void* stream) {
  if (!qkv || !bias_table || !out || !lse) return B200SEG_EINVAL;
  WinGeom g;
  int rc = fill_geom(g, B, D, H, W, heads, dh, window, shift);
  if (rc) return rc;
  const int TBL = (2 * g.full[0] - 1) * (2 * g.full[1] - 1) * (2 * g.full[2] - 1);
  const size_t smem = sizeof(float) * ((size_t)2 * g.n * dh + TBL) + sizeof(int) * 2 * g.n;
  dim3 grid(B * g.nw[0] * g.nw[1] * g.nw[2], heads);
  const float scale = 1.0f / sqrtf((float)dh);
  cudaStream_t st = as_stream(stream);
  if (b200seg_winattn_mma_applies(qkv, heads, dh, dtype) && !(reinterpret_cast<uintptr_t>(out) & 15))
    return b200seg_winattn_mma_fwd(g, qkv, qkv_bias, bias_table, out, lse, scale, st);
  if (dtype == B200SEG_F16) {
    B200_CUDA(cudaFuncSetAttribute(win_attn_fwd_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    win_attn_fwd_kernel<__half><<<grid, kWinThreads, smem, st>>>((const __half*)qkv, qkv_bias, bias_table, (__half*)out, lse, g, scale);
  } else if (dtype == B200SEG_F32) {
    B200_CUDA(cudaFuncSetAttribute(win_attn_fwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    win_attn_fwd_kernel<float><<<grid, kWinThreads, smem, st>>>((const float*)qkv, qkv_bias, bias_table, (float*)out, lse, g, scale);
  } else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("win_attn_fwd_kernel");
  return B200SEG_OK;
}

// dqkv (same layout as qkv; padding tokens' rows do not exist), dtable [T][heads] (+=), dbias_pad [3C] (+=, nullable)
extern "C" int b200seg_window_attn_bwd(const void* qkv, const float* qkv_bias, const float* bias_table, const void* out,
                                       const void* dout, const float* lse, float* delta, void* dqkv, float* dtable,
                                       float* dbias_pad, int B, int D, int H, int W, int heads, int dh, const int* window,
                                       const int* shift, int dtype, void* stream) {
  if (!qkv || !bias_table || !out || !dout || !lse || !delta || !dqkv || !dtable) return B200SEG_EINVAL;
  WinGeom g;
  int rc = fill_geom(g, B, D, H, W, heads, dh, window, shift);
  if (rc) return rc;
  const int TBL = (2 * g.full[0] - 1) * (2 * g.full[1] - 1) * (2 * g.full[2] - 1);
  const size_t smem_q = sizeof(float) * ((size_t)2 * g.n * dh + 2 * TBL) + sizeof(int) * 2 * g.n;
  const size_t smem_kv = sizeof(float) * ((size_t)2 * g.n * dh + TBL + 2 * g.n) + sizeof(int) * 3 * g.n;
  dim3 grid(B * g.nw[0] * g.nw[1] * g.nw[2], heads);
  const float scale = 1.0f / sqrtf((float)dh);
  cudaStream_t st = as_stream(stream);
  if (b200seg_winattn_mma_applies(qkv, heads, dh, dtype) && !((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(dout) |
                                                                reinterpret_cast<uintptr_t>(dqkv)) & 15))
    return b200seg_winattn_mma_bwd(g, qkv, qkv_bias, bias_table, out, dout, lse, delta, dqkv, dtable, dbias_pad, scale, st);
#define WIN_BWD(TT)                                                                                                               \
  do {                                                                                                                            \
    B200_CUDA(cudaFuncSetAttribute(win_attn_bwd_q_kernel<TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_q));          \
    B200_CUDA(cudaFuncSetAttribute(win_attn_bwd_kv_kernel<TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_kv));        \
    win_attn_bwd_q_kernel<TT><<<grid, kWinThreads, smem_q, st>>>((const TT*)qkv, qkv_bias, bias_table, (const TT*)out, (const TT*)dout, \
                                                                 lse, delta, (TT*)dqkv, dtable, g, scale);                         \
    B200_CHECK_LAUNCH("win_attn_bwd_q_kernel");                                                                                   \
    win_attn_bwd_kv_kernel<TT><<<grid, kWinThreads, smem_kv, st>>>((const TT*)qkv, qkv_bias, bias_table, (const TT*)dout, lse, delta, \
                                                                   (TT*)dqkv, dbias_pad, g, scale);                                \
    B200_CHECK_LAUNCH("win_attn_bwd_kv_kernel");                                                                                  \
  } while (0)
  if (dtype == B200SEG_F16) WIN_BWD(__half);
  else if (dtype == B200SEG_F32) WIN_BWD(float);
  else return B200SEG_EINVAL;
#undef WIN_BWD
  return B200SEG_OK;
}

extern "C" int b200seg_swin_merge(const void* x, void* y, int B, int D, int H, int W, int C, int reverse, int v2, int dtype,
                                  void* stream) {
  if (!x || !y || C % 8) return C % 8 ? B200SEG_EUNSUPPORTED : B200SEG_EINVAL;
  const int Do = (D + 1) / 2, Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  cudaStream_t st = as_stream(stream);
  const int64_t total = reverse ? (int64_t)B * D * H * W * (C / 8) : (int64_t)B * Do * Ho * Wo * C;
  int grid = ceil_div(total, 256); if (grid > B200SEG_NUM_SMS * 16) grid = B200SEG_NUM_SMS * 16;
  if (dtype == B200SEG_F16) {
    if (!reverse) merge_gather_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (__half*)y, B, D, H, W, C, Do, Ho, Wo, v2);
    else merge_scatter_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x, (__half*)y, B, D, H, W, C, Do, Ho, Wo, v2);
  } else if (dtype == B200SEG_F32) {
    if (!reverse) merge_gather_kernel<float><<<grid, 256, 0, st>>>((const float*)x, (float*)y, B, D, H, W, C, Do, Ho, Wo, v2);
    else merge_scatter_kernel<float><<<grid, 256, 0, st>>>((const float*)x, (float*)y, B, D, H, W, C, Do, Ho, Wo, v2);
  } else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("swin_merge_kernel");
  return B200SEG_OK;
}
