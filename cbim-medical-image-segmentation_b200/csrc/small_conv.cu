// small_conv.cu — HBM-bound special cases of the weight gradient that are not dense contractions
// (SURVEY.md §8d "HBM bandwidth" rows): the Cin=1 stem (unet_utils.py:14) and the 1x1x1 classifier head
// with a handful of output channels (`outc`, unet.py:47).  One pass over dy / x, warp-per-voxel-run with a
// lane per channel, fp32 register accumulators, one partial per (block, output) at the end, summed over the blocks
// in a fixed order (add_slices).
#include "common.cuh"
#include "conv_args.h"

namespace {

constexpr int kWarpsPerBlock = 8;
constexpr int kSmallGridPerSM = 2;        // persistent blocks per SM (register accumulators live for the whole kernel)

// ---- stem: dW[co][tap] = sum_v dy[v][co] * x[v + tap],  Cin == 1, Cout <= 64, taps <= 27.
// HBM-bound (reads dy once: Cout*s bytes per voxel).  Persistent blocks walk (b, d, 8-row h-groups); the single-channel
// input halo of the group sits zero-padded in shared memory as fp32, so the inner loop has no bounds checks:
// warp = one h row, lane = output channel, per voxel 1 coalesced load of dy + KD*KH broadcast LDS (sliding 3-wide
// window along w kept in registers) + taps FFMA.  One partial per (block, co, tap) at the very end, into the block's slice.
template <typename T, int KD, int KH, int KW, bool TWO>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
wgrad_cin1_kernel(WgradArgs a) {
  constexpr int TAPS = KD * KH * KW, ROWS = kWarpsPerBlock, HR = ROWS + KH - 1, WMAX = 256;
  constexpr int pd = KD / 2, ph = KH / 2, pw = KW / 2;
  // the halo tile (main loop) and the reduction scratch (after it) share one buffer
  constexpr int XW = WMAX + 4, kXFloats = KD * HR * XW, kRFloats = kWarpsPerBlock * 32 * (TAPS + 1);
  __shared__ float s_raw[kXFloats > kRFloats ? kXFloats : kRFloats];
  float (*s_x)[HR][XW] = reinterpret_cast<float (*)[HR][XW]>(s_raw);
  float (*s_red)[32][TAPS + 1] = reinterpret_cast<float (*)[32][TAPS + 1]>(s_raw);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const T* x = (const T*)a.x; const T* dy = (const T*)a.dy;
  float acc0[TAPS], acc1[TWO ? TAPS : 1];
#pragma unroll
  for (int t = 0; t < TAPS; ++t) acc0[t] = 0.f;
#pragma unroll
  for (int t = 0; t < (TWO ? TAPS : 1); ++t) acc1[t] = 0.f;
  const int hgroups = (a.H + ROWS - 1) / ROWS;
  const int wchunks = (a.W + WMAX - 1) / WMAX;
  const int64_t njobs = (int64_t)a.B * a.D * hgroups * wchunks;
  const bool c0ok = lane < a.Cout, c1ok = TWO && (lane + 32 < a.Cout);
  for (int64_t job = blockIdx.x; job < njobs; job += gridDim.x) {
    int64_t q = job;
    const int wc = (int)(q % wchunks); q /= wchunks;
    const int hg = (int)(q % hgroups); q /= hgroups;
    const int d = (int)(q % a.D); const int b = (int)(q / a.D);
    const int h0 = hg * ROWS, w0 = wc * WMAX;
    const int wn = min(WMAX, a.W - w0);
    __syncthreads();                       // previous job's readers are done with s_x
    for (int i = threadIdx.x; i < KD * HR * (wn + 2 * pw); i += kWarpsPerBlock * 32) {
      const int wi = i % (wn + 2 * pw); int r = i / (wn + 2 * pw);
      const int hi = r % HR, zi = r / HR;
      const int dd = d + zi - pd, hh = h0 + hi - ph, ww = w0 + wi - pw;
      float v = 0.f;
      if ((unsigned)dd < (unsigned)a.D && (unsigned)hh < (unsigned)a.H && (unsigned)ww < (unsigned)a.W)
        v = Elem<T>::ld(x + ((((int64_t)b * a.D + dd) * a.H + hh) * a.W + ww) * a.x_ld + a.x_coff);
      s_x[zi][hi][wi] = v;
    }
    __syncthreads();
    const int h = h0 + wid;
    if (h < a.H) {
      const T* dyrow = dy + ((((int64_t)b * a.D + d) * a.H + h) * a.W + w0) * a.dy_ld + a.dy_coff + lane;
      float win[KD][KH][KW];               // x[.., w-1], x[.., w], x[.., w+1] per (zd, zh) row
#pragma unroll
      for (int zd = 0; zd < KD; ++zd)
#pragma unroll
        for (int zh = 0; zh < KH; ++zh)
#pragma unroll
          for (int zw = 0; zw < KW - 1; ++zw) win[zd][zh][zw + 1] = s_x[zd][wid + zh][zw];
      constexpr int U = 4;
      for (int wb = 0; wb < wn; wb += U) {
        float g0[U], g1[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const bool in = wb + u < wn;
          g0[u] = (in && c0ok) ? Elem<T>::ld(dyrow + (int64_t)(wb + u) * a.dy_ld) : 0.f;
          g1[u] = (in && c1ok) ? Elem<T>::ld(dyrow + (int64_t)(wb + u) * a.dy_ld + 32) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (wb + u >= wn) break;
#pragma unroll
          for (int zd = 0; zd < KD; ++zd)
#pragma unroll
            for (int zh = 0; zh < KH; ++zh) {
#pragma unroll
              for (int zw = 0; zw < KW - 1; ++zw) win[zd][zh][zw] = win[zd][zh][zw + 1];
              win[zd][zh][KW - 1] = s_x[zd][wid + zh][wb + u + KW - 1];
#pragma unroll
              for (int zw = 0; zw < KW; ++zw) {
                const int t = (zd * KH + zh) * KW + zw;
                acc0[t] = fmaf(g0[u], win[zd][zh][zw], acc0[t]);
                if (TWO) acc1[t] = fmaf(g1[u], win[zd][zh][zw], acc1[t]);
              }
            }
        }
      }
    }
  }
  // block-level reduction, then one partial per (block, output) into the block's slice
  for (int half = 0; half < (TWO ? 2 : 1); ++half) {
    __syncthreads();
#pragma unroll
    for (int t = 0; t < TAPS; ++t) s_red[wid][lane][t] = (half && TWO) ? acc1[TWO ? t : 0] : acc0[t];
    __syncthreads();
    const int nco = min(32, a.Cout - 32 * half);
    for (int o = threadIdx.x; o < nco * TAPS; o += kWarpsPerBlock * 32) {
      const int co = o / TAPS, t = o % TAPS;
      float sum = 0.f;
#pragma unroll
      for (int w = 0; w < kWarpsPerBlock; ++w) sum += s_red[w][co][t];
      a.part[(int64_t)blockIdx.x * (a.Cout * TAPS) + (int64_t)(co + 32 * half) * TAPS + t] = sum;
    }
  }
}

// ---- head: dW[co][ci] = sum_v dy[v][co] * a[v][ci], 1x1x1, Cout <= 16, Cin <= 128 (multiple of 8);
// dbias[co] = sum_v dy[v][co].  HBM-bound: one 16-byte (fp16) load of 8 input channels per thread per voxel, the
// voxel's Cout gradients as one vector load, CPT x MAXCO FFMA into registers; persistent blocks, smem tree reduction,
// one partial per (block, output) into the block's slice.
template <typename T, int MAXCO, int CPT>
__global__ void __launch_bounds__(256)
wgrad_head_kernel(WgradArgs a) {
  constexpr int U = MAXCO <= 4 ? 4 : 2;
  __shared__ float s_red[256][CPT * MAXCO / 4 + 1][4];       // padded rows: conflict-light float4-free layout
  const int64_t V = (int64_t)a.D * a.H * a.W;
  const T* x = (const T*)a.x; const T* dy = (const T*)a.dy;
  const int ngrp = a.Cin / CPT;                   // threads per voxel
  const int vpi = 256 / ngrp;                     // voxels per block iteration
  const int cg = threadIdx.x % ngrp, vl = threadIdx.x / ngrp;
  const bool active = vl < vpi;
  // the voxel's 4 gradients as one vector load when the layout allows it (the UNet head: dy is [V][4])
  const bool gvec = MAXCO == 4 && a.Cout == 4 && a.dy_ld % 4 == 0 && a.dy_coff % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(a.dy) % (4 * sizeof(T))) == 0;
  float acc[CPT][MAXCO], bacc[MAXCO];
#pragma unroll
  for (int k = 0; k < CPT; ++k)
#pragma unroll
    for (int c = 0; c < MAXCO; ++c) acc[k][c] = 0.f;
#pragma unroll
  for (int c = 0; c < MAXCO; ++c) bacc[c] = 0.f;
  for (int b = 0; b < a.B; ++b) {
    float mean[CPT], rstd[CPT];
#pragma unroll
    for (int k = 0; k < CPT; ++k) {
      mean[k] = 0.f; rstd[k] = 1.f;
      if (a.x_stats) stats_to_mean_rstd(a.x_stats + ((int64_t)b * a.Cin + cg * CPT + k) * 2, (double)V, a.eps, mean[k], rstd[k]);
    }
    const T* xb = x + (int64_t)b * V * a.x_ld + a.x_coff + cg * CPT;
    const T* db = dy + (int64_t)b * V * a.dy_ld + a.dy_coff;
    for (int64_t v0 = (int64_t)blockIdx.x * vpi * U + vl; active && v0 < V; v0 += (int64_t)gridDim.x * vpi * U) {
      float xv[U][CPT], g[U][MAXCO];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t v = v0 + (int64_t)u * vpi;
        const bool in = v < V;
        if (in) {
          if constexpr (CPT == 8) ld8<T>(xb + v * a.x_ld, xv[u]);
          else {
#pragma unroll
            for (int k = 0; k < CPT; ++k) xv[u][k] = Elem<T>::ld(xb + v * a.x_ld + k);
          }
          if (MAXCO == 4 && gvec) {
            if constexpr (sizeof(T) == 2) {
              const uint2 q = *reinterpret_cast<const uint2*>(db + v * a.dy_ld);
              const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&q.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&q.y));
              g[u][0] = f0.x; g[u][1] = f0.y; g[u][2] = f1.x; g[u][3] = f1.y;
            } else {
              const float4 q = *reinterpret_cast<const float4*>(db + v * a.dy_ld);
              g[u][0] = q.x; g[u][1] = q.y; g[u][2] = q.z; g[u][3] = q.w;
            }
          } else {
#pragma unroll
            for (int c = 0; c < MAXCO; ++c) g[u][c] = c < a.Cout ? Elem<T>::ld(db + v * a.dy_ld + c) : 0.f;
          }
        } else {
#pragma unroll
          for (int k = 0; k < CPT; ++k) xv[u][k] = 0.f;
#pragma unroll
          for (int c = 0; c < MAXCO; ++c) g[u][c] = 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const bool in = v0 + (int64_t)u * vpi < V;
#pragma unroll
        for (int k = 0; k < CPT; ++k) {
          float t = xv[u][k];
          if (a.x_stats) t = (t - mean[k]) * rstd[k];
          t = act_apply(t, a.act);
          t = in ? Elem<T>::round(t) : 0.f;
#pragma unroll
          for (int c = 0; c < MAXCO; ++c) acc[k][c] = fmaf(g[u][c], t, acc[k][c]);
        }
        if (cg == 0) {
#pragma unroll
          for (int c = 0; c < MAXCO; ++c) bacc[c] += g[u][c];
        }
      }
    }
  }
  // reduce over the voxel lanes that share a channel group: tree in shared memory
  constexpr int NV = CPT * MAXCO;
  float* mine = &s_red[threadIdx.x][0][0];
#pragma unroll
  for (int k = 0; k < CPT; ++k)
#pragma unroll
    for (int c = 0; c < MAXCO; ++c) mine[k * MAXCO + c] = acc[k][c];
  __syncthreads();
  constexpr int RS = (CPT * MAXCO / 4 + 1) * 4;       // row stride in floats
  for (int o = threadIdx.x; o < ngrp * NV; o += 256) {
    const int g2 = o / NV, e = o % NV;
    float sum = 0.f;
    for (int l = 0; l < vpi; ++l) sum += (&s_red[0][0][0])[(l * ngrp + g2) * RS + e];
    const int k = e / MAXCO, c = e % MAXCO;
    if (c < a.Cout) a.part[(int64_t)blockIdx.x * (a.Cout * a.Cin + a.Cout) + (int64_t)c * a.Cin + g2 * CPT + k] = sum;
  }
  if (a.dbias) {
    __syncthreads();
    if (cg == 0 && active) {
#pragma unroll
      for (int c = 0; c < MAXCO; ++c) mine[c] = bacc[c];
    }
    __syncthreads();
    if (threadIdx.x < a.Cout) {
      float sum = 0.f;
      for (int l = 0; l < vpi; ++l) sum += (&s_red[0][0][0])[(l * ngrp) * RS + threadIdx.x];
      a.part[(int64_t)blockIdx.x * (a.Cout * a.Cin + a.Cout) + a.Cout * a.Cin + threadIdx.x] = sum;
    }
  }
}

}  // namespace

namespace {

__global__ void add_slices_kernel(const float* __restrict__ part, int64_t stride, int S, float* __restrict__ dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < S; ++s) acc += part[(int64_t)s * stride + i];
    dst[i] += acc;
  }
}

// which special case serves this weight gradient: 1 = Cin-1 stem, 2 = 1x1x1 head, 0 = none
int small_wgrad_kind(const WgradArgs& a) {
  const int taps = a.kd * a.kh * a.kw;
  const bool k133 = (a.kd == 1 && a.kh == 3 && a.kw == 3), k333 = (a.kd == 3 && a.kh == 3 && a.kw == 3);
  const bool k111 = taps == 1;         // the 1x1x1 projection of SwinUNETR's encoder1 residual block (Cin = 1)
  if (a.x_affine) return 0;            // neither special case has the per-channel input transform
  if (a.Cin == 1 && a.Cout <= 64 && (k133 || k333 || k111) && !a.x_stats && !a.act && !a.dbias) return 1;
  if (taps == 1 && a.Cout <= 16 && a.Cin <= 128 && a.Cin % 8 == 0 && a.x_ld % 8 == 0 && a.x_coff % 8 == 0 &&
      (reinterpret_cast<uintptr_t>(a.x) & 15) == 0) return 2;
  return 0;
}

}  // namespace

int add_slices(const float* part, int64_t stride, int S, float* dst, int64_t n, cudaStream_t st) {
  if (n <= 0) return B200SEG_OK;
  const int64_t want = (n + 255) / 256, cap = (int64_t)B200SEG_NUM_SMS * 8;
  add_slices_kernel<<<(int)(want < cap ? want : cap), 256, 0, st>>>(part, stride, S, dst, n);
  B200_CHECK_LAUNCH("add_slices_kernel");
  return B200SEG_OK;
}

// one slice per block: the stem's dW, or the head's dW followed by its dbias
size_t conv3d_wgrad_small_workspace(const WgradArgs& a) {
  const int kind = small_wgrad_kind(a);
  if (!kind) return 0;
  const int64_t slice = (int64_t)a.Cout * a.Cin * a.kd * a.kh * a.kw + (kind == 2 ? a.Cout : 0);
  return (size_t)B200SEG_NUM_SMS * kSmallGridPerSM * slice * sizeof(float);
}

// returns B200SEG_EUNSUPPORTED when the shape is not one of the special cases; a.part must hold
// conv3d_wgrad_small_workspace(a) bytes
int conv3d_wgrad_small(const WgradArgs& a, int dtype, cudaStream_t st) {
  const int taps = a.kd * a.kh * a.kw;
  const int grid = B200SEG_NUM_SMS * kSmallGridPerSM;
  const bool k133 = (a.kd == 1 && a.kh == 3 && a.kw == 3);
  const bool k111 = taps == 1;
  const int kind = small_wgrad_kind(a);
  if (kind && (!a.part || (reinterpret_cast<uintptr_t>(a.part) & 15))) return B200SEG_EINVAL;
  if (kind == 1) {
    const int th = kWarpsPerBlock * 32;
#define CIN1(TT, KDD, TWO_) do { if (k111) wgrad_cin1_kernel<TT, 1, 1, 1, TWO_><<<grid, th, 0, st>>>(a); \
                                 else wgrad_cin1_kernel<TT, KDD, 3, 3, TWO_><<<grid, th, 0, st>>>(a); } while (0)
#define CIN1_T(TT) do { if (a.Cout > 32) { if (k133) CIN1(TT, 1, true); else CIN1(TT, 3, true); } \
                        else { if (k133) CIN1(TT, 1, false); else CIN1(TT, 3, false); } } while (0)
    if (dtype == B200SEG_F16) CIN1_T(__half); else CIN1_T(float);
#undef CIN1_T
#undef CIN1
    B200_CHECK_LAUNCH("wgrad_cin1_kernel");
    return add_slices(a.part, (int64_t)a.Cout * taps, grid, a.dw, (int64_t)a.Cout * taps, st);
  }
  if (kind == 2) {
    if (dtype == B200SEG_F16) {
      if (a.Cout <= 4) wgrad_head_kernel<__half, 4, 8><<<grid, 256, 0, st>>>(a);
      else wgrad_head_kernel<__half, 16, 2><<<grid, 256, 0, st>>>(a);
    } else {
      if (a.Cout <= 4) wgrad_head_kernel<float, 4, 8><<<grid, 256, 0, st>>>(a);
      else wgrad_head_kernel<float, 16, 2><<<grid, 256, 0, st>>>(a);
    }
    B200_CHECK_LAUNCH("wgrad_head_kernel");
    const int64_t nw = (int64_t)a.Cout * a.Cin;
    const int rc = add_slices(a.part, nw + a.Cout, grid, a.dw, nw, st);
    if (rc || !a.dbias) return rc;
    return add_slices(a.part + nw, nw + a.Cout, grid, a.dbias, a.Cout, st);
  }
  return B200SEG_EUNSUPPORTED;
}

// ===================================================================== forward special cases
namespace {

__device__ __forceinline__ float col_sum16(float (&v)[16], int lane) {   // see conv_tc.cu::column_sum16
#pragma unroll
  for (int i = 0; i < 8; ++i) { const float s = (lane & 16) ? v[i] : v[i + 8], k = (lane & 16) ? v[i + 8] : v[i]; v[i] = k + __shfl_xor_sync(0xffffffffu, s, 16); }
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float s = (lane & 8) ? v[i] : v[i + 4], k = (lane & 8) ? v[i + 4] : v[i]; v[i] = k + __shfl_xor_sync(0xffffffffu, s, 8); }
#pragma unroll
  for (int i = 0; i < 2; ++i) { const float s = (lane & 4) ? v[i] : v[i + 2], k = (lane & 4) ? v[i + 2] : v[i]; v[i] = k + __shfl_xor_sync(0xffffffffu, s, 4); }
  { const float s = (lane & 2) ? v[0] : v[1], k = (lane & 2) ? v[1] : v[0]; v[0] = k + __shfl_xor_sync(0xffffffffu, s, 2); }
  return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

// ---- stem forward: y[v][0..CO) = sum_tap w[tap][co] * x[v+tap]  (Cin == 1, CO = 16*NG in {32, 48, 64}), + IN sums of the
// stored y.  One thread per voxel (2*CO bytes of output), weights in shared memory.  HBM-bound: writes CO channels per
// voxel.  (32 = the UNet / MedFormer stem; 48 = SwinUNETR's encoder1 at feature_size 48, 3x3x3 and its 1x1x1 projection.)
template <typename T, int KD, int KH, int KW, int NG>
__global__ void __launch_bounds__(256)
stem_fwd_kernel(ConvArgs a) {
  constexpr int TAPS = KD * KH * KW, CO = 16 * NG;
  __shared__ float s_w[TAPS][CO];
  __shared__ float s_red[8][CO][2];
  const int64_t V = (int64_t)a.D * a.H * a.W;
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < TAPS * CO; i += 256) s_w[i / CO][i % CO] = Elem<T>::ld((const T*)a.w + i);   // packed [tap][co][1]
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t v = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const bool valid = v < V;
  float acc[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = 0.f;
  if (valid) {
    const int w0 = (int)(v % a.W); const int64_t t = v / a.W; const int h0 = (int)(t % a.H); const int d0 = (int)(t / a.H);
    const T* xb = (const T*)a.x + (int64_t)b * V * a.x_ld + a.x_coff;
#pragma unroll
    for (int zd = 0; zd < KD; ++zd)
#pragma unroll
      for (int zh = 0; zh < KH; ++zh)
#pragma unroll
        for (int zw = 0; zw < KW; ++zw) {
          const int d = d0 + zd - KD / 2, h = h0 + zh - KH / 2, w = w0 + zw - KW / 2;
          float xv = 0.f;
          if ((unsigned)d < (unsigned)a.D && (unsigned)h < (unsigned)a.H && (unsigned)w < (unsigned)a.W)
            xv = Elem<T>::ld(xb + (((int64_t)d * a.H + h) * a.W + w) * a.x_ld);
          const float* wt = s_w[(zd * KH + zh) * KW + zw];
#pragma unroll
          for (int c = 0; c < CO; ++c) acc[c] = fmaf(xv, wt[c], acc[c]);
        }
  }
#pragma unroll
  for (int c = 0; c < CO; ++c) acc[c] = valid ? Elem<T>::round(acc[c]) : 0.f;
  if (valid) {
    T* yp = (T*)a.y + ((int64_t)b * V + v) * a.y_ld + a.y_coff;
#pragma unroll
    for (int c = 0; c < CO; c += 8) st8<T>(yp + c, reinterpret_cast<const float(&)[8]>(acc[c]));
  }
  if (a.y_stats) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      float sq[16];
#pragma unroll
      for (int c = 0; c < 16; ++c) sq[c] = acc[16 * g + c] * acc[16 * g + c];
      const float u = col_sum16(reinterpret_cast<float(&)[16]>(acc[16 * g]), lane), q = col_sum16(sq, lane);
      if ((lane & 1) == 0) {
        const int col = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
        s_red[wid][16 * g + col][0] = u; s_red[wid][16 * g + col][1] = q;
      }
    }
    __syncthreads();
    if (threadIdx.x < 2 * CO) {
      const int c = threadIdx.x >> 1, k = threadIdx.x & 1;
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += (double)s_red[w][c][k];
      atomicAdd(&a.y_stats[((int64_t)b * CO + c) * 2 + k], s);
    }
  }
}

// ---- 1x1x1 conv with few channels on one side (the classifier head forward 32->4 and its data-gradient 4->32):
// one thread per voxel, weights + bias in shared memory, vector loads/stores.  Cin, Cout multiples of 4, <= 64.
template <typename T, int CIN>
__global__ void __launch_bounds__(256)
pointwise_small_kernel(ConvArgs a) {
  extern __shared__ float s_wb[];                 // [Cout][Cin] then [Cout] bias
  const int n = a.Cout * a.Cin;
  for (int i = threadIdx.x; i < n; i += 256) s_wb[i] = Elem<T>::ld((const T*)a.w + i);     // packed [1][Cout][Cin]
  for (int i = threadIdx.x; i < a.Cout; i += 256) s_wb[n + i] = a.bias ? a.bias[i] : 0.f;
  __syncthreads();
  const int64_t total = (int64_t)a.B * a.D * a.H * a.W;
  const int64_t v = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (v >= total) return;
  const T* xp = (const T*)a.x + v * a.x_ld + a.x_coff;
  T* yp = (T*)a.y + v * a.y_ld + a.y_coff;
  float xin[CIN];
#pragma unroll
  for (int c = 0; c < CIN; c += 4) {
    {
      if constexpr (sizeof(T) == 2) {
        const uint2 u = *reinterpret_cast<const uint2*>(xp + c);
        const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        xin[c] = f0.x; xin[c + 1] = f0.y; xin[c + 2] = f1.x; xin[c + 3] = f1.y;
      } else {
        const float4 f = *reinterpret_cast<const float4*>(xp + c);
        xin[c] = f.x; xin[c + 1] = f.y; xin[c + 2] = f.z; xin[c + 3] = f.w;
      }
    }
  }
  for (int co = 0; co < a.Cout; co += 4) {
    float o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float s = s_wb[n + co + q];
      const float4* wr = reinterpret_cast<const float4*>(s_wb + (co + q) * CIN);
#pragma unroll
      for (int c = 0; c < CIN / 4; ++c) {
        const float4 w4 = wr[c];
        s = fmaf(xin[4 * c], w4.x, s); s = fmaf(xin[4 * c + 1], w4.y, s); s = fmaf(xin[4 * c + 2], w4.z, s); s = fmaf(xin[4 * c + 3], w4.w, s);
      }
      o[q] = s;
    }
    if constexpr (sizeof(T) == 2) {
      uint2 u;
      *reinterpret_cast<__half2*>(&u.x) = __floats2half2_rn(o[0], o[1]);
      *reinterpret_cast<__half2*>(&u.y) = __floats2half2_rn(o[2], o[3]);
      *reinterpret_cast<uint2*>(yp + co) = u;
    } else {
      *reinterpret_cast<float4*>(yp + co) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

}  // namespace

int conv3d_fwd_small(const ConvArgs& a, int dtype, cudaStream_t st) {
  const int64_t V = (int64_t)a.D * a.H * a.W;
  const bool plain = !a.x_stats && !a.x_affine && !a.act && !a.res && !a.gx;
  const bool k133 = (a.kd == 1 && a.kh == 3 && a.kw == 3), k333 = (a.kd == 3 && a.kh == 3 && a.kw == 3);
  const bool k111s = (a.kd == 1 && a.kh == 1 && a.kw == 1);
  // stem_fwd_kernel stores y in 16-byte groups of 8 channels; pointwise_small_kernel moves x and y in 4-channel vectors
  const uintptr_t xa = reinterpret_cast<uintptr_t>(a.x), ya = reinterpret_cast<uintptr_t>(a.y);
  const uintptr_t vec4 = 4 * (dtype == B200SEG_F16 ? sizeof(__half) : sizeof(float));
  if (plain && !a.bias && a.Cin == 1 && (a.Cout == 32 || a.Cout == 48 || a.Cout == 64) && (k133 || k333 || k111s) && (a.y_ld % 8 == 0) &&
      (a.y_coff % 8 == 0) && ya % 16 == 0) {
    dim3 grid(ceil_div(V, 256), a.B);
#define STEM(TT, NG)                                                                   \
  do {                                                                                 \
    if (k133) stem_fwd_kernel<TT, 1, 3, 3, NG><<<grid, 256, 0, st>>>(a);               \
    else if (k333) stem_fwd_kernel<TT, 3, 3, 3, NG><<<grid, 256, 0, st>>>(a);          \
    else stem_fwd_kernel<TT, 1, 1, 1, NG><<<grid, 256, 0, st>>>(a);                    \
  } while (0)
#define STEM_T(TT) do { if (a.Cout == 32) STEM(TT, 2); else if (a.Cout == 48) STEM(TT, 3); else STEM(TT, 4); } while (0)
    if (dtype == B200SEG_F16) STEM_T(__half); else STEM_T(float);
#undef STEM_T
#undef STEM
    B200_CHECK_LAUNCH("stem_fwd_kernel");
    return B200SEG_OK;
  }
  const bool k111 = (a.kd == 1 && a.kh == 1 && a.kw == 1);
  if (plain && !a.y_stats && k111 && (a.Cin == 4 || a.Cin == 8 || a.Cin == 16 || a.Cin == 32 || a.Cin == 64) &&
      a.Cout % 4 == 0 && a.Cout <= 64 && a.x_ld % 4 == 0 && a.x_coff % 4 == 0 && a.y_ld % 4 == 0 && a.y_coff % 4 == 0 &&
      xa % vec4 == 0 && ya % vec4 == 0) {
    const int64_t total = (int64_t)a.B * V;
    const size_t sm = sizeof(float) * ((size_t)a.Cout * a.Cin + a.Cout);
    const int grid = ceil_div(total, 256);
#define PW(TT, CI) pointwise_small_kernel<TT, CI><<<grid, 256, sm, st>>>(a)
#define PWT(TT) switch (a.Cin) { case 4: PW(TT, 4); break; case 8: PW(TT, 8); break; case 16: PW(TT, 16); break; case 32: PW(TT, 32); break; default: PW(TT, 64); }
    if (dtype == B200SEG_F16) { PWT(__half) } else { PWT(float) }
#undef PWT
#undef PW
    B200_CHECK_LAUNCH("pointwise_small_kernel");
    return B200SEG_OK;
  }
  return B200SEG_EUNSUPPORTED;
}
