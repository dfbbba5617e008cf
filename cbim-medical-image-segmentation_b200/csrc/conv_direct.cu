// conv_direct.cu — CUDA-core (FFMA, fp32 accumulate) conv3d forward / data-gradient / weight-gradient.
// This is (a) the fp32 parity path, (b) the path for shapes that are not dense contractions
// (Cin=1 stem, Cout=4/14 heads: SURVEY.md §8d "HBM bandwidth" rows) and (c) the cross-check for the
// wgmma implicit-GEMM kernels in conv_tc.cu.  Same fusions as the tensor-core path: InstanceNorm
// normalise + ReLU of the INPUT applied in the loader, bias / residual / IN-sums in the epilogue,
// ReLU-mask + IN-backward sums in the dgrad epilogue.
// Reference call sites: nn.Conv3d in conv_layers.py:29-38 (ConvNormAct), unet_utils.py:14 (stem),
// unet.py:47 (outc); autograd of the same (train_ddp.py:193/208).
#include "common.cuh"
#include "conv_args.h"
#include "tc_common.cuh"

namespace {

constexpr int kVoxTile = 128;   // output voxels per block (one per thread)
constexpr int kCoTile = 16;     // output channels per block

template <typename T, int CIV> struct InVec;
template <typename T> struct InVec<T, 8> {
  static __device__ __forceinline__ void ld(const T* p, float (&v)[8]) { ld8<T>(p, v); }
};
template <typename T> struct InVec<T, 1> {
  static __device__ __forceinline__ void ld(const T* p, float (&v)[1]) { v[0] = Elem<T>::ld(p); }
};


// grid: (ceil(V/128), ceil(Cout/16), B)   block: 128
template <typename T, int CIV>
__global__ void __launch_bounds__(kVoxTile)
conv_fwd_direct_kernel(ConvArgs a) {
  extern __shared__ float smem[];
  const int taps = a.kd * a.kh * a.kw;
  float* s_w = smem;                                  // [taps][kCoTile][CIV]
  float* s_mean = s_w + taps * kCoTile * CIV;         // [Cin]
  float* s_rstd = s_mean + a.Cin;                     // [Cin]
  float* s_red = s_rstd + a.Cin;                      // [4 warps][kCoTile][2]

  const int b = blockIdx.z;
  const int co0 = blockIdx.y * kCoTile;
  const int64_t V = (int64_t)a.D * a.H * a.W;
  const int64_t v = (int64_t)blockIdx.x * kVoxTile + threadIdx.x;
  const bool valid = v < V;
  int w0 = 0, h0 = 0, d0 = 0;
  if (valid) { w0 = (int)(v % a.W); int64_t t = v / a.W; h0 = (int)(t % a.H); d0 = (int)(t / a.H); }

  const bool norm = a.x_stats != nullptr;
  const bool affine = a.x_affine != nullptr;        // per-channel transform: s_mean holds the scale, s_rstd the shift
  if (norm) {
    for (int c = threadIdx.x; c < a.Cin; c += kVoxTile)
      stats_to_mean_rstd(a.x_stats + ((int64_t)b * a.Cin + c) * 2, (double)V, a.eps, s_mean[c], s_rstd[c]);
  } else if (affine) {
    for (int c = threadIdx.x; c < a.Cin; c += kVoxTile) { s_mean[c] = a.x_affine[2 * c]; s_rstd[c] = a.x_affine[2 * c + 1]; }
  }
  const T* xb = (const T*)a.x + (int64_t)b * V * a.x_ld + a.x_coff;
  const T* wp = (const T*)a.w;
  const int pd = a.kd / 2, ph = a.kh / 2, pw = a.kw / 2;

  float acc[kCoTile];
#pragma unroll
  for (int i = 0; i < kCoTile; ++i) acc[i] = 0.f;

  for (int ci0 = 0; ci0 < a.Cin; ci0 += CIV) {
    __syncthreads();
    for (int i = threadIdx.x; i < taps * kCoTile * CIV; i += kVoxTile) {
      int j = i % CIV, co = (i / CIV) % kCoTile, tap = i / (CIV * kCoTile);
      float wv = 0.f;
      if (co0 + co < a.Cout) wv = Elem<T>::ld(wp + ((int64_t)tap * a.Cout + co0 + co) * a.Cin + ci0 + j);
      s_w[i] = wv;
    }
    __syncthreads();
    if (valid) {
      int tap = 0;
      for (int zd = 0; zd < a.kd; ++zd) {
        int d = d0 + zd - pd;
        for (int zh = 0; zh < a.kh; ++zh) {
          int h = h0 + zh - ph;
          for (int zw = 0; zw < a.kw; ++zw, ++tap) {
            int w = w0 + zw - pw;
            if ((unsigned)d >= (unsigned)a.D || (unsigned)h >= (unsigned)a.H || (unsigned)w >= (unsigned)a.W) continue;
            float xv[CIV];
            InVec<T, CIV>::ld(xb + (((int64_t)d * a.H + h) * a.W + w) * a.x_ld + ci0, xv);
            if (norm) {
#pragma unroll
              for (int j = 0; j < CIV; ++j) xv[j] = (xv[j] - s_mean[ci0 + j]) * s_rstd[ci0 + j];
            } else if (affine) {
#pragma unroll
              for (int j = 0; j < CIV; ++j) xv[j] = fmaf(xv[j], s_mean[ci0 + j], s_rstd[ci0 + j]);
            }
            if (a.act) {
#pragma unroll
              for (int j = 0; j < CIV; ++j) xv[j] = act_apply(xv[j], a.act);
            }
            // operands are rounded to the storage dtype exactly as the tensor-core path feeds them
#pragma unroll
            for (int j = 0; j < CIV; ++j) xv[j] = Elem<T>::round(xv[j]);
            const float* wt = s_w + tap * kCoTile * CIV;
#pragma unroll
            for (int co = 0; co < kCoTile; ++co) {
#pragma unroll
              for (int j = 0; j < CIV; ++j) acc[co] = fmaf(xv[j], wt[co * CIV + j], acc[co]);
            }
          }
        }
      }
    }
  }

  // ---- epilogue
  const bool dgrad = a.gx != nullptr;
  float s1[kCoTile], s2[kCoTile];
#pragma unroll
  for (int co = 0; co < kCoTile; ++co) { s1[co] = 0.f; s2[co] = 0.f; }
  if (valid) {
    const int64_t gv = (int64_t)b * V + v;
    T* yp = (T*)a.y + gv * a.y_ld + a.y_coff + co0;
    const T* rp = a.res ? (const T*)a.res + gv * a.r_ld + a.r_coff + co0 : nullptr;
    const T* gp = dgrad ? (const T*)a.gx + gv * a.gx_ld + a.gx_coff + co0 : nullptr;
#pragma unroll
    for (int co = 0; co < kCoTile; ++co) {
      if (co0 + co >= a.Cout) break;
      float r = acc[co];
      if (a.bias) r += a.bias[co0 + co];
      if (dgrad) {
        float mean, rstd;
        stats_to_mean_rstd(a.g_stats + ((int64_t)b * a.Cout + co0 + co) * 2, (double)V, a.g_eps, mean, rstd);
        float hx = (Elem<T>::ld(gp + co) - mean) * rstd;
        r *= act_grad(hx, a.g_act);
        r = Elem<T>::round(r);
        s1[co] = r; s2[co] = r * hx;
      } else {
        r = Elem<T>::round(r);
        if (rp) r = Elem<T>::round(r + Elem<T>::ld(rp + co));
        s1[co] = r; s2[co] = r * r;
      }
      Elem<T>::st(yp + co, r);
    }
  }
  if (a.y_stats) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int co = 0; co < kCoTile; ++co) {
      float u = warp_sum(s1[co]), q = warp_sum(s2[co]);
      if (lane == 0) { s_red[(wid * kCoTile + co) * 2] = u; s_red[(wid * kCoTile + co) * 2 + 1] = q; }
    }
    __syncthreads();
    if (threadIdx.x < kCoTile * 2) {
      int co = threadIdx.x >> 1, k = threadIdx.x & 1;
      if (co0 + co < a.Cout) {
        double s = 0.0;
        for (int w = 0; w < kVoxTile / 32; ++w) s += (double)s_red[(w * kCoTile + co) * 2 + k];
        atomicAdd(&a.y_stats[((int64_t)b * a.Cout + co0 + co) * 2 + k], s);
      }
    }
  }
}

// ---------------------------------------------------------------- weight gradient (direct)
constexpr int kWT = 32;       // co / ci tile
constexpr int kWV = 32;       // voxels staged per iteration

// grid: (voxel chunks, taps, B * coTiles * ciTiles)   block: 256 = 16x16 threads, 2x2 outputs each
template <typename T>
__global__ void __launch_bounds__(256)
conv_wgrad_direct_kernel(WgradArgs a) {
  __shared__ float s_dy[kWV][kWT + 1];
  __shared__ float s_a[kWV][kWT + 1];
  const int taps = a.kd * a.kh * a.kw;
  const int tap = blockIdx.y;
  const int coT = (a.Cout + kWT - 1) / kWT, ciT = (a.Cin + kWT - 1) / kWT;
  int z = blockIdx.z;
  const int cit = z % ciT; z /= ciT;
  const int cot = z % coT; z /= coT;
  const int b = z;
  const int co0 = cot * kWT, ci0 = cit * kWT;
  const int64_t V = (int64_t)a.D * a.H * a.W;
  const int64_t v0 = (int64_t)blockIdx.x * a.vox_per_block;
  int64_t v1 = v0 + a.vox_per_block; if (v1 > V) v1 = V;
  const int zd = tap / (a.kh * a.kw) - a.kd / 2, zh = (tap / a.kw) % a.kh - a.kh / 2, zw = tap % a.kw - a.kw / 2;
  const bool norm = a.x_stats != nullptr, affine = a.x_affine != nullptr;
  const T* xb = (const T*)a.x + (int64_t)b * V * a.x_ld + a.x_coff;
  const T* dyb = (const T*)a.dy + (int64_t)b * V * a.dy_ld + a.dy_coff;

  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  float bacc = 0.f;
  // this thread's fixed channel for the staging loads: element e = threadIdx.x + 256*k -> (vox e/32, ch e%32)
  const int lc = threadIdx.x & 31;
  float mean = 0.f, rstd = 1.f;
  if (norm && ci0 + lc < a.Cin)
    stats_to_mean_rstd(a.x_stats + ((int64_t)b * a.Cin + ci0 + lc) * 2, (double)V, a.eps, mean, rstd);
  float scale = 1.f, shift = 0.f;
  if (affine && ci0 + lc < a.Cin) { scale = a.x_affine[2 * (ci0 + lc)]; shift = a.x_affine[2 * (ci0 + lc) + 1]; }

  for (int64_t vb = v0; vb < v1; vb += kWV) {
    __syncthreads();
#pragma unroll
    for (int k = 0; k < (kWV * kWT) / 256; ++k) {
      int e = threadIdx.x + 256 * k;
      int vl = e >> 5;
      int64_t v = vb + vl;
      float dv = 0.f, av = 0.f;
      if (v < v1) {
        if (co0 + lc < a.Cout) dv = Elem<T>::ld(dyb + v * a.dy_ld + co0 + lc);
        if (ci0 + lc < a.Cin) {
          int w = (int)(v % a.W); int64_t t = v / a.W; int h = (int)(t % a.H); int d = (int)(t / a.H);
          d += zd; h += zh; w += zw;
          if ((unsigned)d < (unsigned)a.D && (unsigned)h < (unsigned)a.H && (unsigned)w < (unsigned)a.W) {
            av = Elem<T>::ld(xb + (((int64_t)d * a.H + h) * a.W + w) * a.x_ld + ci0 + lc);
            if (norm) av = (av - mean) * rstd;
            else if (affine) av = fmaf(av, scale, shift);
            av = act_apply(av, a.act);
            av = Elem<T>::round(av);
          }
        }
      }
      s_dy[vl][lc] = dv;
      s_a[vl][lc] = av;
    }
    __syncthreads();
#pragma unroll 8
    for (int vl = 0; vl < kWV; ++vl) {
      float d0 = s_dy[vl][2 * ty], d1 = s_dy[vl][2 * ty + 1];
      float a0 = s_a[vl][2 * tx], a1 = s_a[vl][2 * tx + 1];
      acc[0][0] = fmaf(d0, a0, acc[0][0]); acc[0][1] = fmaf(d0, a1, acc[0][1]);
      acc[1][0] = fmaf(d1, a0, acc[1][0]); acc[1][1] = fmaf(d1, a1, acc[1][1]);
    }
    if (a.dbias && tap == 0 && cit == 0 && threadIdx.x < kWT) {
      for (int vl = 0; vl < kWV; ++vl) bacc += s_dy[vl][threadIdx.x];
    }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      int co = co0 + 2 * ty + i, ci = ci0 + 2 * tx + j;
      if (co < a.Cout && ci < a.Cin) atomicAdd(&a.dw[((int64_t)co * a.Cin + ci) * taps + tap], acc[i][j]);
    }
  if (a.dbias && tap == 0 && cit == 0 && threadIdx.x < kWT && co0 + threadIdx.x < a.Cout)
    atomicAdd(&a.dbias[co0 + threadIdx.x], bacc);
}

// packed position of element i of a [Cout][Cin][taps] fp32 parameter (see b200seg_pack_weight).  layout: 0 = DIRECT,
// 1 = TC (16-byte planes of 8 fp16 channels), 2 = TC_TF32 (16-byte planes of 4 fp32 channels)
__device__ __forceinline__ int64_t pack_index(int64_t i, int Cout, int Cin, int taps, int transpose_flip, int co_off,
                                              int co_total, int layout) {
  // virtual packed tensor [taps][R][Cc]: fwd: R = co_total rows (cout), Cc = Cin cols; dgrad operand: R = Cin, Cc = co_total
  const int R = transpose_flip ? Cin : co_total, Cc = transpose_flip ? co_total : Cin;
  const int tap = (int)(i % taps); const int64_t t = i / taps; const int ci = (int)(t % Cin); const int co = (int)(t / Cin);
  const int tp = transpose_flip ? taps - 1 - tap : tap;
  const int row = transpose_flip ? ci : co_off + co;
  const int col = transpose_flip ? co_off + co : ci;
  if (!layout) return ((int64_t)tp * R + row) * Cc + col;
  const int epp = layout == 2 ? 4 : 8;
  const int NT = tc_pick_nt(R), KC = layout == 2 ? tc_pick_kc_tf32(Cc) : tc_pick_kc(Cc), NKC = Cc / KC;
  const int ntile = row / NT, nn = row % NT, kc = col / KC, kk = col % KC, kp = kk / epp, e = kk % epp;
  return ((((int64_t)(ntile * taps + tp) * NKC + kc) * (KC / epp) + kp) * NT + nn) * epp + e;
}

// the value stored for weight v: TF32 operands are rounded once here (cvt.rna), so the tensor core sees exact TF32
__device__ __forceinline__ float pack_value(float v, int layout) { return layout == 2 ? tc::round_tf32(v) : v; }

template <typename T>
__global__ void pack_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, T* __restrict__ wp,
                                   int transpose_flip, int co_off, int co_total, int layout) {
  int64_t n = (int64_t)Cout * Cin * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    Elem<T>::st(wp + pack_index(i, Cout, Cin, taps, transpose_flip, co_off, co_total, layout), pack_value(w[i], layout));
}

// Multi-tensor variant: every conv weight of a model is re-packed by ONE launch per forward (the per-weight
// launches were ~90 x 12 us per step).  jobs[j] = {w, out, Cout, Cin, taps, dtype, transpose_flip, co_off, co_total,
// layout (0 / 1 / 2, as pack_index)}; one block per chunk.  chunks[c] = {job, code}:
//   code >= 0 : ELEMENT chunk — kPackChunk consecutive source elements from `code`, each written to its packed
//               position (2-byte scattered stores: 580 us per forward for the 40 M-parameter ResUNet, 10x the HBM time);
//   code <  0 : TILE chunk (Cout, Cin multiples of 8) — -(code+1) = co0 * 65536 + ci0: eight output channels x up to
//               pack_tile_ci(taps) input channels x all taps are staged through shared memory (coalesced row reads) and
//               written as 16-byte groups of the packed image's contiguous 8-element runs (8 consecutive ci of one
//               (co, tap) in the forward image, 8 consecutive co of one (ci, tap) in the flipped-transposed one; in
//               the TC_TF32 image such a run is two 4-element planes, stored as two 16-byte groups).
constexpr int kPackChunk = 4096;
__host__ __device__ inline int pack_tile_ci(int taps) {       // input channels per tile: largest multiple of 8 with 8*ci*taps <= kPackChunk
  const int c = kPackChunk / (8 * taps) / 8 * 8;
  return c;                                                     // 0 -> no tile path for this kernel size
}

template <typename T>
__device__ __forceinline__ void pack_tile(const float* __restrict__ w, T* __restrict__ o, int Cout, int Cin, int taps, int tf, int co_off,
                                          int co_total, int layout, int co0, int ci0, float* tile) {
  const int cit = min(pack_tile_ci(taps), Cin - ci0), seg = cit * taps;
  for (int idx = threadIdx.x; idx < 8 * seg; idx += 256) {
    const int r = idx / seg, k = idx - r * seg;
    tile[idx] = w[((int64_t)(co0 + r) * Cin + ci0) * taps + k];
  }
  __syncthreads();
  for (int g = threadIdx.x; g < seg; g += 256) {
    float v[8];
    int64_t first;                          // source index of the group's first element (-> its packed position)
    if (!tf) {                              // 8 consecutive ci of (co0 + r, tap); r fastest: neighbouring threads write neighbouring rows
      const int r = g & 7, q = g >> 3, tap = q % taps, c8 = q / taps;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = tile[r * seg + (c8 * 8 + e) * taps + tap];
      first = ((int64_t)(co0 + r) * Cin + ci0 + c8 * 8) * taps + tap;
    } else {                                // 8 consecutive co of (ci0 + ci, tap); ci fastest
      const int ci = g % cit, tap = g / cit;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = tile[e * seg + ci * taps + tap];
      first = ((int64_t)co0 * Cin + ci0 + ci) * taps + tap;
    }
    if constexpr (sizeof(T) == 4) {
      if (layout == 2) {
        const int64_t step = 4 * (tf ? (int64_t)Cin * taps : (int64_t)taps);   // source distance of the run's 5th element
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float4*>(o + pack_index(first + h * step, Cout, Cin, taps, tf, co_off, co_total, layout)) =
              make_float4(pack_value(v[4 * h], 2), pack_value(v[4 * h + 1], 2), pack_value(v[4 * h + 2], 2), pack_value(v[4 * h + 3], 2));
        continue;
      }
    }
    st8<T>(o + pack_index(first, Cout, Cin, taps, tf, co_off, co_total, layout), v);
  }
}

__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const int64_t* __restrict__ jobs, const int64_t* __restrict__ chunks) {
  __shared__ float tile[kPackChunk];
  const int64_t* c = chunks + 2 * (int64_t)blockIdx.x;
  const int64_t* j = jobs + 10 * c[0];
  const float* w = reinterpret_cast<const float*>(j[0]);
  const int Cout = (int)j[2], Cin = (int)j[3], taps = (int)j[4], dtype = (int)j[5], tf = (int)j[6], co_off = (int)j[7],
            co_total = (int)j[8], layout = (int)j[9];
  if (c[1] < 0) {
    const int64_t code = -(c[1] + 1);
    const int co0 = (int)(code >> 16), ci0 = (int)(code & 65535);
    if (dtype == B200SEG_F16) pack_tile<__half>(w, reinterpret_cast<__half*>(j[1]), Cout, Cin, taps, tf, co_off, co_total, layout, co0, ci0, tile);
    else pack_tile<float>(w, reinterpret_cast<float*>(j[1]), Cout, Cin, taps, tf, co_off, co_total, layout, co0, ci0, tile);
    return;
  }
  const int64_t n = (int64_t)Cout * Cin * taps, i0 = c[1];
  const int64_t i1 = i0 + kPackChunk < n ? i0 + kPackChunk : n;
  if (dtype == B200SEG_F16) {
    __half* o = reinterpret_cast<__half*>(j[1]);
    for (int64_t i = i0 + threadIdx.x; i < i1; i += 256) o[pack_index(i, Cout, Cin, taps, tf, co_off, co_total, layout)] = __float2half_rn(w[i]);
  } else {
    float* o = reinterpret_cast<float*>(j[1]);
    for (int64_t i = i0 + threadIdx.x; i < i1; i += 256) o[pack_index(i, Cout, Cin, taps, tf, co_off, co_total, layout)] = pack_value(w[i], layout);
  }
}

}  // namespace

int conv3d_fwd_direct(const ConvArgs& a, int dtype, cudaStream_t st) {
  const int taps = a.kd * a.kh * a.kw;
  const int64_t V = (int64_t)a.D * a.H * a.W;
  dim3 grid(ceil_div(V, kVoxTile), ceil_div(a.Cout, kCoTile), a.B);
  bool civ8 = (a.Cin % 8 == 0) && (a.x_ld % 8 == 0) && (a.x_coff % 8 == 0) && ((reinterpret_cast<uintptr_t>(a.x) % 16) == 0);
  int civ = civ8 ? 8 : 1;
  size_t sm = sizeof(float) * ((size_t)taps * kCoTile * civ + 2 * a.Cin + 4 * kCoTile * 2);
  if (sm > 200 * 1024) return B200SEG_EUNSUPPORTED;
#define LAUNCH(TT, CIVV)                                                                                          \
  do {                                                                                                            \
    if (sm > 48 * 1024) cudaFuncSetAttribute(conv_fwd_direct_kernel<TT, CIVV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); \
    conv_fwd_direct_kernel<TT, CIVV><<<grid, kVoxTile, sm, st>>>(a);                                              \
  } while (0)
  if (dtype == B200SEG_F16) { if (civ8) LAUNCH(__half, 8); else LAUNCH(__half, 1); }
  else if (dtype == B200SEG_F32) { if (civ8) LAUNCH(float, 8); else LAUNCH(float, 1); }
  else return B200SEG_EINVAL;
#undef LAUNCH
  B200_CHECK_LAUNCH("conv_fwd_direct_kernel");
  return B200SEG_OK;
}

int conv3d_wgrad_direct(const WgradArgs& a_in, int dtype, cudaStream_t st) {
  WgradArgs a = a_in;
  const int B = a.B, D = a.D, H = a.H, W = a.W, Cin = a.Cin, Cout = a.Cout, kd = a.kd, kh = a.kh, kw = a.kw;
  const int64_t V = (int64_t)D * H * W;
  const int taps = kd * kh * kw;
  const int coT = (Cout + kWT - 1) / kWT, ciT = (Cin + kWT - 1) / kWT;
  int64_t zblocks = (int64_t)B * coT * ciT;
  if (zblocks > 65535 || taps > 65535) return B200SEG_EUNSUPPORTED;
  // enough voxel chunks to fill the machine, but >= 1024 voxels each to amortise the atomics
  int64_t want = (int64_t)B200SEG_NUM_SMS * 8 / (taps * zblocks) + 1;
  int64_t vpb = (V + want - 1) / want;
  if (vpb < 1024) vpb = 1024;
  vpb = (vpb + kWV - 1) / kWV * kWV;
  a.vox_per_block = (int)vpb;
  dim3 grid(ceil_div(V, vpb), taps, (unsigned)zblocks);
  if (dtype == B200SEG_F16) conv_wgrad_direct_kernel<__half><<<grid, 256, 0, st>>>(a);
  else if (dtype == B200SEG_F32) conv_wgrad_direct_kernel<float><<<grid, 256, 0, st>>>(a);
  else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("conv_wgrad_direct_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_pack_weight(const float* w, int Cout, int Cin, int taps, void* w_packed, int dtype,
                                   int transpose_flip, int co_off, int co_total, int layout, void* stream) {
  if (!w || !w_packed || Cout <= 0 || Cin <= 0 || taps <= 0 || co_off < 0 || co_off + Cout > co_total) return B200SEG_EINVAL;
  if (layout != B200SEG_ALGO_DIRECT && layout != B200SEG_ALGO_TC && layout != B200SEG_ALGO_TC_TF32) return B200SEG_EINVAL;
  const int tc = layout == B200SEG_ALGO_TC ? 1 : layout == B200SEG_ALGO_TC_TF32 ? 2 : 0;     // pack_index layout code
  if (tc) {
    const int R = transpose_flip ? Cin : co_total, Cc = transpose_flip ? co_total : Cin;
    if (!tc_pick_nt(R) || !(tc == 1 ? tc_pick_kc(Cc) : tc_pick_kc_tf32(Cc)) || dtype != (tc == 1 ? B200SEG_F16 : B200SEG_F32))
      return B200SEG_EUNSUPPORTED;
  }
  cudaStream_t st = as_stream(stream);
  int64_t n = (int64_t)Cout * Cin * taps;
  int grid = ceil_div(n, 256); if (grid > B200SEG_NUM_SMS * 8) grid = B200SEG_NUM_SMS * 8;
  if (dtype == B200SEG_F16) pack_weight_kernel<__half><<<grid, 256, 0, st>>>(w, Cout, Cin, taps, (__half*)w_packed, transpose_flip, co_off, co_total, tc);
  else if (dtype == B200SEG_F32) pack_weight_kernel<float><<<grid, 256, 0, st>>>(w, Cout, Cin, taps, (float*)w_packed, transpose_flip, co_off, co_total, tc);
  else return B200SEG_EINVAL;
  B200_CHECK_LAUNCH("pack_weight_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_pack_chunk_elems(void) { return kPackChunk; }
// input channels per TILE chunk for a `taps`-tap kernel (0: use element chunks); see pack_weights_multi_kernel
extern "C" int b200seg_pack_tile_ci(int taps) { return taps > 0 ? pack_tile_ci(taps) : 0; }

extern "C" int b200seg_pack_weights_multi(const int64_t* jobs_dev, const int64_t* chunks_dev, int nchunks, void* stream) {
  if (nchunks == 0) return B200SEG_OK;
  if (!jobs_dev || !chunks_dev || nchunks < 0) return B200SEG_EINVAL;
  pack_weights_multi_kernel<<<nchunks, 256, 0, as_stream(stream)>>>(jobs_dev, chunks_dev);
  B200_CHECK_LAUNCH("pack_weights_multi_kernel");
  return B200SEG_OK;
}
