// medformer_small.cu — the bandwidth-/latency-bound MedFormer operators that are not convolutions:
//   space_to_depth      PatchMerging's strided-slice gather        medformer_utils.py:165-171
//   mapgen_fwd/bwd      SemanticMapGeneration softmax-over-voxels  medformer_utils.py:216-228
//   se_gate_fwd/bwd     SEBlock squeeze/excitation                 conv_layers.py:159-174
//   channel_scale_*     x * gate                                   conv_layers.py:174
//   layernorm_fwd/bwd   nn.LayerNorm in PreNorm                    trans_layers.py:36-41
//   gelu_fwd/bwd        nn.GELU in Mlp                             trans_layers.py:22,28
//   mhsa_fwd/bwd        Attention over the fused map tokens        trans_layers.py:45-100
// All tensors channels-last; activations in T (fp16/fp32), parameters and statistics fp32/fp64.
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ space to depth (and its inverse)
template <typename T, int VEC>
__global__ void s2d_kernel(const T* __restrict__ x, T* __restrict__ y, int B, int Do, int Ho, int Wo, int C,
                           int sd, int sh, int sw, int reverse) {
  // forward: y[b,d,h,w,(q,c)] = x[b, d*sd+i, h*sh+j, w*sw+k, c],  q = (i*sh + j)*sw + k   (:165-169 nesting)
  // VEC = 8 channels per thread (16-byte accesses) when C % 8 == 0, else 1 (e.g. the single-channel SwinUNETR input)
  const int ncg = C / VEC, Q = sd * sh * sw;
  const int64_t total = (int64_t)B * Do * Ho * Wo * Q * ncg;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = it;
    const int cg = (int)(r % ncg); r /= ncg;
    const int q = (int)(r % Q); r /= Q;
    const int w = (int)(r % Wo); r /= Wo;
    const int h = (int)(r % Ho); r /= Ho;
    const int d = (int)(r % Do); const int b = (int)(r / Do);
    const int k = q % sw, j = (q / sw) % sh, i = q / (sw * sh);
    const int64_t xo = ((((int64_t)b * Do * sd + d * sd + i) * (Ho * sh) + h * sh + j) * (Wo * sw) + w * sw + k) * C + cg * VEC;
    const int64_t yo = ((((int64_t)b * Do + d) * Ho + h) * Wo + w) * ((int64_t)Q * C) + (int64_t)q * C + cg * VEC;
    if constexpr (VEC == 8) {
      float v[8];
      if (!reverse) { ld8<T>(x + xo, v); st8<T>(y + yo, v); }
      else { ld8<T>(y + yo, v); st8<T>(const_cast<T*>(x) + xo, v); }
    } else {
      if (!reverse) y[yo] = x[xo]; else const_cast<T*>(x)[xo] = y[yo];
    }
  }
}

// ------------------------------------------------------------------ semantic map generation
constexpr int MG_T = 128, MG_KCAP = 80, MG_CC = 48;   // kernels are built for 32, 64 and 80 map codes (80: ACDC's 72)

struct MgArgs {
  const void* f; int f_ld, f_coff; const void* wl; int w_ld, w_coff;   // features [B][N][*], logits [B][N][*]
  void* map; int map_ld;                                                // [B][K][C]
  float* colstat; float* partial;                                       // [B][K][2]; [B][nblk][K][2+C]
  const void* dmap; void* df; int df_ld, df_coff; void* dwl; int dw_ld, dw_coff, dw_pad;
  int B, K, C; int64_t N;
};

template <typename T, int MG_K>
__global__ void __launch_bounds__(MG_T) mapgen_fwd_kernel(MgArgs a) {
  extern __shared__ float mg_sm[];
  float (*s_e)[MG_K + 1] = reinterpret_cast<float (*)[MG_K + 1]>(mg_sm);
  float (*s_f)[MG_CC + 1] = reinterpret_cast<float (*)[MG_CC + 1]>(mg_sm + MG_T * (MG_K + 1));
  float (*s_max)[MG_K] = reinterpret_cast<float (*)[MG_K]>(mg_sm + MG_T * (MG_K + 1) + MG_T * (MG_CC + 1));
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, K = a.K, C = a.C;
  const int64_t i = (int64_t)blockIdx.x * MG_T + tid;
  const bool valid = i < a.N;
  const T* wrow = (const T*)a.wl + ((int64_t)b * a.N + i) * a.w_ld + a.w_coff;
  // the 64- and 32-code builds keep the row's logits in registers; the 80-code build stages them in its own row of
  // s_e instead (80 live logits next to the shuffles spill)
  float lg[MG_K > 64 ? 1 : MG_K];
  if constexpr (MG_K > 64) {
    for (int k = 0; k < MG_K; ++k) s_e[tid][k] = (valid && k < K) ? Elem<T>::ld(wrow + k) : -INFINITY;
  } else {
#pragma unroll
    for (int k = 0; k < MG_K; ++k) lg[k] = (valid && k < K) ? Elem<T>::ld(wrow + k) : -INFINITY;
  }
#pragma unroll
  for (int k = 0; k < MG_K; ++k) {
    float m;
    if constexpr (MG_K > 64) m = s_e[tid][k]; else m = lg[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_max[wid][k] = m;
  }
  __syncthreads();
  if (tid < MG_K) s_max[4][tid] = fmaxf(fmaxf(s_max[0][tid], s_max[1][tid]), fmaxf(s_max[2][tid], s_max[3][tid]));
  __syncthreads();
  if constexpr (MG_K > 64) {
    for (int k = 0; k < MG_K; ++k) s_e[tid][k] = (valid && k < K) ? __expf(s_e[tid][k] - s_max[4][k]) : 0.f;
  } else {
#pragma unroll
    for (int k = 0; k < MG_K; ++k) s_e[tid][k] = (valid && k < K) ? __expf(lg[k] - s_max[4][k]) : 0.f;
  }
  float* pb = a.partial + (((int64_t)b * gridDim.x + blockIdx.x) * K) * (2 + C);
  __syncthreads();
  if (tid < K) {
    float s = 0.f;
    for (int r = 0; r < MG_T; ++r) s += s_e[r][tid];
    pb[tid * (2 + C)] = s_max[4][tid]; pb[tid * (2 + C) + 1] = s;
  }
  const T* frow = (const T*)a.f + ((int64_t)b * a.N + i) * a.f_ld + a.f_coff;
  for (int c0 = 0; c0 < C; c0 += MG_CC) {
    const int cc = min(MG_CC, C - c0);
    __syncthreads();
    for (int c = 0; c < cc; ++c) s_f[tid][c] = valid ? Elem<T>::ld(frow + c0 + c) : 0.f;
    __syncthreads();
    for (int o = tid; o < K * cc; o += MG_T) {
      const int k = o / cc, c = o % cc;
      float acc = 0.f;
      for (int r = 0; r < MG_T; ++r) acc = fmaf(s_e[r][k], s_f[r][c], acc);
      pb[k * (2 + C) + 2 + c0 + c] = acc;
    }
  }
}

// grid (K, B): threads stride the channels; every thread runs the online max/sum over the blocks itself
// (reads of q[0], q[1] are warp-broadcasts), so no serial prologue.
template <typename T>
__global__ void mapgen_merge_kernel(MgArgs a, int nblk) {
  const int k = blockIdx.x, b = blockIdx.y, K = a.K, C = a.C;
  const float* pb = a.partial + ((int64_t)b * nblk * K + k) * (2 + C);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float m = -INFINITY, sum = 0.f, acc = 0.f;
    for (int n = 0; n < nblk; ++n) {
      const float* q = pb + (int64_t)n * K * (2 + C);
      const float mk = q[0];
      if (mk > m) { const float sc = __expf(m - mk); sum *= sc; acc *= sc; m = mk; }
      const float e = __expf(mk - m);
      sum = fmaf(q[1], e, sum); acc = fmaf(q[2 + c], e, acc);
    }
    Elem<T>::st((T*)a.map + ((int64_t)b * K + k) * a.map_ld + c, acc / sum);
    if (c == 0) { a.colstat[((int64_t)b * K + k) * 2] = m; a.colstat[((int64_t)b * K + k) * 2 + 1] = sum; }
  }
}

// backward: p_jk = exp(w_jk - gmax_k)/gsum_k ; df_j = sum_k p_jk dmap_k ; dw_jk = p_jk (<dmap_k, f_j> - <dmap_k, map_k>)
template <typename T, int MG_K>
__global__ void __launch_bounds__(MG_T) mapgen_bwd_kernel(MgArgs a) {
  extern __shared__ float sm[];
  const int K = a.K, C = a.C, b = blockIdx.y, tid = threadIdx.x;
  float* s_dm = sm;                 // [K][C]
  float* s_col = s_dm + K * C;      // [K][3] gmax, 1/gsum, c_k
  for (int o = tid; o < K * C; o += MG_T) s_dm[o] = Elem<T>::ld((const T*)a.dmap + (int64_t)b * K * C + o);
  __syncthreads();
  if (tid < K) {
    float c = 0.f;
    for (int ch = 0; ch < C; ++ch) c = fmaf(s_dm[tid * C + ch], Elem<T>::ld((const T*)a.map + ((int64_t)b * K + tid) * a.map_ld + ch), c);
    s_col[tid * 3] = a.colstat[((int64_t)b * K + tid) * 2]; s_col[tid * 3 + 1] = 1.f / a.colstat[((int64_t)b * K + tid) * 2 + 1];
    s_col[tid * 3 + 2] = c;
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * MG_T + tid;
  if (i >= a.N) return;
  const int64_t row = (int64_t)b * a.N + i;
  const T* wrow = (const T*)a.wl + row * a.w_ld + a.w_coff;
  const T* frow = (const T*)a.f + row * a.f_ld + a.f_coff;
  T* dfrow = (T*)a.df + row * a.df_ld + a.df_coff;
  T* dwrow = (T*)a.dwl + row * a.dw_ld + a.dw_coff;
  float p[MG_K], dA[MG_K];
#pragma unroll
  for (int k = 0; k < MG_K; ++k) { p[k] = (k < K) ? __expf(Elem<T>::ld(wrow + k) - s_col[k * 3]) * s_col[k * 3 + 1] : 0.f; dA[k] = 0.f; }
  for (int c0 = 0; c0 < C; c0 += 8) {
    float f[8], o[8];
    ld8<T>(frow + c0, f);
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] = 0.f;
#pragma unroll
    for (int k = 0; k < MG_K; ++k) {
      if (k < K) {
        const float* dm = s_dm + k * C + c0;
#pragma unroll
        for (int c = 0; c < 8; ++c) { dA[k] = fmaf(dm[c], f[c], dA[k]); o[c] = fmaf(p[k], dm[c], o[c]); }
      }
    }
    st8<T>(dfrow + c0, o);
  }
#pragma unroll
  for (int k = 0; k < MG_K; ++k) if (k < a.dw_pad) Elem<T>::st(dwrow + k, (k < K) ? p[k] * (dA[k] - s_col[k * 3 + 2]) : 0.f);
}

// ------------------------------------------------------------------ SE gate (one block, loops over the batch)
struct SeArgs {
  const double* stats; double n; const float *w1, *b1, *w2, *b2;   // w1 [R][C], w2 [C][R]
  float *gate, *hidden, *mean;                                     // [B][C], [B][R], [B][C]
  const float* dgate; float *dw1, *db1, *dw2, *db2, *dmean;        // backward
  int B, C, R;
};

// forward: every block recomputes the R hidden units (R*C MACs, cheap) and produces its slice of the C gates;
// warps walk weight rows so the loads are coalesced.
__global__ void se_gate_fwd_kernel(SeArgs a) {
  extern __shared__ float sm[];
  float* s_mean = sm; float* s_h = sm + a.C;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int cper = (a.C + gridDim.x - 1) / gridDim.x, c0 = blockIdx.x * cper, c1 = min(a.C, c0 + cper);
  for (int b = 0; b < a.B; ++b) {
    for (int c = threadIdx.x; c < a.C; c += blockDim.x) {
      const float m = (float)(a.stats[((int64_t)b * a.C + c) * 2] / a.n);
      s_mean[c] = m;
      if (blockIdx.x == 0) a.mean[b * a.C + c] = m;
    }
    __syncthreads();
    for (int r = wid; r < a.R; r += nw) {
      float acc = 0.f;
      for (int c = lane; c < a.C; c += 32) acc = fmaf(a.w1[(int64_t)r * a.C + c], s_mean[c], acc);
      acc = warp_sum(acc);
      if (lane == 0) { const float h = fmaxf(acc + a.b1[r], 0.f); s_h[r] = h; if (blockIdx.x == 0) a.hidden[b * a.R + r] = h; }
    }
    __syncthreads();
    for (int c = c0 + wid; c < c1; c += nw) {
      float acc = 0.f;
      for (int r = lane; r < a.R; r += 32) acc = fmaf(a.w2[(int64_t)c * a.R + r], s_h[r], acc);
      acc = warp_sum(acc);
      if (lane == 0) a.gate[b * a.C + c] = 1.f / (1.f + __expf(-(acc + a.b2[c])));
    }
    __syncthreads();
  }
}

// backward: every block recomputes dz2 (C) and dz1 (R, a C x R column reduction) and owns a slice of the C axis
// for dw2/db2/dw1/dmean; block 0 also writes db1.  Each output element is touched by exactly one thread, and every
// partial sum is combined in a fixed order (per-warp / per-part partials in shared memory), so dz1 and dmean -- which
// reach the SE input's gradient and everything upstream -- are the same on every run.
constexpr int SE_RED = 16 * 256;           // [warps][256 r values] of the dz1 reduction; >= blockDim for dmean
__global__ void se_gate_bwd_kernel(SeArgs a) {
  extern __shared__ float sm[];
  float* s_dz2 = sm; float* s_dz1 = sm + a.C; float* s_h = s_dz1 + a.R;     // [C], [R], [R]
  float* s_red = s_h + a.R;                                                 // [SE_RED]
  const int tid = threadIdx.x;
  const int cper = (a.C + gridDim.x - 1) / gridDim.x, c0 = blockIdx.x * cper, c1 = min(a.C, c0 + cper);
  for (int b = 0; b < a.B; ++b) {
    for (int c = tid; c < a.C; c += blockDim.x) {
      const float s = a.gate[b * a.C + c];
      s_dz2[c] = a.dgate[b * a.C + c] * s * (1.f - s);
    }
    for (int r = tid; r < a.R; r += blockDim.x) { s_dz1[r] = 0.f; s_h[r] = a.hidden[b * a.R + r]; }
    __syncthreads();
    // dh[r] = sum_c w2[c][r] dz2[c]: a warp strides the c axis, its lanes hold up to 8 r values each (8 loads in
    // flight per lane, coalesced along r); the per-warp partials are summed in warp order
    {
      const int lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
      for (int rb = 0; rb < a.R; rb += 256) {
        float acc[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] = 0.f;
        for (int c = wid; c < a.C; c += nw) {
          const float z = s_dz2[c];
          const float* wr = a.w2 + (int64_t)c * a.R + rb + lane;
#pragma unroll
          for (int u = 0; u < 8; ++u) if (rb + u * 32 + lane < a.R) acc[u] = fmaf(wr[u * 32], z, acc[u]);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) s_red[wid * 256 + u * 32 + lane] = acc[u];
        __syncthreads();
        for (int r = tid; r < 256 && rb + r < a.R; r += blockDim.x) {
          float s = 0.f;
          for (int w = 0; w < nw; ++w) s += s_red[w * 256 + r];
          s_dz1[rb + r] = s;
        }
        __syncthreads();
      }
    }
    for (int r = tid; r < a.R; r += blockDim.x) {
      const float dz1 = s_h[r] > 0.f ? s_dz1[r] : 0.f;
      s_dz1[r] = dz1;
      if (blockIdx.x == 0) a.db1[r] += dz1;
    }
    __syncthreads();
    // slice-owned outputs
    for (int o = tid; o < (c1 - c0) * a.R; o += blockDim.x) {
      const int c = c0 + o / a.R, r = o % a.R;
      a.dw2[(int64_t)c * a.R + r] += s_dz2[c] * s_h[r];
    }
    for (int o = tid; o < (c1 - c0) * a.R; o += blockDim.x) {      // dw1[r][c], c fastest for coalescing
      const int r = o / (c1 - c0), c = c0 + o % (c1 - c0);
      a.dw1[(int64_t)r * a.C + c] += s_dz1[r] * a.mean[b * a.C + c];
    }
    for (int c = c0 + tid; c < c1; c += blockDim.x) a.db2[c] += s_dz2[c];
    // dmean[c] = sum_r w1[r][c] dz1[r] for the slice: threads (c, r-part), the parts summed in order
    const int ncs = c1 - c0;                   // < blockDim: 132 blocks and the shared-memory cap keep C < 512 * 132
    const int parts = ncs > 0 ? max(1, (int)blockDim.x / ncs) : 0;
    if (ncs > 0) {
      const int part = tid / ncs, cc = tid % ncs;
      if (part < parts) {
        float dm = 0.f;
        for (int r = part; r < a.R; r += parts) dm = fmaf(a.w1[(int64_t)r * a.C + c0 + cc], s_dz1[r], dm);
        s_red[part * ncs + cc] = dm;
      }
    }
    __syncthreads();
    for (int c = tid; c < ncs; c += blockDim.x) {
      float s = 0.f;
      for (int p = 0; p < parts; ++p) s += s_red[p * ncs + c];
      a.dmean[b * a.C + c0 + c] = s;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ channel scale: y = x * g[b][c]
template <typename T>
__global__ void scale_fwd_kernel(const T* x, const float* g, T* y, int64_t V, int C, int64_t total) {
  const int ncg = C >> 3;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(it % ncg); const int64_t vox = it / ncg; const int b = (int)(vox / V);
    float v[8]; ld8<T>(x + vox * C + cg * 8, v);
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] *= g[b * C + cg * 8 + c];
    st8<T>(y + vox * C + cg * 8, v);
  }
}
// dg[b][c] = sum_vox dy * x in two passes that add in a fixed order (DESIGN §4a): grid (gx, B) blocks each write
// the sum of their threads' partials to part[b][block][C]; the second pass adds the gx partials in block order.
template <typename T>
__global__ void scale_bwd_reduce_kernel(const T* dy, const T* x, float* part, int64_t V, int C) {
  extern __shared__ float s_part[];          // [threads][8]: thread tid = rl * ncg + cg at [rl * C + cg * 8]
  const int b = blockIdx.y, ncg = C >> 3, cg = threadIdx.x % ncg;
  float acc[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) acc[c] = 0.f;
  const int64_t items = V * ncg;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (int64_t)gridDim.x * blockDim.x) {
    const int64_t vox = (int64_t)b * V + it / ncg;
    float g[8], v[8]; ld8<T>(dy + vox * C + cg * 8, g); ld8<T>(x + vox * C + cg * 8, v);
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = fmaf(g[c], v[c], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < 8; ++c) s_part[threadIdx.x * 8 + c] = acc[c];
  __syncthreads();
  const int rb = blockDim.x / ncg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int r = 0; r < rb; ++r) s += s_part[r * C + c];
    part[((int64_t)b * gridDim.x + blockIdx.x) * C + c] = s;
  }
}
__global__ void scale_bwd_sum_kernel(const float* part, float* dg, int nblk, int C) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float* p = part + (int64_t)b * nblk * C + c;
  float s = 0.f;
  for (int k = 0; k < nblk; ++k) s += p[(int64_t)k * C];
  dg[b * C + c] += s;
}
// dx = dy * g[b][c] + dmean[b][c] / V
template <typename T>
__global__ void scale_bwd_apply_kernel(const T* dy, const float* g, const float* dmean, T* dx, int64_t V, int C, int64_t total) {
  const int ncg = C >> 3; const float invV = 1.f / (float)V;
  for (int64_t it = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; it < total; it += (int64_t)gridDim.x * blockDim.x) {
    const int cg = (int)(it % ncg); const int64_t vox = it / ncg; const int b = (int)(vox / V);
    float v[8]; ld8<T>(dy + vox * C + cg * 8, v);
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = fmaf(v[c], g[b * C + cg * 8 + c], dmean ? dmean[b * C + cg * 8 + c] * invV : 0.f);
    st8<T>(dx + vox * C + cg * 8, v);
  }
}

// ------------------------------------------------------------------ LayerNorm over the last dim, one warp per row
template <typename T>
__global__ void layernorm_fwd_kernel(const T* x, const float* gamma, const float* beta, T* y, float* mr, int R, int C, float eps) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= R) return;
  const T* xr = x + (int64_t)row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += Elem<T>::ld(xr + c);
  const float mean = warp_sum(s) / C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = Elem<T>::ld(xr + c) - mean; q = fmaf(d, d, q); }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  for (int c = lane; c < C; c += 32) Elem<T>::st(y + (int64_t)row * C + c, (Elem<T>::ld(xr + c) - mean) * rstd * gamma[c] + beta[c]);
  if (lane == 0) { mr[row * 2] = mean; mr[row * 2 + 1] = rstd; }
}
// Persistent blocks (4 warps, one row per warp per step); d(gamma) / d(beta) are accumulated in shared memory and
// flushed with ONE global atomic per (block, channel) — the Swin token streams have 10^5..10^6 rows per LayerNorm.
template <typename T>
__global__ void layernorm_bwd_kernel(const T* dy, const T* x, const float* gamma, const float* mr, T* dx, float* dgamma, float* dbeta, int R, int C) {
  extern __shared__ float s_gb[];               // [2][C]
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) s_gb[c] = 0.f;
  __syncthreads();
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (int row = blockIdx.x * wpb + (threadIdx.x >> 5); row < R; row += gridDim.x * wpb) {
    const float mean = mr[row * 2], rstd = mr[row * 2 + 1];
    const T* xr = x + (int64_t)row * C; const T* gr = dy + (int64_t)row * C;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (Elem<T>::ld(xr + c) - mean) * rstd, g = Elem<T>::ld(gr + c);
      const float gg = g * gamma[c];
      s1 += gg; s2 = fmaf(gg, xh, s2);
      atomicAdd(&s_gb[c], g * xh); atomicAdd(&s_gb[C + c], g);
    }
    s1 = warp_sum(s1) / C; s2 = warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) {
      const float xh = (Elem<T>::ld(xr + c) - mean) * rstd, gg = Elem<T>::ld(gr + c) * gamma[c];
      Elem<T>::st(dx + (int64_t)row * C + c, rstd * (gg - s1 - xh * s2));
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    if (s_gb[c] != 0.f) atomicAdd(&dgamma[c], s_gb[c]);
    if (s_gb[C + c] != 0.f) atomicAdd(&dbeta[c], s_gb[C + c]);
  }
}

// ------------------------------------------------------------------ GELU (exact, erf)
template <typename T>
__global__ void gelu_kernel(const T* x, const T* dy, T* out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = Elem<T>::ld(x + i);
    const float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752f));
    if (!dy) Elem<T>::st(out + i, v * cdf);
    else Elem<T>::st(out + i, Elem<T>::ld(dy + i) * (cdf + v * 0.3989422804014327f * __expf(-0.5f * v * v)));
  }
}

// ------------------------------------------------------------------ MHSA over L <= 192 tokens, dim_head 32
// qkv [B][L][3*inner], channel = which*inner + h*32 + d ('b l (heads dim_head)', trans_layers.py:58-66);
// out [B][L][inner] with channel h*32 + d (rearrange2 really yields (heads dim_head), SURVEY.md a14).
constexpr int MH_D = 32, MH_RT = 64;       // head dim; query rows per score tile
// One block per (head, batch).  q/k/v (and dO) of the head live in shared memory; the L x L scores are walked in
// tiles of MH_RT query rows so L = 192 (three 4x4x4 maps) fits; dK/dV accumulate in shared fp32 across the tiles.
template <typename T>
__global__ void mhsa_kernel(const T* qkv, const T* dout, T* out, T* dqkv, int L, int heads, float scale) {
  extern __shared__ float sm[];
  const int inner = heads * MH_D, h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int P33 = MH_D + 1;
  float* s_q = sm; float* s_k = s_q + L * P33; float* s_v = s_k + L * P33;
  float* s_p = s_v + L * P33;                        // [MH_RT][L+1]
  float* s_do = s_p + MH_RT * (L + 1);               // backward only: [L][33], then dK and dV accumulators
  float* s_dk = s_do + L * P33; float* s_dv = s_dk + L * P33;
  const bool bwd = dout != nullptr;
  const T* base = qkv + (int64_t)b * L * 3 * inner + h * MH_D;
  for (int o = tid; o < L * MH_D; o += blockDim.x) {
    const int l = o / MH_D, d = o % MH_D;
    s_q[l * P33 + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + d);
    s_k[l * P33 + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + inner + d);
    s_v[l * P33 + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + 2 * inner + d);
    if (bwd) {
      s_do[l * P33 + d] = Elem<T>::ld(dout + ((int64_t)b * L + l) * inner + h * MH_D + d);
      s_dk[l * P33 + d] = 0.f; s_dv[l * P33 + d] = 0.f;
    }
  }
  __syncthreads();
  T* dbase = bwd ? dqkv + (int64_t)b * L * 3 * inner + h * MH_D : nullptr;
  for (int r0 = 0; r0 < L; r0 += MH_RT) {
    const int rows = min(MH_RT, L - r0);
    for (int o = tid; o < rows * L; o += blockDim.x) {
      const int i = o / L, j = o % L;
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < MH_D; ++d) acc = fmaf(s_q[(r0 + i) * P33 + d], s_k[j * P33 + d], acc);
      s_p[i * (L + 1) + j] = acc * scale;
    }
    __syncthreads();
    for (int i = tid; i < rows; i += blockDim.x) {
      float m = -INFINITY;
      for (int j = 0; j < L; ++j) m = fmaxf(m, s_p[i * (L + 1) + j]);
      float sum = 0.f;
      for (int j = 0; j < L; ++j) { const float e = __expf(s_p[i * (L + 1) + j] - m); s_p[i * (L + 1) + j] = e; sum += e; }
      const float inv = 1.f / sum;
      for (int j = 0; j < L; ++j) s_p[i * (L + 1) + j] *= inv;
    }
    __syncthreads();
    if (!bwd) {
      for (int o = tid; o < rows * MH_D; o += blockDim.x) {
        const int i = o / MH_D, d = o % MH_D;
        float acc = 0.f;
        for (int j = 0; j < L; ++j) acc = fmaf(s_p[i * (L + 1) + j], s_v[j * P33 + d], acc);
        Elem<T>::st(out + ((int64_t)b * L + r0 + i) * inner + h * MH_D + d, acc);
      }
      __syncthreads();
      continue;
    }
    // dV += P^T dO over this tile's rows
    for (int o = tid; o < L * MH_D; o += blockDim.x) {
      const int j = o / MH_D, d = o % MH_D;
      float acc = 0.f;
      for (int i = 0; i < rows; ++i) acc = fmaf(s_p[i * (L + 1) + j], s_do[(r0 + i) * P33 + d], acc);
      s_dv[j * P33 + d] += acc;
    }
    __syncthreads();
    // dS = P o (dP - rowsum(dP o P)) * scale, dP = dO V^T   (written over P row by row)
    for (int i = tid; i < rows; i += blockDim.x) {
      float t = 0.f;
      for (int j = 0; j < L; ++j) {
        float dp = 0.f;
#pragma unroll
        for (int d = 0; d < MH_D; ++d) dp = fmaf(s_do[(r0 + i) * P33 + d], s_v[j * P33 + d], dp);
        t = fmaf(dp, s_p[i * (L + 1) + j], t);
      }
      for (int j = 0; j < L; ++j) {
        float dp = 0.f;
#pragma unroll
        for (int d = 0; d < MH_D; ++d) dp = fmaf(s_do[(r0 + i) * P33 + d], s_v[j * P33 + d], dp);
        s_p[i * (L + 1) + j] *= (dp - t) * scale;
      }
    }
    __syncthreads();
    for (int o = tid; o < rows * MH_D; o += blockDim.x) {          // dQ rows of this tile
      const int i = o / MH_D, d = o % MH_D;
      float aq = 0.f;
      for (int j = 0; j < L; ++j) aq = fmaf(s_p[i * (L + 1) + j], s_k[j * P33 + d], aq);
      Elem<T>::st(dbase + (int64_t)(r0 + i) * 3 * inner + d, aq);
    }
    for (int o = tid; o < L * MH_D; o += blockDim.x) {             // dK += dS^T Q over this tile's rows
      const int j = o / MH_D, d = o % MH_D;
      float ak = 0.f;
      for (int i = 0; i < rows; ++i) ak = fmaf(s_p[i * (L + 1) + j], s_q[(r0 + i) * P33 + d], ak);
      s_dk[j * P33 + d] += ak;
    }
    __syncthreads();
  }
  if (bwd) {
    for (int o = tid; o < L * MH_D; o += blockDim.x) {
      const int j = o / MH_D, d = o % MH_D;
      Elem<T>::st(dbase + (int64_t)j * 3 * inner + inner + d, s_dk[j * P33 + d]);
      Elem<T>::st(dbase + (int64_t)j * 3 * inner + 2 * inner + d, s_dv[j * P33 + d]);
    }
  }
}

// ------------------------------------------------------------------ MHSA over L <= 216 tokens, dim_head 64
// The map fusion of the ACDC configuration: 3 x 72 tokens, 4 heads of 64.  The tiled scheme above would need K, V,
// the probability tile, dO and the dK/dV accumulators (~335 KB) at this size, so here one block per (head, batch)
// stages Q, K, V (and dO) at a 65-float row stride and runs one warp per row: no L x L tile is stored.
//   forward / dQ pass   warp per query row i: scores over the keys in registers (lane owns keys lane + 32t),
//                       softmax by shuffles, out_i / dQ_i with the lane owning channels lane and lane + 32; the
//                       backward keeps {row max, 1 / row sum, D_i = sum_j P_ij dP_ij} per row in shared memory;
//   dK / dV pass        warp per key row j: P_ij and dS_ij over the queries recomputed from those row statistics.
constexpr int MH64_D = 64, MH64_LD = MH64_D + 1, MH64_LMAX = 216, MH64_JT = (MH64_LMAX + 31) / 32, MH64_T = 512;

template <typename T>
__global__ void __launch_bounds__(MH64_T) mhsa64_kernel(const T* qkv, const T* dout, T* out, T* dqkv, int L, int heads, float scale) {
  extern __shared__ float sm[];
  const int inner = heads * MH64_D, h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int lane = tid & 31, wid = tid >> 5, nw = MH64_T / 32;
  float* s_q = sm; float* s_k = s_q + L * MH64_LD; float* s_v = s_k + L * MH64_LD;
  float* s_do = s_v + L * MH64_LD;                   // backward only: [L][65], then [L][3] row statistics
  float* s_st = s_do + L * MH64_LD;
  const bool bwd = dout != nullptr;
  const T* base = qkv + (int64_t)b * L * 3 * inner + h * MH64_D;
  for (int o = tid; o < L * MH64_D; o += MH64_T) {
    const int l = o / MH64_D, d = o % MH64_D;
    s_q[l * MH64_LD + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + d);
    s_k[l * MH64_LD + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + inner + d);
    s_v[l * MH64_LD + d] = Elem<T>::ld(base + (int64_t)l * 3 * inner + 2 * inner + d);
    if (bwd) s_do[l * MH64_LD + d] = Elem<T>::ld(dout + ((int64_t)b * L + l) * inner + h * MH64_D + d);
  }
  __syncthreads();
  T* dbase = bwd ? dqkv + (int64_t)b * L * 3 * inner + h * MH64_D : nullptr;
  for (int i = wid; i < L; i += nw) {
    const float* qi = s_q + i * MH64_LD;
    float p[MH64_JT], m = -INFINITY;
#pragma unroll
    for (int t = 0; t < MH64_JT; ++t) {
      const int j = lane + 32 * t;
      float acc = -INFINITY;
      if (j < L) {
        acc = 0.f;
        const float* kj = s_k + j * MH64_LD;
#pragma unroll 16
        for (int d = 0; d < MH64_D; ++d) acc = fmaf(qi[d], kj[d], acc);
        acc *= scale;
      }
      p[t] = acc; m = fmaxf(m, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < MH64_JT; ++t) { p[t] = __expf(p[t] - m); sum += p[t]; }
    const float inv = 1.f / warp_sum(sum);
#pragma unroll
    for (int t = 0; t < MH64_JT; ++t) p[t] *= inv;
    if (!bwd) {
      float o0 = 0.f, o1 = 0.f;
#pragma unroll
      for (int t = 0; t < MH64_JT; ++t)
        for (int src = 0; src < 32; ++src) {
          const int j = 32 * t + src;
          const float pj = __shfl_sync(0xffffffffu, p[t], src);
          if (j < L) { o0 = fmaf(pj, s_v[j * MH64_LD + lane], o0); o1 = fmaf(pj, s_v[j * MH64_LD + lane + 32], o1); }
        }
      T* op = out + ((int64_t)b * L + i) * inner + h * MH64_D;
      Elem<T>::st(op + lane, o0); Elem<T>::st(op + lane + 32, o1);
      continue;
    }
    // dP_ij = <dO_i, V_j>; D_i = sum_j P_ij dP_ij; dS_ij = P_ij (dP_ij - D_i) * scale; dQ_i = sum_j dS_ij K_j
    const float* gi = s_do + i * MH64_LD;
    float dp[MH64_JT], dsum = 0.f;
#pragma unroll
    for (int t = 0; t < MH64_JT; ++t) {
      const int j = lane + 32 * t;
      float acc = 0.f;
      if (j < L) {
        const float* vj = s_v + j * MH64_LD;
#pragma unroll 16
        for (int d = 0; d < MH64_D; ++d) acc = fmaf(gi[d], vj[d], acc);
      }
      dp[t] = acc; dsum = fmaf(p[t], acc, dsum);
    }
    const float Di = warp_sum(dsum);
    float q0 = 0.f, q1 = 0.f;
#pragma unroll
    for (int t = 0; t < MH64_JT; ++t) {
      const float ds = p[t] * (dp[t] - Di) * scale;
      for (int src = 0; src < 32; ++src) {
        const int j = 32 * t + src;
        const float dsj = __shfl_sync(0xffffffffu, ds, src);
        if (j < L) { q0 = fmaf(dsj, s_k[j * MH64_LD + lane], q0); q1 = fmaf(dsj, s_k[j * MH64_LD + lane + 32], q1); }
      }
    }
    T* dq = dbase + (int64_t)i * 3 * inner;
    Elem<T>::st(dq + lane, q0); Elem<T>::st(dq + lane + 32, q1);
    if (lane == 0) { s_st[3 * i] = m; s_st[3 * i + 1] = inv; s_st[3 * i + 2] = Di; }
  }
  if (!bwd) return;
  __syncthreads();
  // dV_j = sum_i P_ij dO_i ; dK_j = sum_i dS_ij Q_i
  for (int j = wid; j < L; j += nw) {
    const float* kj = s_k + j * MH64_LD;
    const float* vj = s_v + j * MH64_LD;
    float k0 = 0.f, k1 = 0.f, v0 = 0.f, v1 = 0.f;
#pragma unroll 1
    for (int i0 = 0; i0 < L; i0 += 32) {
      const int i = i0 + lane;
      float pij = 0.f, ds = 0.f;
      if (i < L) {
        float s = 0.f, dp = 0.f;
        const float* qi = s_q + i * MH64_LD;
        const float* gi = s_do + i * MH64_LD;
#pragma unroll 16
        for (int d = 0; d < MH64_D; ++d) { s = fmaf(qi[d], kj[d], s); dp = fmaf(gi[d], vj[d], dp); }
        pij = __expf(s * scale - s_st[3 * i]) * s_st[3 * i + 1];
        ds = pij * (dp - s_st[3 * i + 2]) * scale;
      }
      for (int src = 0; src < 32; ++src) {
        const float ps = __shfl_sync(0xffffffffu, pij, src), dss = __shfl_sync(0xffffffffu, ds, src);
        const int r = i0 + src;
        if (r < L) {
          v0 = fmaf(ps, s_do[r * MH64_LD + lane], v0); v1 = fmaf(ps, s_do[r * MH64_LD + lane + 32], v1);
          k0 = fmaf(dss, s_q[r * MH64_LD + lane], k0); k1 = fmaf(dss, s_q[r * MH64_LD + lane + 32], k1);
        }
      }
    }
    T* dk = dbase + (int64_t)j * 3 * inner + inner;
    Elem<T>::st(dk + lane, k0); Elem<T>::st(dk + lane + 32, k1);
    Elem<T>::st(dk + inner + lane, v0); Elem<T>::st(dk + inner + lane + 32, v1);
  }
}

inline int grid_for(int64_t items, int threads) {
  int64_t g = (items + threads - 1) / threads;
  const int64_t cap = B200SEG_NUM_SMS * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
inline bool ok_dtype(int d) { return d == B200SEG_F16 || d == B200SEG_F32; }

}  // namespace

#define DISPATCH_T(dtype, ...)                                   \
  do { if ((dtype) == B200SEG_F16) { using T = __half; __VA_ARGS__; } else { using T = float; __VA_ARGS__; } } while (0)

extern "C" int b200seg_space_to_depth(void* x, void* y, int B, int Do, int Ho, int Wo, int C, int sd, int sh, int sw,
                                      int reverse, int dtype, void* stream) {
  if (!x || !y || B <= 0 || Do <= 0 || Ho <= 0 || Wo <= 0 || sd <= 0 || sh <= 0 || sw <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  const bool vec = (C % 8) == 0;
  const int64_t total = (int64_t)B * Do * Ho * Wo * sd * sh * sw * (vec ? C / 8 : C);
  if (vec) { DISPATCH_T(dtype, s2d_kernel<T, 8><<<grid_for(total, 256), 256, 0, as_stream(stream)>>>((const T*)x, (T*)y, B, Do, Ho, Wo, C, sd, sh, sw, reverse)); }
  else { DISPATCH_T(dtype, s2d_kernel<T, 1><<<grid_for(total, 256), 256, 0, as_stream(stream)>>>((const T*)x, (T*)y, B, Do, Ho, Wo, C, sd, sh, sw, reverse)); }
  B200_CHECK_LAUNCH("space_to_depth");
  return B200SEG_OK;
}

extern "C" size_t b200seg_mapgen_workspace(int B, int64_t N, int K, int C) {
  return (size_t)B * ((N + MG_T - 1) / MG_T) * K * (2 + C) * sizeof(float);
}

extern "C" int b200seg_mapgen_fwd(const void* f, int f_ld, int f_coff, const void* wl, int w_ld, int w_coff,
                                  void* map, float* colstat, float* workspace, int B, int64_t N, int K, int C,
                                  int dtype, void* stream) {
  if (!f || !wl || !map || !colstat || !workspace || B <= 0 || N <= 0 || K <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (K > MG_KCAP) return B200SEG_EUNSUPPORTED;
  MgArgs a; memset(&a, 0, sizeof(a));
  a.f = f; a.f_ld = f_ld; a.f_coff = f_coff; a.wl = wl; a.w_ld = w_ld; a.w_coff = w_coff; a.map = map; a.map_ld = C;
  a.colstat = colstat; a.partial = workspace; a.B = B; a.N = N; a.K = K; a.C = C;
  const int nblk = (int)((N + MG_T - 1) / MG_T);
  cudaStream_t st = as_stream(stream);
  const int KC = K <= 32 ? 32 : (K <= 64 ? 64 : 80);
  const size_t fsm = sizeof(float) * ((size_t)MG_T * (KC + 1) + MG_T * (MG_CC + 1) + 5 * KC);
#define B200_MAPGEN_FWD(TT, KK)                                                                                \
  do {                                                                                                         \
    B200_CUDA(cudaFuncSetAttribute(mapgen_fwd_kernel<TT, KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsm)); \
    mapgen_fwd_kernel<TT, KK><<<dim3(nblk, B), MG_T, fsm, st>>>(a);                                            \
    mapgen_merge_kernel<TT><<<dim3(K, B), 128, 0, st>>>(a, nblk);                                              \
  } while (0)
  if (dtype == B200SEG_F16) { if (KC == 32) B200_MAPGEN_FWD(__half, 32); else if (KC == 64) B200_MAPGEN_FWD(__half, 64); else B200_MAPGEN_FWD(__half, 80); }
  else { if (KC == 32) B200_MAPGEN_FWD(float, 32); else if (KC == 64) B200_MAPGEN_FWD(float, 64); else B200_MAPGEN_FWD(float, 80); }
#undef B200_MAPGEN_FWD
  B200_CHECK_LAUNCH("mapgen_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_mapgen_bwd(const void* f, int f_ld, int f_coff, const void* wl, int w_ld, int w_coff,
                                  const void* map, const float* colstat, const void* dmap,
                                  void* df, int df_ld, int df_coff, void* dwl, int dw_ld, int dw_coff, int dw_pad,
                                  int B, int64_t N, int K, int C, int dtype, void* stream) {
  if (!f || !wl || !map || !colstat || !dmap || !df || !dwl || B <= 0 || N <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (K > MG_KCAP || dw_pad > MG_KCAP || dw_pad < K || C % 8 || f_ld % 8 || f_coff % 8 || df_ld % 8 || df_coff % 8) return B200SEG_EUNSUPPORTED;
  const size_t smem = sizeof(float) * ((size_t)K * C + 3 * K);
  if (smem > 200 * 1024) return B200SEG_EUNSUPPORTED;
  MgArgs a; memset(&a, 0, sizeof(a));
  a.f = f; a.f_ld = f_ld; a.f_coff = f_coff; a.wl = wl; a.w_ld = w_ld; a.w_coff = w_coff;
  a.map = const_cast<void*>(map); a.map_ld = C; a.colstat = const_cast<float*>(colstat); a.dmap = dmap;
  a.df = df; a.df_ld = df_ld; a.df_coff = df_coff; a.dwl = dwl; a.dw_ld = dw_ld; a.dw_coff = dw_coff; a.dw_pad = dw_pad;
  a.B = B; a.N = N; a.K = K; a.C = C;
  const int nblk = (int)((N + MG_T - 1) / MG_T);
  cudaStream_t st = as_stream(stream);
  const int KC = dw_pad <= 32 ? 32 : (dw_pad <= 64 ? 64 : 80);
#define B200_MAPGEN_BWD(TT, KK)                                                                                \
  do {                                                                                                         \
    B200_CUDA(cudaFuncSetAttribute(mapgen_bwd_kernel<TT, KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    mapgen_bwd_kernel<TT, KK><<<dim3(nblk, B), MG_T, smem, st>>>(a);                                           \
  } while (0)
  if (dtype == B200SEG_F16) { if (KC == 32) B200_MAPGEN_BWD(__half, 32); else if (KC == 64) B200_MAPGEN_BWD(__half, 64); else B200_MAPGEN_BWD(__half, 80); }
  else { if (KC == 32) B200_MAPGEN_BWD(float, 32); else if (KC == 64) B200_MAPGEN_BWD(float, 64); else B200_MAPGEN_BWD(float, 80); }
#undef B200_MAPGEN_BWD
  B200_CHECK_LAUNCH("mapgen_bwd");
  return B200SEG_OK;
}

extern "C" int b200seg_se_gate_fwd(const double* stats, int64_t nvox, const float* w1, const float* b1, const float* w2,
                                   const float* b2, float* gate, float* hidden, float* mean, int B, int C, int R, void* stream) {
  if (!stats || !w1 || !b1 || !w2 || !b2 || !gate || !hidden || !mean || B <= 0 || C <= 0 || R <= 0 || nvox <= 0) return B200SEG_EINVAL;
  SeArgs a; memset(&a, 0, sizeof(a));
  a.stats = stats; a.n = (double)nvox; a.w1 = w1; a.b1 = b1; a.w2 = w2; a.b2 = b2; a.gate = gate; a.hidden = hidden; a.mean = mean;
  a.B = B; a.C = C; a.R = R;
  se_gate_fwd_kernel<<<(C + 63) / 64 < B200SEG_NUM_SMS ? (C + 63) / 64 : B200SEG_NUM_SMS, 512, sizeof(float) * (C + R), as_stream(stream)>>>(a);
  B200_CHECK_LAUNCH("se_gate_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_se_gate_bwd(const float* dgate, const float* gate, const float* hidden, const float* mean,
                                   const float* w1, const float* w2, float* dw1, float* db1, float* dw2, float* db2,
                                   float* dmean, int B, int C, int R, void* stream) {
  if (!dgate || !gate || !hidden || !mean || !w1 || !w2 || !dw1 || !db1 || !dw2 || !db2 || !dmean || B <= 0 || C <= 0 || R <= 0) return B200SEG_EINVAL;
  SeArgs a; memset(&a, 0, sizeof(a));
  a.dgate = dgate; a.gate = const_cast<float*>(gate); a.hidden = const_cast<float*>(hidden); a.mean = const_cast<float*>(mean);
  a.w1 = w1; a.w2 = w2; a.dw1 = dw1; a.db1 = db1; a.dw2 = dw2; a.db2 = db2; a.dmean = dmean; a.B = B; a.C = C; a.R = R;
  const size_t smem = sizeof(float) * ((size_t)C + 2 * (size_t)R + SE_RED);
  if (smem > 200 * 1024) return B200SEG_EUNSUPPORTED;
  B200_CUDA(cudaFuncSetAttribute(se_gate_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  se_gate_bwd_kernel<<<(C + 31) / 32 < B200SEG_NUM_SMS ? (C + 31) / 32 : B200SEG_NUM_SMS, 512, smem, as_stream(stream)>>>(a);
  B200_CHECK_LAUNCH("se_gate_bwd");
  return B200SEG_OK;
}

extern "C" int b200seg_channel_scale_fwd(const void* x, const float* gate, void* y, int B, int64_t V, int C, int dtype, void* stream) {
  if (!x || !gate || !y || B <= 0 || V <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (C % 8) return B200SEG_EUNSUPPORTED;
  const int64_t total = (int64_t)B * V * (C / 8);
  DISPATCH_T(dtype, scale_fwd_kernel<T><<<grid_for(total, 256), 256, 0, as_stream(stream)>>>((const T*)x, gate, (T*)y, V, C, total));
  B200_CHECK_LAUNCH("channel_scale_fwd");
  return B200SEG_OK;
}

// thread shape and block count of the first reduction pass; the workspace holds one [C] partial per (b, block)
static int scale_bwd_shape(int64_t V, int C, int* threads) {
  const int ncg = C / 8;
  *threads = ncg >= 256 ? ncg : (256 / ncg) * ncg;
  const int gx = grid_for(V * ncg, *threads);
  return gx > 592 ? 592 : gx;
}

extern "C" size_t b200seg_channel_scale_bwd_workspace(int B, int64_t V, int C) {
  if (B <= 0 || V <= 0 || C <= 0 || C % 8) return 0;
  int threads;
  return (size_t)B * scale_bwd_shape(V, C, &threads) * C * sizeof(float);
}

extern "C" int b200seg_channel_scale_bwd_reduce(const void* dy, const void* x, float* dgate, float* workspace, int B,
                                                int64_t V, int C, int dtype, void* stream) {
  if (!dy || !x || !dgate || !workspace || B <= 0 || V <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (C % 8 || C > 8192) return B200SEG_EUNSUPPORTED;
  int threads;
  const int gx = scale_bwd_shape(V, C, &threads);
  if (threads > 1024) return B200SEG_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  DISPATCH_T(dtype, scale_bwd_reduce_kernel<T><<<dim3(gx, B), threads, sizeof(float) * 8 * threads, st>>>((const T*)dy, (const T*)x, workspace, V, C));
  scale_bwd_sum_kernel<<<dim3((C + 255) / 256, B), 256, 0, st>>>(workspace, dgate, gx, C);
  B200_CHECK_LAUNCH("channel_scale_bwd_reduce");
  return B200SEG_OK;
}

extern "C" int b200seg_channel_scale_bwd_apply(const void* dy, const float* gate, const float* dmean, void* dx, int B, int64_t V, int C, int dtype, void* stream) {
  if (!dy || !gate || !dx || B <= 0 || V <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (C % 8) return B200SEG_EUNSUPPORTED;
  const int64_t total = (int64_t)B * V * (C / 8);
  DISPATCH_T(dtype, scale_bwd_apply_kernel<T><<<grid_for(total, 256), 256, 0, as_stream(stream)>>>((const T*)dy, gate, dmean, (T*)dx, V, C, total));
  B200_CHECK_LAUNCH("channel_scale_bwd_apply");
  return B200SEG_OK;
}

extern "C" int b200seg_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean_rstd,
                                     int R, int C, float eps, int dtype, void* stream) {
  if (!x || !gamma || !beta || !y || !mean_rstd || R <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  DISPATCH_T(dtype, layernorm_fwd_kernel<T><<<(R + 3) / 4, 128, 0, as_stream(stream)>>>((const T*)x, gamma, beta, (T*)y, mean_rstd, R, C, eps));
  B200_CHECK_LAUNCH("layernorm_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_layernorm_bwd(const void* dy, const void* x, const float* gamma, const float* mean_rstd, void* dx,
                                     float* dgamma, float* dbeta, int R, int C, int dtype, void* stream) {
  if (!dy || !x || !gamma || !mean_rstd || !dx || !dgamma || !dbeta || R <= 0 || C <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if (C > 6000) return B200SEG_EUNSUPPORTED;
  int grid = (R + 3) / 4; if (grid > B200SEG_NUM_SMS * 8) grid = B200SEG_NUM_SMS * 8;
  const size_t sm = sizeof(float) * 2 * (size_t)C;
  DISPATCH_T(dtype, layernorm_bwd_kernel<T><<<grid, 128, sm, as_stream(stream)>>>((const T*)dy, (const T*)x, gamma, mean_rstd, (T*)dx, dgamma, dbeta, R, C));
  B200_CHECK_LAUNCH("layernorm_bwd");
  return B200SEG_OK;
}

extern "C" int b200seg_gelu(const void* x, const void* dy, void* out, int64_t n, int dtype, void* stream) {
  if (!x || !out || n <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  DISPATCH_T(dtype, gelu_kernel<T><<<grid_for(n, 256), 256, 0, as_stream(stream)>>>((const T*)x, (const T*)dy, (T*)out, n));
  B200_CHECK_LAUNCH("gelu");
  return B200SEG_OK;
}

extern "C" int b200seg_mhsa(const void* qkv, const void* dout, void* out, void* dqkv, int B, int L, int heads, int dim_head,
                            float scale, int dtype, void* stream) {
  if (!qkv || B <= 0 || L <= 0 || heads <= 0 || !ok_dtype(dtype)) return B200SEG_EINVAL;
  if ((dout == nullptr) == (out == nullptr) || (dout && !dqkv)) return B200SEG_EINVAL;
  if (dim_head == MH64_D) {
    if (L > MH64_LMAX || heads > 65535 || B > 65535) return B200SEG_EUNSUPPORTED;
    const size_t smem = sizeof(float) * ((size_t)(dout ? 4 : 3) * L * MH64_LD + (dout ? 3 * (size_t)L : 0));
    if (dtype == B200SEG_F16) {
      B200_CUDA(cudaFuncSetAttribute(mhsa64_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      mhsa64_kernel<__half><<<dim3(heads, B), MH64_T, smem, as_stream(stream)>>>((const __half*)qkv, (const __half*)dout, (__half*)out, (__half*)dqkv, L, heads, scale);
    } else {
      B200_CUDA(cudaFuncSetAttribute(mhsa64_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      mhsa64_kernel<float><<<dim3(heads, B), MH64_T, smem, as_stream(stream)>>>((const float*)qkv, (const float*)dout, (float*)out, (float*)dqkv, L, heads, scale);
    }
    B200_CHECK_LAUNCH("mhsa");
    return B200SEG_OK;
  }
  if (dim_head != MH_D || L > 192) return B200SEG_EUNSUPPORTED;
  const size_t smem = sizeof(float) * ((size_t)(dout ? 6 : 3) * L * (MH_D + 1) + (size_t)MH_RT * (L + 1));
  if (dtype == B200SEG_F16) {
    B200_CUDA(cudaFuncSetAttribute(mhsa_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mhsa_kernel<__half><<<dim3(heads, B), 256, smem, as_stream(stream)>>>((const __half*)qkv, (const __half*)dout, (__half*)out, (__half*)dqkv, L, heads, scale);
  } else {
    B200_CUDA(cudaFuncSetAttribute(mhsa_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mhsa_kernel<float><<<dim3(heads, B), 256, smem, as_stream(stream)>>>((const float*)qkv, (const float*)dout, (float*)out, (float*)dqkv, L, heads, scale);
  }
  B200_CHECK_LAUNCH("mhsa");
  return B200SEG_OK;
}
