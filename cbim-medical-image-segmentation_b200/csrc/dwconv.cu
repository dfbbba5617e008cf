// dwconv.cu — depthwise 3-D convolution (groups == channels), forward / data-gradient / weight-gradient.
// Reference: DepthwiseSeparableConv.depthwise, model/dim3/conv_layers.py:135-143 (stride 1, "same" padding,
// bias=False), used by MedFormer's attention projections (medformer_utils.py:30-31) and MBConv
// (conv_layers.py MBConv.conv2).  One FMA per loaded byte pair -> HBM/L2 bound; no tensor-core shape here
// (the contraction is over the 27 taps only), so this is the coalesced 128-bit direct path of the north star.
// Layout: channels-last [B][D][H][W][ld]; a thread owns 8 consecutive channels (one 16 B vector for fp16) and a
// run of 4 voxels along W, sliding the 3-wide window so each input vector is loaded once per (kd,kh) row.
// Optional fused prologue: a = act(IN(x)) from the producer's {sum,sumsq}; optional epilogue: IN sums of y.
#include "common.cuh"

namespace {

constexpr int RUN = 4;       // output voxels per thread along W
constexpr int MAXK = 3;      // kernel extent per axis (1 or 3 in every reference config)

struct DwArgs {
  const void* x; int x_ld, x_coff; const double* x_stats; float eps; int act;
  const float* w; int flip;
  int wlay;                  // 0: weights / weight gradient as [taps][Ctot]; 1: [Ctot][taps] (the module's own [C,1,kd,kh,kw] parameter)
  void* y; int y_ld, y_coff; double* y_stats;
  const void* dy; int dy_ld, dy_coff; float* dw;
  int B, D, H, W, C, kd, kh, kw;
  int Ctot, c0;              // the launch covers channels [c0, c0+C) of a Ctot-channel layer (stats / weight rows)
};

// spatial tile covered by one pass of a block (rb = threads / channel-groups positions)
struct Tile { int td, th, tw, nd, nh, nw; int64_t ntiles; };
__host__ __device__ inline Tile make_tile(int rb, int D, int H, int Wn) {
  Tile t;
  if (rb % 8 == 0 && D > 1) { t.td = 2; t.th = 4; t.tw = rb / 8; }
  else if (rb % 4 == 0) { t.td = 1; t.th = 4; t.tw = rb / 4; }
  else { t.td = 1; t.th = 1; t.tw = rb; }
  t.nd = (D + t.td - 1) / t.td; t.nh = (H + t.th - 1) / t.th; t.nw = (Wn + t.tw - 1) / t.tw;
  t.ntiles = (int64_t)t.nd * t.nh * t.nw;
  return t;
}

// 8 channels as loaded (no conversion yet) + validity, so a whole row of loads can be issued back to back
template <typename T> struct Raw;
template <> struct Raw<__half> {
  uint4 u; bool ok;
  __device__ __forceinline__ void load(const __half* p, bool valid) { ok = valid; if (valid) u = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void get(float (&v)[8]) const {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
  }
};
template <> struct Raw<float> {
  float4 a, b; bool ok;
  __device__ __forceinline__ void load(const float* p, bool valid) {
    ok = valid;
    if (valid) { a = *reinterpret_cast<const float4*>(p); b = *reinterpret_cast<const float4*>(p + 4); }
  }
  __device__ __forceinline__ void get(float (&v)[8]) const { v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w; }
};

// KD/KH/KW > 0 fix the filter extents at compile time (3x3x3 and 1x3x3 cover every reference config: the tap loops
// unroll and the index arithmetic folds); 0 = run-time extents.  NR: 0 raw input, 1 IN, 2 IN+ReLU, 3 run-time flags.
template <typename T, int KD, int KH, int KW, int NR>
__global__ void __launch_bounds__(256, 2) dwconv_fwd_kernel(DwArgs a) {
  extern __shared__ float sm[];
  const int kd = KD > 0 ? KD : a.kd, kh = KH > 0 ? KH : a.kh, kw = KW > 0 ? KW : a.kw;
  const int D = a.D, H = a.H, W = a.W, x_ld = a.x_ld, y_ld = a.y_ld;
  const int C = a.C, taps = kd * kh * kw;
  float* s_w = sm;                         // [taps][C]
  float* s_scale = s_w + taps * C;         // [C]
  float* s_shift = s_scale + C;            // [C]
  float* s_psum = s_shift + C;             // with y_stats: [threads][8] per-thread sums, then [threads][8] squares
  float* s_psq = s_psum + blockDim.x * 8;
  const int b = blockIdx.y, tid = threadIdx.x;
  const int c0 = blockIdx.z * C;            // this block's channel slice [c0, c0 + C) of the Ctot-channel layer
  const double nvox = (double)D * H * W;
  for (int o = tid; o < taps * C; o += blockDim.x) {
    const int t = o / C, c = o % C;
    // [tap][half][cg][4]: a warp's float4 reads (lane = channel group) are contiguous -> no bank conflicts
    s_w[((t * 2 + ((c & 7) >> 2)) * (C >> 3) + (c >> 3)) * 4 + (c & 3)] = a.wlay ? a.w[(int64_t)(c0 + c) * taps + (a.flip ? taps - 1 - t : t)]
                                                                                    : a.w[(a.flip ? taps - 1 - t : t) * a.Ctot + c0 + c];
  }
  for (int c = tid; c < C; c += blockDim.x) {
    float mean = 0.f, rstd = 1.f;
    if (a.x_stats) stats_to_mean_rstd(a.x_stats + ((int64_t)b * a.Ctot + c0 + c) * 2, nvox, a.eps, mean, rstd);
    // IN constants transposed [c%8][cg] for the same reason
    s_scale[(c & 7) * (C >> 3) + (c >> 3)] = rstd; s_shift[(c & 7) * (C >> 3) + (c >> 3)] = -mean * rstd;
  }
  __syncthreads();
  const int ncg = C >> 3, WR = (W + RUN - 1) / RUN;
  const int cg = tid % ncg;                // blockDim.x and the grid stride are multiples of ncg
  const int pd = kd >> 1, ph = kh >> 1, pw = kw >> 1;
  const bool norm = NR == 3 ? a.x_stats != nullptr : NR != 0, relu = NR == 3 ? a.act == 1 : NR == 2;
  const float* sc = s_scale + cg;          // element c at sc[c * ncg]; read at the use site (keeps 16 registers free)
  const float* sh = s_shift + cg;
  float tsum[8], tsq[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) { tsum[c] = 0.f; tsq[c] = 0.f; }
  const T* xb = (const T*)a.x + (int64_t)b * D * H * W * x_ld + a.x_coff + c0 + cg * 8;
  T* yb = (T*)a.y + (int64_t)b * D * H * W * y_ld + a.y_coff + c0 + cg * 8;
  // a block pass covers a compact 2(d) x 4(h) x TWR(w-runs) tile so the 3x3x3 neighbourhoods of its threads
  // overlap in L1 instead of each being fetched from L2
  const Tile tl = make_tile(blockDim.x / ncg, D, H, WR);
  const int rl = tid / ncg, lw = rl % tl.tw, lh = (rl / tl.tw) % tl.th, ldp = rl / (tl.tw * tl.th);
  // 32-bit tile arithmetic: 64-bit div/mod here cost several hundred instructions per item (ncu, round 1)
  const unsigned ntiles = (unsigned)tl.ntiles, nwh = (unsigned)(tl.nw * tl.nh);
  for (unsigned tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const unsigned td_ = tile / nwh, rem = tile - td_ * nwh, th_ = rem / (unsigned)tl.nw, tw_ = rem - th_ * (unsigned)tl.nw;
    const int wr = (int)tw_ * tl.tw + lw;
    const int h = (int)th_ * tl.th + lh;
    const int d = (int)td_ * tl.td + ldp;
    if (wr >= WR || h >= H || d >= D) continue;
    const int w0 = wr * RUN;
    float acc[RUN][8];
#pragma unroll
    for (int o = 0; o < RUN; ++o)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[o][c] = 0.f;
#pragma unroll
    for (int zd = 0; zd < (KD > 0 ? KD : MAXK); ++zd) {
      const int id = d + zd - pd;
      if (zd >= kd || (unsigned)id >= (unsigned)D) continue;
#pragma unroll
      for (int zh = 0; zh < (KH > 0 ? KH : MAXK); ++zh) {
        const int ih = h + zh - ph;
        if (zh >= kh || (unsigned)ih >= (unsigned)H) continue;
        const T* row = xb + ((int64_t)id * H + ih) * W * x_ld;
        const float* wrow = s_w + (zd * kh + zh) * kw * C + cg * 4;
        // all loads of the row first (independent, in flight together), then the arithmetic
        Raw<T> raw[RUN + MAXK - 1];
#pragma unroll
        for (int j = 0; j < RUN + MAXK - 1; ++j) {            // input column w0 - pw + j
          const int iw = w0 - pw + j;
          const bool ok = (j < RUN + kw - 1) && (unsigned)iw < (unsigned)W;
          raw[j].load(row + iw * x_ld, ok);
        }
        float wt[MAXK][8];
#pragma unroll
        for (int k = 0; k < MAXK; ++k) {
          if (k < kw) {
            const float4 w0v = *reinterpret_cast<const float4*>(wrow + k * C), w1v = *reinterpret_cast<const float4*>(wrow + k * C + ncg * 4);
            wt[k][0] = w0v.x; wt[k][1] = w0v.y; wt[k][2] = w0v.z; wt[k][3] = w0v.w;
            wt[k][4] = w1v.x; wt[k][5] = w1v.y; wt[k][6] = w1v.z; wt[k][7] = w1v.w;
          } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) wt[k][c] = 0.f;
          }
        }
#pragma unroll
        for (int j = 0; j < RUN + MAXK - 1; ++j) {
          if (!raw[j].ok) continue;
          float v[8];
          raw[j].get(v);
          if (norm) {
#pragma unroll
            for (int c = 0; c < 8; ++c) { v[c] = fmaf(v[c], sc[c * ncg], sh[c * ncg]); if (relu) v[c] = fmaxf(v[c], 0.f); v[c] = Elem<T>::round(v[c]); }
          } else if (relu) {
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = fmaxf(v[c], 0.f);
          }
#pragma unroll
          for (int o = 0; o < RUN; ++o) {
            const int k = j - o;                               // tap index along W
            if (k >= 0 && k < MAXK) {
#pragma unroll
              for (int c = 0; c < 8; ++c) acc[o][c] = fmaf(v[c], wt[k][c], acc[o][c]);
            }
          }
        }
      }
    }
    T* yrow = yb + (((int64_t)d * H + h) * W + w0) * y_ld;
#pragma unroll
    for (int o = 0; o < RUN; ++o) {
      if (w0 + o < W) {
        st8<T>(yrow + o * y_ld, acc[o]);
        if (a.y_stats) {
#pragma unroll
          for (int c = 0; c < 8; ++c) { const float r2 = Elem<T>::round(acc[o][c]); tsum[c] += r2; tsq[c] = fmaf(r2, r2, tsq[c]); }
        }
      }
    }
  }
  if (a.y_stats) {
    // thread tid = rl * ncg + cg parks its 8 channel partials at [tid * 8] = [rl * C + c]; each channel then sums its
    // rl partials in order, so the block's contribution does not depend on warp timing (DESIGN §4a), and only the
    // order of the fp64 atomics across blocks is free
    *reinterpret_cast<float4*>(s_psum + tid * 8) = make_float4(tsum[0], tsum[1], tsum[2], tsum[3]);
    *reinterpret_cast<float4*>(s_psum + tid * 8 + 4) = make_float4(tsum[4], tsum[5], tsum[6], tsum[7]);
    *reinterpret_cast<float4*>(s_psq + tid * 8) = make_float4(tsq[0], tsq[1], tsq[2], tsq[3]);
    *reinterpret_cast<float4*>(s_psq + tid * 8 + 4) = make_float4(tsq[4], tsq[5], tsq[6], tsq[7]);
    __syncthreads();
    const int rb = blockDim.x / ncg;
    for (int c = tid; c < C; c += blockDim.x) {
      float s = 0.f, q = 0.f;
      for (int r = 0; r < rb; ++r) { s += s_psum[r * C + c]; q += s_psq[r * C + c]; }
      double* st = a.y_stats + ((int64_t)b * a.Ctot + c0 + c) * 2;
      atomicAdd(st, (double)s); atomicAdd(st + 1, (double)q);
    }
  }
}

// dw[tap][c] += sum_{b,voxel} dy[voxel][c] * a[voxel + tap][c];  grid.y = B * kd (one depth tap per block row)
// KHW: 3 = in-plane extent 3x3 fixed at compile time (every reference config), 0 = run-time extents
template <typename T, int KHW>
__global__ void __launch_bounds__(256, 2) dwconv_wgrad_kernel(DwArgs a) {
  extern __shared__ float sm[];
  const int kh = KHW > 0 ? KHW : a.kh, kw = KHW > 0 ? KHW : a.kw;
  const int D = a.D, H = a.H, W = a.W, x_ld = a.x_ld, dy_ld = a.dy_ld;
  const int C = a.C;
  float* s_scale = sm;                     // [C]
  float* s_shift = s_scale + C;
  float* s_acc = s_shift + C;              // [kh*kw][C]
  const int b = blockIdx.y / a.kd, zd = blockIdx.y % a.kd, tid = threadIdx.x;
  const int c0 = blockIdx.z * C;
  const int thw = kh * kw;
  const double nvox = (double)D * H * W;
  for (int c = tid; c < C; c += blockDim.x) {
    float mean = 0.f, rstd = 1.f;
    if (a.x_stats) stats_to_mean_rstd(a.x_stats + ((int64_t)b * a.Ctot + c0 + c) * 2, nvox, a.eps, mean, rstd);
    s_scale[(c & 7) * (C >> 3) + (c >> 3)] = rstd; s_shift[(c & 7) * (C >> 3) + (c >> 3)] = -mean * rstd;
  }
  for (int o = tid; o < thw * C; o += blockDim.x) s_acc[o] = 0.f;
  __syncthreads();
  const int ncg = C >> 3, cg = tid % ncg;
  const int pd = a.kd >> 1, ph = kh >> 1, pw = kw >> 1;
  const bool norm = a.x_stats != nullptr, relu = a.act == 1;
  const float* sc = s_scale + cg;
  const float* sh = s_shift + cg;
  float acc[MAXK * MAXK][8];
#pragma unroll
  for (int t = 0; t < MAXK * MAXK; ++t)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[t][c] = 0.f;
  const T* xb = (const T*)a.x + (int64_t)b * D * H * W * x_ld + a.x_coff + c0 + cg * 8;
  const T* gb = (const T*)a.dy + (int64_t)b * D * H * W * dy_ld + a.dy_coff + c0 + cg * 8;
  const Tile tl = make_tile(blockDim.x / ncg, D, H, W);
  const int rl = tid / ncg, lw = rl % tl.tw, lh = (rl / tl.tw) % tl.th, ldp = rl / (tl.tw * tl.th);
  const unsigned ntiles = (unsigned)tl.ntiles, nwh = (unsigned)(tl.nw * tl.nh);
  for (unsigned tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    // input-stationary: the thread owns one INPUT vector (normalised once) and meets the 9 output gradients
    // of this depth tap that it contributes to:  dw[zd][zh][zw] += dy[id-zd+pd, ih-zh+ph, iw-zw+pw] * a[id,ih,iw]
    const unsigned td_ = tile / nwh, rem = tile - td_ * nwh, th_ = rem / (unsigned)tl.nw, tw_ = rem - th_ * (unsigned)tl.nw;
    const int iw = (int)tw_ * tl.tw + lw;
    const int ih = (int)th_ * tl.th + lh;
    const int id = (int)td_ * tl.td + ldp;
    const int d = id - zd + pd;
    if (iw >= W || ih >= H || id >= D || (unsigned)d >= (unsigned)D) continue;
    Raw<T> rx, rg[MAXK * MAXK];
    rx.load(xb + (((int64_t)id * H + ih) * W + iw) * x_ld, true);
    const T* gc = gb + (((int64_t)d * H + ih) * W + iw) * dy_ld;      // the centre output voxel; neighbours by 32-bit offsets
#pragma unroll
    for (int zh = 0; zh < MAXK; ++zh) {
#pragma unroll
      for (int zw = 0; zw < MAXK; ++zw) {
        const int h = ih - zh + ph, w = iw - zw + pw;
        const bool ok = zh < kh && zw < kw && (unsigned)h < (unsigned)H && (unsigned)w < (unsigned)W;
        rg[zh * MAXK + zw].load(gc + ((ph - zh) * W + (pw - zw)) * dy_ld, ok);
      }
    }
    float v[8];
    rx.get(v);
    if (norm) {
#pragma unroll
      for (int c = 0; c < 8; ++c) { v[c] = fmaf(v[c], sc[c * ncg], sh[c * ncg]); if (relu) v[c] = fmaxf(v[c], 0.f); v[c] = Elem<T>::round(v[c]); }
    } else if (relu) {
#pragma unroll
      for (int c = 0; c < 8; ++c) v[c] = fmaxf(v[c], 0.f);
    }
#pragma unroll
    for (int t = 0; t < MAXK * MAXK; ++t) {
      if (!rg[t].ok) continue;
      float g[8];
      rg[t].get(g);
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[t][c] = fmaf(g[c], v[c], acc[t][c]);
    }
  }
#pragma unroll
  for (int zh = 0; zh < MAXK; ++zh)
#pragma unroll
    for (int zw = 0; zw < MAXK; ++zw)
      if (zh < kh && zw < kw) {
#pragma unroll
        for (int c = 0; c < 8; ++c) atomicAdd(&s_acc[(zh * kw + zw) * C + cg * 8 + c], acc[zh * MAXK + zw][c]);
      }
  __syncthreads();
  for (int o = tid; o < thw * C; o += blockDim.x)
    atomicAdd(a.wlay ? &a.dw[(int64_t)(c0 + o % C) * (a.kd * thw) + zd * thw + o / C]
                     : &a.dw[((int64_t)zd * thw + o / C) * a.Ctot + c0 + o % C], s_acc[o]);
}

int check(const DwArgs& a, int dtype) {
  if (a.B <= 0 || a.D <= 0 || a.H <= 0 || a.W <= 0 || a.C <= 0) return B200SEG_EINVAL;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  if ((a.kd != 1 && a.kd != 3) || (a.kh != 1 && a.kh != 3) || (a.kw != 1 && a.kw != 3)) return B200SEG_EUNSUPPORTED;
  if (a.C % 8 || a.C > 8192 || a.x_ld % 8 || a.x_coff % 8) return B200SEG_EUNSUPPORTED;
  if (a.act != 0 && a.act != 1) return B200SEG_EUNSUPPORTED;
  return B200SEG_OK;
}

// largest multiple-of-8 divisor of C not above 128
int pick_chunk(int C) { for (int ch = 128; ch >= 8; ch -= 8) if (C % ch == 0) return ch; return C; }

int pick_threads(int ncg) { int t = (256 / ncg) * ncg; return t > 0 ? t : ncg; }

}  // namespace

extern "C" int b200seg_dwconv3d_fwd(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                                    const float* w, int flip, void* y, int y_ld, int y_coff, double* y_stats,
                                    int B, int D, int H, int W, int C, int kd, int kh, int kw, int dtype, void* stream) {
  DwArgs a; memset(&a, 0, sizeof(a));
  a.x = x; a.x_ld = x_ld; a.x_coff = x_coff; a.x_stats = x_stats; a.eps = eps; a.act = act; a.w = w; a.flip = flip & 1; a.wlay = (flip >> 1) & 1;
  a.y = y; a.y_ld = y_ld; a.y_coff = y_coff; a.y_stats = y_stats;
  a.B = B; a.D = D; a.H = H; a.W = W; a.C = C; a.kd = kd; a.kh = kh; a.kw = kw;
  int rc = check(a, dtype);
  if (rc) return rc;
  if (!x || !w || !y || y_ld % 8 || y_coff % 8) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  const int taps = kd * kh * kw;
  // channel slices ride in grid.z: a block stages only its slice's filter taps / IN constants and issues only
  // 2*slice statistics atomics, so wide layers (1280-2048 channels on a few hundred voxels) do not drown in
  // per-block setup
  const int chunk = pick_chunk(C);
  a.Ctot = C; a.C = chunk; a.c0 = 0;
  const int nchunk = C / chunk, ncg = chunk / 8, threads = pick_threads(ncg);
  const Tile tl = make_tile(threads / ncg, D, H, (W + RUN - 1) / RUN);
  if (tl.ntiles >= (1LL << 31)) return B200SEG_EUNSUPPORTED;
  int gx = (int)(tl.ntiles < (1 << 30) ? tl.ntiles : (1 << 30));
  int cap = (B200SEG_NUM_SMS * 8 + B * nchunk - 1) / (B * nchunk);
  if (cap < 1) cap = 1;
  if (gx > cap) gx = cap;
  const size_t sm = sizeof(float) * ((size_t)taps * chunk + 2 * chunk + (y_stats ? 16 * (size_t)threads : 0));
  const int nr = !x_stats ? (act ? 3 : 0) : (act == 1 ? 2 : 1);
  const dim3 grid(gx, B, nchunk);
#define B200_DW_FWD(TT, A, Bk, Ck, NRk) dwconv_fwd_kernel<TT, A, Bk, Ck, NRk><<<grid, threads, sm, st>>>(a)
#define B200_DW_FWD_NR(TT, A, Bk, Ck)                                                          \
  do {                                                                                          \
    if (nr == 0) B200_DW_FWD(TT, A, Bk, Ck, 0); else if (nr == 1) B200_DW_FWD(TT, A, Bk, Ck, 1); \
    else if (nr == 2) B200_DW_FWD(TT, A, Bk, Ck, 2); else B200_DW_FWD(TT, A, Bk, Ck, 3);        \
  } while (0)
#define B200_DW_FWD_K(TT)                                                                       \
  do {                                                                                          \
    if (kd == 3 && kh == 3 && kw == 3) B200_DW_FWD_NR(TT, 3, 3, 3);                             \
    else if (kd == 1 && kh == 3 && kw == 3) B200_DW_FWD_NR(TT, 1, 3, 3);                        \
    else B200_DW_FWD(TT, 0, 0, 0, 3);                                                           \
  } while (0)
  if (dtype == B200SEG_F16) B200_DW_FWD_K(__half); else B200_DW_FWD_K(float);
#undef B200_DW_FWD_K
#undef B200_DW_FWD_NR
#undef B200_DW_FWD
  B200_CHECK_LAUNCH("dwconv3d_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_dwconv3d_wgrad(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                                      const void* dy, int dy_ld, int dy_coff, float* dw, int dw_layout,
                                      int B, int D, int H, int W, int C, int kd, int kh, int kw, int dtype, void* stream) {
  DwArgs a; memset(&a, 0, sizeof(a));
  a.wlay = dw_layout ? 1 : 0;
  a.x = x; a.x_ld = x_ld; a.x_coff = x_coff; a.x_stats = x_stats; a.eps = eps; a.act = act;
  a.dy = dy; a.dy_ld = dy_ld; a.dy_coff = dy_coff; a.dw = dw; a.Ctot = C; a.c0 = 0;
  a.B = B; a.D = D; a.H = H; a.W = W; a.C = C; a.kd = kd; a.kh = kh; a.kw = kw;
  int rc = check(a, dtype);
  if (rc) return rc;
  if (!x || !dy || !dw || dy_ld % 8 || dy_coff % 8) return B200SEG_EINVAL;
  const int chunk = pick_chunk(C), nchunk = C / chunk;
  a.Ctot = C; a.C = chunk; a.c0 = 0;
  const int ncg = chunk / 8, threads = pick_threads(ncg);
  const Tile tl = make_tile(threads / ncg, D, H, W);
  if (tl.ntiles >= (1LL << 31)) return B200SEG_EUNSUPPORTED;
  int gx = (int)(tl.ntiles < (1 << 30) ? tl.ntiles : (1 << 30));
  int cap = (B200SEG_NUM_SMS * 4 + B * kd * nchunk - 1) / (B * kd * nchunk);
  if (cap < 1) cap = 1;
  if (gx > cap) gx = cap;
  const size_t sm = sizeof(float) * ((size_t)kh * kw * chunk + 2 * chunk);
  cudaStream_t st = as_stream(stream);
  if (dtype == B200SEG_F16) {
    if (kh == 3 && kw == 3) dwconv_wgrad_kernel<__half, 3><<<dim3(gx, B * kd, nchunk), threads, sm, st>>>(a);
    else dwconv_wgrad_kernel<__half, 0><<<dim3(gx, B * kd, nchunk), threads, sm, st>>>(a);
  } else {
    if (kh == 3 && kw == 3) dwconv_wgrad_kernel<float, 3><<<dim3(gx, B * kd, nchunk), threads, sm, st>>>(a);
    else dwconv_wgrad_kernel<float, 0><<<dim3(gx, B * kd, nchunk), threads, sm, st>>>(a);
  }
  B200_CHECK_LAUNCH("dwconv3d_wgrad");
  return B200SEG_OK;
}
