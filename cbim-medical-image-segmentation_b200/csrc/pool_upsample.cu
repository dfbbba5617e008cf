// pool_upsample.cu — MaxPool3d (kernel==stride) and trilinear upsample (align_corners=True) fused
// with the channel-concat write, both producing the InstanceNorm sums of what they store.
// Reference: nn.MaxPool3d at unet_utils.py:36; F.interpolate(..., 'trilinear', align_corners=True)
// + torch.cat at unet_utils.py:69-71.  HBM-bound; 128-bit channel chunks per thread.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;

template <int VEC, typename T> struct VecIO;
template <typename T> struct VecIO<8, T> {
  static __device__ __forceinline__ void ld(const T* p, float (&v)[8]) { ld8<T>(p, v); }
  static __device__ __forceinline__ void st(T* p, const float (&v)[8]) { st8<T>(p, v); }
};
template <typename T> struct VecIO<1, T> {
  static __device__ __forceinline__ void ld(const T* p, float (&v)[1]) { v[0] = Elem<T>::ld(p); }
  static __device__ __forceinline__ void st(T* p, const float (&v)[1]) { Elem<T>::st(p, v[0]); }
};

// thread -> (voxel slot, channel chunk) mapping, same scheme as instnorm.cu
struct Map { int cpv, vpp, cchunk, vloc; bool active; };
template <int VEC> __device__ __forceinline__ Map make_map(int C) {
  Map m; m.cpv = C / VEC; m.vpp = kThreads / m.cpv; if (m.vpp < 1) m.vpp = 1;
  m.cchunk = threadIdx.x % m.cpv; m.vloc = threadIdx.x / m.cpv; m.active = m.vloc < m.vpp; return m;
}

template <int VEC>
__device__ __forceinline__ void reduce_stats(const float* acc, const Map& m, float* smem, double* gdst, int C) {
  constexpr int W = 2 * VEC;
#pragma unroll
  for (int i = 0; i < W; ++i) smem[threadIdx.x * W + i] = m.active ? acc[i] : 0.f;
  __syncthreads();
  for (int o = threadIdx.x; o < C * 2; o += kThreads) {
    int c = o >> 1, k = o & 1, chunk = c / VEC, e = c % VEC;
    double s = 0.0;
    for (int vl = 0; vl < m.vpp; ++vl) s += (double)smem[(vl * m.cpv + chunk) * W + k * VEC + e];
    atomicAdd(&gdst[c * 2 + k], s);
  }
}

// ------------------------------------------------------------------ max pool
template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
maxpool_fwd_kernel(const T* __restrict__ x, int x_ld, int x_coff, T* __restrict__ y, int y_ld, int y_coff,
                   uint8_t* __restrict__ idx, double* __restrict__ stats, int D, int H, int W, int C,
                   int sd, int sh, int sw, int64_t vpb) {
  extern __shared__ float smem[];
  const int Do = D / sd, Ho = H / sh, Wo = W / sw;
  const int64_t Vo = (int64_t)Do * Ho * Wo;
  const int b = blockIdx.y;
  Map m = make_map<VEC>(C);
  float acc[2 * VEC];
#pragma unroll
  for (int i = 0; i < 2 * VEC; ++i) acc[i] = 0.f;
  if (m.active) {
    int64_t v0 = (int64_t)blockIdx.x * vpb, v1 = v0 + vpb; if (v1 > Vo) v1 = Vo;
    const T* xb = x + (int64_t)b * D * H * W * x_ld + x_coff + m.cchunk * VEC;
    for (int64_t v = v0 + m.vloc; v < v1; v += m.vpp) {
      int wo = (int)(v % Wo); int64_t t = v / Wo; int ho = (int)(t % Ho); int d_o = (int)(t / Ho);
      float best[VEC]; int bi[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) { best[i] = -INFINITY; bi[i] = 0; }
      int k = 0;
      for (int a = 0; a < sd; ++a)
        for (int bq = 0; bq < sh; ++bq)
          for (int c = 0; c < sw; ++c, ++k) {
            int64_t iv = ((int64_t)(d_o * sd + a) * H + (ho * sh + bq)) * W + (wo * sw + c);
            float val[VEC];
            VecIO<VEC, T>::ld(xb + iv * x_ld, val);
#pragma unroll
            for (int i = 0; i < VEC; ++i) if (val[i] > best[i] || k == 0) { best[i] = val[i]; bi[i] = k; }
          }
      int64_t ov = (int64_t)b * Vo + v;
      VecIO<VEC, T>::st(y + ov * y_ld + y_coff + m.cchunk * VEC, best);
      uint8_t* ip = idx + ov * C + m.cchunk * VEC;
      if constexpr (VEC == 8) {
        uint2 pk;
        pk.x = (uint32_t)bi[0] | ((uint32_t)bi[1] << 8) | ((uint32_t)bi[2] << 16) | ((uint32_t)bi[3] << 24);
        pk.y = (uint32_t)bi[4] | ((uint32_t)bi[5] << 8) | ((uint32_t)bi[6] << 16) | ((uint32_t)bi[7] << 24);
        *reinterpret_cast<uint2*>(ip) = pk;
      } else {
        ip[0] = (uint8_t)bi[0];
      }
#pragma unroll
      for (int i = 0; i < VEC; ++i) { acc[i] += best[i]; acc[VEC + i] += best[i] * best[i]; }
    }
  }
  if (stats) reduce_stats<VEC>(acc, m, smem, stats + (int64_t)b * C * 2, C);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
maxpool_bwd_kernel(const T* __restrict__ dy, int dy_ld, int dy_coff, const uint8_t* __restrict__ idx,
                   T* __restrict__ dx, int dx_ld, int dx_coff, int D, int H, int W, int C,
                   int sd, int sh, int sw, int64_t vpb) {
  const int Do = D / sd, Ho = H / sh, Wo = W / sw;
  const int64_t Vo = (int64_t)Do * Ho * Wo;
  const int b = blockIdx.y;
  Map m = make_map<VEC>(C);
  if (!m.active) return;
  int64_t v0 = (int64_t)blockIdx.x * vpb, v1 = v0 + vpb; if (v1 > Vo) v1 = Vo;
  T* dxb = dx + (int64_t)b * D * H * W * dx_ld + dx_coff + m.cchunk * VEC;
  for (int64_t v = v0 + m.vloc; v < v1; v += m.vpp) {
    int wo = (int)(v % Wo); int64_t t = v / Wo; int ho = (int)(t % Ho); int d_o = (int)(t / Ho);
    int64_t ov = (int64_t)b * Vo + v;
    float g[VEC]; int bi[VEC];
    VecIO<VEC, T>::ld(dy + ov * dy_ld + dy_coff + m.cchunk * VEC, g);
    const uint8_t* ip = idx + ov * C + m.cchunk * VEC;
    if constexpr (VEC == 8) {
      uint2 pk = *reinterpret_cast<const uint2*>(ip);
#pragma unroll
      for (int i = 0; i < 4; ++i) { bi[i] = (pk.x >> (8 * i)) & 255; bi[4 + i] = (pk.y >> (8 * i)) & 255; }
    } else {
      bi[0] = ip[0];
    }
    int k = 0;
    for (int a = 0; a < sd; ++a)
      for (int bq = 0; bq < sh; ++bq)
        for (int c = 0; c < sw; ++c, ++k) {
          int64_t iv = ((int64_t)(d_o * sd + a) * H + (ho * sh + bq)) * W + (wo * sw + c);
          float o[VEC];
#pragma unroll
          for (int i = 0; i < VEC; ++i) o[i] = (bi[i] == k) ? g[i] : 0.f;
          VecIO<VEC, T>::st(dxb + iv * dx_ld, o);
        }
  }
}

// ------------------------------------------------------------------ trilinear upsample
// Source index math follows ATen's upsample_trilinear3d (align_corners=True): fp32 scale
// (in-1)/(out-1), src = scale*dst, i0 = (int)src, i1 = i0 + (i0 < in-1), lambda = src - i0.
__device__ __forceinline__ void src_index(float scale, int o, int in_size, int& i0, int& ip, float& l0, float& l1) {
  float s = scale * (float)o;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  ip = (i0 < in_size - 1) ? 1 : 0;
  l1 = s - (float)i0;
  l0 = 1.f - l1;
}
static inline float host_scale(int in_size, int out_size) {
  return out_size > 1 ? (float)(in_size - 1) / (float)(out_size - 1) : 0.f;
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
upsample_fwd_kernel(const T* __restrict__ x, int x_ld, int x_coff, T* __restrict__ y, int y_ld, int y_coff,
                    double* __restrict__ stats, int Di, int Hi, int Wi, int Do, int Ho, int Wo, int C,
                    float rd, float rh, float rw, int64_t vpb) {
  extern __shared__ float smem[];
  const int64_t Vo = (int64_t)Do * Ho * Wo;
  const int b = blockIdx.y;
  Map m = make_map<VEC>(C);
  float acc[2 * VEC];
#pragma unroll
  for (int i = 0; i < 2 * VEC; ++i) acc[i] = 0.f;
  if (m.active) {
    int64_t v0 = (int64_t)blockIdx.x * vpb, v1 = v0 + vpb; if (v1 > Vo) v1 = Vo;
    const T* xb = x + (int64_t)b * Di * Hi * Wi * x_ld + x_coff + m.cchunk * VEC;
    for (int64_t v = v0 + m.vloc; v < v1; v += m.vpp) {
      int wo = (int)(v % Wo); int64_t t = v / Wo; int ho = (int)(t % Ho); int d_o = (int)(t / Ho);
      int d0, dp, h0, hp, w0, wp; float ld0, ld1, lh0, lh1, lw0, lw1;
      src_index(rd, d_o, Di, d0, dp, ld0, ld1);
      src_index(rh, ho, Hi, h0, hp, lh0, lh1);
      src_index(rw, wo, Wi, w0, wp, lw0, lw1);
      float v000[VEC], v001[VEC], v010[VEC], v011[VEC], v100[VEC], v101[VEC], v110[VEC], v111[VEC];
      auto at = [&](int d, int h, int w) { return xb + (((int64_t)d * Hi + h) * Wi + w) * x_ld; };
      VecIO<VEC, T>::ld(at(d0, h0, w0), v000);
      VecIO<VEC, T>::ld(at(d0, h0, w0 + wp), v001);
      VecIO<VEC, T>::ld(at(d0, h0 + hp, w0), v010);
      VecIO<VEC, T>::ld(at(d0, h0 + hp, w0 + wp), v011);
      VecIO<VEC, T>::ld(at(d0 + dp, h0, w0), v100);
      VecIO<VEC, T>::ld(at(d0 + dp, h0, w0 + wp), v101);
      VecIO<VEC, T>::ld(at(d0 + dp, h0 + hp, w0), v110);
      VecIO<VEC, T>::ld(at(d0 + dp, h0 + hp, w0 + wp), v111);
      float o[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float r = ld0 * (lh0 * (lw0 * v000[i] + lw1 * v001[i]) + lh1 * (lw0 * v010[i] + lw1 * v011[i])) +
                  ld1 * (lh0 * (lw0 * v100[i] + lw1 * v101[i]) + lh1 * (lw0 * v110[i] + lw1 * v111[i]));
        r = Elem<T>::round(r);
        o[i] = r; acc[i] += r; acc[VEC + i] += r * r;
      }
      VecIO<VEC, T>::st(y + ((int64_t)b * Vo + v) * y_ld + y_coff + m.cchunk * VEC, o);
    }
  }
  if (stats) reduce_stats<VEC>(acc, m, smem, stats + (int64_t)b * C * 2, C);
}

// gather-form backward: each INPUT voxel collects from the output voxels whose stencil touches it
// (deterministic, no atomics, no zero-fill).  Per axis at most kMaxTaps output indices contribute, except along an
// input axis of length 1, which every output index reads (see AxisTab).
constexpr int kMaxTaps = 12;
__device__ __forceinline__ int axis_taps(float scale, int i, int in_size, int out_size, int (&oo)[kMaxTaps], float (&ww)[kMaxTaps]) {
  int n = 0;
  int lo, hi;
  if (scale > 0.f) {
    lo = (int)floorf((float)(i - 1) / scale) - 1;
    hi = (int)ceilf((float)(i + 1) / scale) + 1;
  } else { lo = 0; hi = out_size - 1; }
  if (lo < 0) lo = 0;
  if (hi > out_size - 1) hi = out_size - 1;
  for (int o = lo; o <= hi; ++o) {
    int i0, ip; float l0, l1;
    src_index(scale, o, in_size, i0, ip, l0, l1);
    float w = 0.f;
    if (i0 == i) w += l0;
    if (i0 + ip == i) w += (ip ? l1 : l1);   // when ip==0 both corners alias the same voxel
    if (i0 != i && i0 + ip != i) continue;
    if (n < kMaxTaps) { oo[n] = o; ww[n] = w; ++n; }
  }
  return n;
}

// per-axis tap tables, built once per block in shared memory: for input index i the output indices whose
// stencil touches i and their (non-zero) weights.  An input axis of length 1 feeds every output index with weight 1,
// however many there are: its single entry says so with n = -out_size instead of listing taps.
struct AxisTab { int n; int o[kMaxTaps]; float w[kMaxTaps]; };
__device__ __forceinline__ int tap_count(const AxisTab& t) { return t.n < 0 ? -t.n : t.n; }
__device__ __forceinline__ int tap_out(const AxisTab& t, int k) { return t.n < 0 ? k : t.o[k]; }
__device__ __forceinline__ float tap_w(const AxisTab& t, int k) { return t.n < 0 ? 1.f : t.w[k]; }

__device__ __forceinline__ void build_axis_table(AxisTab* tab, float scale, int in_size, int out_size) {
  if (in_size == 1) {
    if (threadIdx.x == 0) tab[0].n = -out_size;
    return;
  }
  for (int i = threadIdx.x; i < in_size; i += kThreads) {
    int oo[kMaxTaps]; float ww[kMaxTaps];
    const int n = axis_taps(scale, i, in_size, out_size, oo, ww);
    int m = 0;
    for (int k = 0; k < n; ++k)
      if (ww[k] != 0.f) { tab[i].o[m] = oo[k]; tab[i].w[m] = ww[k]; ++m; }
    tab[i].n = m;
  }
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads)
upsample_bwd_kernel(const T* __restrict__ dy, int dy_ld, int dy_coff, T* __restrict__ dx, int dx_ld, int dx_coff,
                    int accumulate, int Di, int Hi, int Wi, int Do, int Ho, int Wo, int C,
                    float rd, float rh, float rw, int64_t vpb) {
  extern __shared__ float smem[];
  AxisTab* td = reinterpret_cast<AxisTab*>(smem);
  AxisTab* th = td + Di;
  AxisTab* tw = th + Hi;
  build_axis_table(td, rd, Di, Do);
  build_axis_table(th, rh, Hi, Ho);
  build_axis_table(tw, rw, Wi, Wo);
  __syncthreads();
  const int64_t Vi = (int64_t)Di * Hi * Wi;
  const int b = blockIdx.y;
  Map m = make_map<VEC>(C);
  if (!m.active) return;
  int64_t v0 = (int64_t)blockIdx.x * vpb, v1 = v0 + vpb; if (v1 > Vi) v1 = Vi;
  const T* dyb = dy + (int64_t)b * Do * Ho * Wo * dy_ld + dy_coff + m.cchunk * VEC;
  for (int64_t v = v0 + m.vloc; v < v1; v += m.vpp) {
    int wi = (int)(v % Wi); int64_t t = v / Wi; int hi = (int)(t % Hi); int di = (int)(t / Hi);
    const AxisTab& ad = td[di]; const AxisTab& ah = th[hi]; const AxisTab& aw = tw[wi];
    float acc[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    const int nd = tap_count(ad), nh = tap_count(ah), nw = tap_count(aw);
    for (int a = 0; a < nd; ++a)
      for (int bq = 0; bq < nh; ++bq) {
        const float wdh = tap_w(ad, a) * tap_w(ah, bq);
        const T* row = dyb + (((int64_t)tap_out(ad, a) * Ho + tap_out(ah, bq)) * Wo) * dy_ld;
        for (int c = 0; c < nw; ++c) {
          float g[VEC];
          VecIO<VEC, T>::ld(row + (int64_t)tap_out(aw, c) * dy_ld, g);
          const float wt = wdh * tap_w(aw, c);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] += wt * g[i];
        }
      }
    T* dp = dx + ((int64_t)b * Vi + v) * dx_ld + dx_coff + m.cchunk * VEC;
    if (accumulate) {
      float o[VEC];
      VecIO<VEC, T>::ld(dp, o);
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[i] += o[i];
    }
    VecIO<VEC, T>::st(dp, acc);
  }
}

inline bool vec_ok(const void* p, int ld, int coff, int C) {
  return (C % 8 == 0) && (ld % 8 == 0) && (coff % 8 == 0) && (C / 8 <= kThreads) &&
         ((reinterpret_cast<uintptr_t>(p) % 16) == 0);
}
inline int64_t pick_vpb(int64_t V, int B) {
  int64_t want = (int64_t)B200SEG_NUM_SMS * 8 / (B > 0 ? B : 1);
  if (want < 1) want = 1;
  int64_t vpb = (V + want - 1) / want;
  if (vpb < 16) vpb = 16;          // small, channel-heavy levels still need >= one block per SM
  return vpb;
}

}  // namespace

#define DISPATCH_TV(DT, VECOK, ...)                                         \
  if ((DT) == B200SEG_F16) {                                                 \
    using T = __half;                                                        \
    if (VECOK) { constexpr int VEC = 8; __VA_ARGS__ } else { constexpr int VEC = 1; __VA_ARGS__ } \
  } else if ((DT) == B200SEG_F32) {                                          \
    using T = float;                                                         \
    if (VECOK) { constexpr int VEC = 8; __VA_ARGS__ } else { constexpr int VEC = 1; __VA_ARGS__ } \
  } else return B200SEG_EINVAL;

extern "C" int b200seg_maxpool3d_fwd(const void* x, int x_ld, int x_coff, void* y, int y_ld, int y_coff,
                                     uint8_t* idx, double* y_stats, int B, int D, int H, int W, int C,
                                     int sd, int sh, int sw, int dtype, void* stream) {
  if (!x || !y || !idx || B <= 0 || D <= 0 || H <= 0 || W <= 0 || C <= 0 || sd <= 0 || sh <= 0 || sw <= 0) return B200SEG_EINVAL;
  if (sd * sh * sw > 255 || D / sd < 1 || H / sh < 1 || W / sw < 1) return B200SEG_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  int64_t Vo = (int64_t)(D / sd) * (H / sh) * (W / sw);
  int64_t vpb = pick_vpb(Vo, B);
  dim3 grid(ceil_div(Vo, vpb), B);
  bool vok = vec_ok(x, x_ld, x_coff, C) && vec_ok(y, y_ld, y_coff, C) && ((reinterpret_cast<uintptr_t>(idx) % 8) == 0);
  if (!vok && C > kThreads) return B200SEG_EUNSUPPORTED;
  DISPATCH_TV(dtype, vok, {
    size_t sm = sizeof(float) * kThreads * 2 * VEC;
    maxpool_fwd_kernel<T, VEC><<<grid, kThreads, sm, st>>>((const T*)x, x_ld, x_coff, (T*)y, y_ld, y_coff, idx, y_stats,
                                                          D, H, W, C, sd, sh, sw, vpb);
  })
  B200_CHECK_LAUNCH("maxpool_fwd_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_maxpool3d_bwd(const void* dy, int dy_ld, int dy_coff, const uint8_t* idx, void* dx,
                                     int dx_ld, int dx_coff, int B, int D, int H, int W, int C, int sd, int sh,
                                     int sw, int dtype, void* stream) {
  if (!dy || !dx || !idx || B <= 0 || D <= 0 || H <= 0 || W <= 0 || C <= 0 || sd <= 0 || sh <= 0 || sw <= 0) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  int64_t Vo = (int64_t)(D / sd) * (H / sh) * (W / sw);
  int64_t vpb = pick_vpb(Vo, B);
  dim3 grid(ceil_div(Vo, vpb), B);
  bool vok = vec_ok(dy, dy_ld, dy_coff, C) && vec_ok(dx, dx_ld, dx_coff, C) && ((reinterpret_cast<uintptr_t>(idx) % 8) == 0);
  if (!vok && C > kThreads) return B200SEG_EUNSUPPORTED;
  DISPATCH_TV(dtype, vok, {
    maxpool_bwd_kernel<T, VEC><<<grid, kThreads, 0, st>>>((const T*)dy, dy_ld, dy_coff, idx, (T*)dx, dx_ld, dx_coff,
                                                          D, H, W, C, sd, sh, sw, vpb);
  })
  B200_CHECK_LAUNCH("maxpool_bwd_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_upsample_trilinear_fwd(const void* x, int x_ld, int x_coff, void* y, int y_ld, int y_coff,
                                              double* y_stats, int B, int Di, int Hi, int Wi, int Do, int Ho,
                                              int Wo, int C, int dtype, void* stream) {
  if (!x || !y || B <= 0 || Di <= 0 || Hi <= 0 || Wi <= 0 || Do <= 0 || Ho <= 0 || Wo <= 0 || C <= 0) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  int64_t Vo = (int64_t)Do * Ho * Wo;
  int64_t vpb = pick_vpb(Vo, B);
  dim3 grid(ceil_div(Vo, vpb), B);
  bool vok = vec_ok(x, x_ld, x_coff, C) && vec_ok(y, y_ld, y_coff, C);
  if (!vok && C > kThreads) return B200SEG_EUNSUPPORTED;
  float rd = host_scale(Di, Do), rh = host_scale(Hi, Ho), rw = host_scale(Wi, Wo);
  DISPATCH_TV(dtype, vok, {
    size_t sm = sizeof(float) * kThreads * 2 * VEC;
    upsample_fwd_kernel<T, VEC><<<grid, kThreads, sm, st>>>((const T*)x, x_ld, x_coff, (T*)y, y_ld, y_coff, y_stats,
                                                           Di, Hi, Wi, Do, Ho, Wo, C, rd, rh, rw, vpb);
  })
  B200_CHECK_LAUNCH("upsample_fwd_kernel");
  return B200SEG_OK;
}

extern "C" int b200seg_upsample_trilinear_bwd(const void* dy, int dy_ld, int dy_coff, void* dx, int dx_ld,
                                              int dx_coff, int accumulate, int B, int Di, int Hi, int Wi,
                                              int Do, int Ho, int Wo, int C, int dtype, void* stream) {
  if (!dy || !dx || B <= 0 || Di <= 0 || Hi <= 0 || Wi <= 0 || Do <= 0 || Ho <= 0 || Wo <= 0 || C <= 0) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  int64_t Vi = (int64_t)Di * Hi * Wi;
  int64_t vpb = pick_vpb(Vi, B);
  dim3 grid(ceil_div(Vi, vpb), B);
  bool vok = vec_ok(dy, dy_ld, dy_coff, C) && vec_ok(dx, dx_ld, dx_coff, C);
  if (!vok && C > kThreads) return B200SEG_EUNSUPPORTED;
  float rd = host_scale(Di, Do), rh = host_scale(Hi, Ho), rw = host_scale(Wi, Wo);
  // the gather needs every contributing output index to fit in kMaxTaps per axis (a length-1 input axis, rd == 0
  // with Di == 1, lists none: its table entry covers every output index)
  if ((Do > 1 && rd > 0.f && 2.0f / rd + 3.0f > (float)kMaxTaps && Do > kMaxTaps) ||
      (Ho > 1 && rh > 0.f && 2.0f / rh + 3.0f > (float)kMaxTaps && Ho > kMaxTaps) ||
      (Wo > 1 && rw > 0.f && 2.0f / rw + 3.0f > (float)kMaxTaps && Wo > kMaxTaps))
    return B200SEG_EUNSUPPORTED;
  const size_t tab_bytes = sizeof(AxisTab) * (size_t)(Di + Hi + Wi);
  if (tab_bytes > 96 * 1024) return B200SEG_EUNSUPPORTED;
  DISPATCH_TV(dtype, vok, {
    if (tab_bytes > 48 * 1024) cudaFuncSetAttribute(upsample_bwd_kernel<T, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tab_bytes);
    upsample_bwd_kernel<T, VEC><<<grid, kThreads, tab_bytes, st>>>((const T*)dy, dy_ld, dy_coff, (T*)dx, dx_ld, dx_coff, accumulate,
                                                           Di, Hi, Wi, Do, Ho, Wo, C, rd, rh, rw, vpb);
  })
  B200_CHECK_LAUNCH("upsample_bwd_kernel");
  return B200SEG_OK;
}
