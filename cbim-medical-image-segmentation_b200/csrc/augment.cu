// augment.cu — device side of the reference's GPU augmentation path (`aug_device: gpu`, SURVEY.md §8f.3):
// training/augmentation.py and its caller training/dataset/dim3/dataset_kits.py:116-153.
//
//   * aug_resample: crop_3d(random, size+60) -> random_scale_rotate_translate_3d (F.affine_grid + F.grid_sample,
//     trilinear for the image / nearest for the label, zeros padding, align_corners=True; augmentation.py:226-291)
//     -> crop_3d(center) (:320-343) -> mirror x3 (:176-197) as ONE gather: only the voxels of the final training patch
//     are ever computed, the 60-voxel margin and the three flips never exist in HBM.  With `theta == NULL` it is the
//     exact-copy branch (random crop + flips).  The epilogue leaves {min, max, sum, sum^2} of the produced image in
//     `stats`, so the first intensity op needs no extra pass.
//   * aug_pointwise: brightness_multiply / brightness_additive / gamma (pow pass + renormalise pass) / contrast /
//     gaussian_noise (augmentation.py:14-16,66-173) — each reads the statistics its predecessor left on the device and
//     leaves those of its own output, so the chain has no reduction passes and no host synchronisation.
//   * aug_gaussian_blur: gaussian_blur (:18-64).  The reference convolves with the dense k^3 kernel (k = 5 or 7); the
//     3-D Gaussian is the outer product of three 1-D ones, so one CTA stages a halo tile in shared memory and runs
//     the x, y and z passes on chip: 1 read + 1 write of the volume instead of k^3 MACs per voxel.
// All HBM-bound (gather / elementwise); images fp32 [C][D][H][W] (the reference's [1,C,D,H,W]), labels uint8 or int64.
#include "common.cuh"

namespace {

// ---- order-preserving float <-> uint key, so min / max can use integer atomics
__device__ __forceinline__ unsigned f2key(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// stats row (32 bytes): {uint64 min key, uint64 max key, double sum, double sumsq}; init {0xffffffff, 0, 0.0, 0.0}
struct StatRow { unsigned long long kmin, kmax; double sum, sumsq; };

struct RowStats { float mn, mx; double n, mean, std; };     // std unbiased (torch.Tensor.std default)
__device__ __forceinline__ RowStats read_stats(const StatRow* s, double n) {
  RowStats r;
  r.mn = key2f((unsigned)s->kmin); r.mx = key2f((unsigned)s->kmax);
  r.n = n; r.mean = s->sum / n;
  double var = (s->sumsq - n * r.mean * r.mean) / (n > 1.0 ? n - 1.0 : 1.0);
  r.std = sqrt(var > 0.0 ? var : 0.0);
  return r;
}

// block-wide merge of per-thread {min, max, sum, sumsq} into one stats row (256 threads)
__device__ __forceinline__ void block_stats_commit(float mn, float mx, double s, double q, StatRow* out) {
  __shared__ float s_mn[8], s_mx[8];
  __shared__ double s_s[8], s_q[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  s = warp_sum_d(s); q = warp_sum_d(q);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_mn[w] = mn; s_mx[w] = mx; s_s[w] = s; s_q[w] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = blockDim.x >> 5;
    for (int i = 1; i < nw; ++i) { mn = fminf(mn, s_mn[i]); mx = fmaxf(mx, s_mx[i]); s += s_s[i]; q += s_q[i]; }
    atomicMin(&out->kmin, (unsigned long long)f2key(mn));
    atomicMax(&out->kmax, (unsigned long long)f2key(mx));
    atomicAdd(&out->sum, s);
    atomicAdd(&out->sumsq, q);
  }
  __syncthreads();
}

struct Geom {
  int D, H, W;          // full source volume
  int z0, y0, x0;       // origin of the sub-volume the affine grid is defined on (first crop)
  int Ds, Hs, Ws;       // its extent
  int oz, oy, ox;       // origin of the output patch inside the sub-volume (second, centre crop)
  int Do, Ho, Wo;       // output patch
  int flip;             // bit0: flip D (axis 0), bit1: flip H, bit2: flip W — applied to the OUTPUT index
  float th[12];         // theta rows (x, y, z) as handed to F.affine_grid; unused in copy mode
};

// one thread = one output voxel (all image channels + the label); writes coalesced along W
template <typename TL, typename TLO, bool AFFINE>
__global__ void __launch_bounds__(256) aug_resample_kernel(const float* __restrict__ img, const TL* __restrict__ lab, int C, Geom g,
                                                           float* __restrict__ oimg, TLO* __restrict__ olab, StatRow* __restrict__ stats,
                                                           int stats_rows) {
  const int64_t Vo = (int64_t)g.Do * g.Ho * g.Wo, Vs = (int64_t)g.D * g.H * g.W;
  float mn = INFINITY, mx = -INFINITY; double sm = 0.0, sq = 0.0;
  // per-row statistics need one accumulator set per channel; rows > 1 only when stats_rows == C (per-channel use)
  for (int c0 = 0; c0 < (stats_rows > 1 ? C : 1); ++c0) {
    mn = INFINITY; mx = -INFINITY; sm = 0.0; sq = 0.0;
    const int cb = stats_rows > 1 ? c0 : 0, ce = stats_rows > 1 ? c0 + 1 : C;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < Vo; i += (int64_t)gridDim.x * 256) {
      const int wo = (int)(i % g.Wo); const int64_t t = i / g.Wo; const int ho = (int)(t % g.Ho); const int dd = (int)(t / g.Ho);
      // mirror: output index o holds the un-mirrored patch's element (extent-1-o)
      const int pd = (g.flip & 1) ? g.Do - 1 - dd : dd, ph = (g.flip & 2) ? g.Ho - 1 - ho : ho, pw = (g.flip & 4) ? g.Wo - 1 - wo : wo;
      const int sd = pd + g.oz, sh = ph + g.oy, sw = pw + g.ox;       // index in the sub-volume's grid
      if (!AFFINE) {
        const int64_t src = ((int64_t)(sd + g.z0) * g.H + (sh + g.y0)) * g.W + (sw + g.x0);
        for (int c = cb; c < ce; ++c) {
          const float v = img[c * Vs + src];
          oimg[c * Vo + i] = v;
          mn = fminf(mn, v); mx = fmaxf(mx, v); sm += v; sq += (double)v * v;
        }
        if (c0 == 0 && lab) olab[i] = (TLO)lab[src];
        continue;
      }
      // F.affine_grid(align_corners=True): base coordinate of index j on an axis of n points = 2j/(n-1) - 1 (0 if n == 1)
      const float bx = g.Ws > 1 ? (2.f * sw) / (float)(g.Ws - 1) - 1.f : 0.f;
      const float by = g.Hs > 1 ? (2.f * sh) / (float)(g.Hs - 1) - 1.f : 0.f;
      const float bz = g.Ds > 1 ? (2.f * sd) / (float)(g.Ds - 1) - 1.f : 0.f;
      const float gx = fmaf(bx, g.th[0], fmaf(by, g.th[1], fmaf(bz, g.th[2], g.th[3])));
      const float gy = fmaf(bx, g.th[4], fmaf(by, g.th[5], fmaf(bz, g.th[6], g.th[7])));
      const float gz = fmaf(bx, g.th[8], fmaf(by, g.th[9], fmaf(bz, g.th[10], g.th[11])));
      // F.grid_sample(align_corners=True): unnormalise ((g+1)/2)*(n-1)
      const float ix = (gx + 1.f) * 0.5f * (float)(g.Ws - 1);
      const float iy = (gy + 1.f) * 0.5f * (float)(g.Hs - 1);
      const float iz = (gz + 1.f) * 0.5f * (float)(g.Ds - 1);
      const float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
      const int x_0 = (int)fx, y_0 = (int)fy, z_0 = (int)fz;
      const float tx = ix - fx, ty = iy - fy, tz = iz - fz;
      // zeros padding: a corner outside the SUB-volume contributes nothing (the first crop happened before sampling)
      const bool vx0 = (unsigned)x_0 < (unsigned)g.Ws, vx1 = (unsigned)(x_0 + 1) < (unsigned)g.Ws;
      const bool vy0 = (unsigned)y_0 < (unsigned)g.Hs, vy1 = (unsigned)(y_0 + 1) < (unsigned)g.Hs;
      const bool vz0 = (unsigned)z_0 < (unsigned)g.Ds, vz1 = (unsigned)(z_0 + 1) < (unsigned)g.Ds;
      const int64_t base = ((int64_t)(z_0 + g.z0) * g.H + (y_0 + g.y0)) * g.W + (x_0 + g.x0);
      const int64_t sH = g.W, sD = (int64_t)g.H * g.W;
      // corner weights in grid_sample's naming: tnw = (1-tx)(1-ty)(1-tz) ... bse = tx*ty*tz
      const float w000 = (1.f - tx) * (1.f - ty) * (1.f - tz), w001 = tx * (1.f - ty) * (1.f - tz);
      const float w010 = (1.f - tx) * ty * (1.f - tz), w011 = tx * ty * (1.f - tz);
      const float w100 = (1.f - tx) * (1.f - ty) * tz, w101 = tx * (1.f - ty) * tz;
      const float w110 = (1.f - tx) * ty * tz, w111 = tx * ty * tz;
      for (int c = cb; c < ce; ++c) {
        const float* p = img + c * Vs + base;
        float v = 0.f;
        if (vz0 && vy0 && vx0) v += p[0] * w000;
        if (vz0 && vy0 && vx1) v += p[1] * w001;
        if (vz0 && vy1 && vx0) v += p[sH] * w010;
        if (vz0 && vy1 && vx1) v += p[sH + 1] * w011;
        if (vz1 && vy0 && vx0) v += p[sD] * w100;
        if (vz1 && vy0 && vx1) v += p[sD + 1] * w101;
        if (vz1 && vy1 && vx0) v += p[sD + sH] * w110;
        if (vz1 && vy1 && vx1) v += p[sD + sH + 1] * w111;
        oimg[c * Vo + i] = v;
        mn = fminf(mn, v); mx = fmaxf(mx, v); sm += v; sq += (double)v * v;
      }
      if (c0 == 0 && lab) {
        // mode='nearest': std::nearbyint (round half to even), zeros outside
        const int nx = (int)nearbyintf(ix), ny = (int)nearbyintf(iy), nz = (int)nearbyintf(iz);
        TLO l = 0;
        if ((unsigned)nx < (unsigned)g.Ws && (unsigned)ny < (unsigned)g.Hs && (unsigned)nz < (unsigned)g.Ds)
          l = (TLO)lab[((int64_t)(nz + g.z0) * g.H + (ny + g.y0)) * g.W + (nx + g.x0)];
        olab[i] = l;
      }
    }
    if (stats) block_stats_commit(mn, mx, sm, sq, stats + (stats_rows > 1 ? c0 : 0));
  }
}

// ---- counter-based normal generator: Philox4x32-10 keyed by (seed), counter = element index / 4, Box-Muller
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ __forceinline__ void philox_normal4(uint64_t seed, uint64_t ctr, float (&z)[4]) {
  uint32_t c[4] = {(uint32_t)ctr, (uint32_t)(ctr >> 32), 0u, 0u};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) { philox_round(c, k0, k1); k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
  const float inv = 2.3283064365386963e-10f;   // 2^-32
  const float u0 = ((float)c[0] + 0.5f) * inv, u1 = ((float)c[1] + 0.5f) * inv;
  const float u2 = ((float)c[2] + 0.5f) * inv, u3 = ((float)c[3] + 0.5f) * inv;
  const float r0 = sqrtf(-2.f * __logf(fmaxf(u0, 1e-30f))), r1 = sqrtf(-2.f * __logf(fmaxf(u2, 1e-30f)));
  float s0, c0, s1, c1;
  __sincosf(6.283185307179586f * u1, &s0, &c0);
  __sincosf(6.283185307179586f * u3, &s1, &c1);
  z[0] = r0 * c0; z[1] = r0 * s0; z[2] = r1 * c1; z[3] = r1 * s1;
}

enum { OP_MUL = 0, OP_ADD = 1, OP_GAMMA_POW = 2, OP_RENORM = 3, OP_CONTRAST = 4, OP_NOISE = 5, OP_STATS = 6 };
struct PwParams { float a[8]; float b[8]; };     // per-row scalars (rows <= 8)

// y = op(x); rows = number of independent statistic rows (the reference's view(tmp_C, -1)); n = elements per row.
// sin = statistics of x (ops that need them), sin2 = statistics saved before the gamma pow pass (RENORM),
// sout = statistics of y (nullable), accumulated.
template <int OP>
__global__ void __launch_bounds__(256) aug_pointwise_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int64_t n,
                                                            PwParams p, const StatRow* __restrict__ sin, const StatRow* __restrict__ sin2,
                                                            StatRow* __restrict__ sout, uint64_t seed) {
  for (int r = 0; r < rows; ++r) {
    const float* xr = x + (int64_t)r * n;
    float* yr = y ? y + (int64_t)r * n : nullptr;
    RowStats st = {}, st2 = {};
    if (OP == OP_GAMMA_POW || OP == OP_RENORM || OP == OP_CONTRAST) st = read_stats(sin + r, (double)n);
    if (OP == OP_RENORM) st2 = read_stats(sin2 + r, (double)n);
    const float a = p.a[r], b = p.b[r];
    const float rng = st.mx - st.mn, mean = (float)st.mean;
    // RENORM: y = (x - mean_now) / std_now * std_before + mean_before   (augmentation.py:133-135)
    const float rn_mean = (float)st.mean, rn_std = (float)st.std, rn_std0 = (float)st2.std, rn_mean0 = (float)st2.mean;
    float mn = INFINITY, mx = -INFINITY; double sm = 0.0, sq = 0.0;
    const int64_t n4 = (n + 3) / 4;
    const bool vec = ((reinterpret_cast<uintptr_t>(xr) | reinterpret_cast<uintptr_t>(yr)) & 15) == 0;     // 16-byte rows
    for (int64_t i4 = (int64_t)blockIdx.x * 256 + threadIdx.x; i4 < n4; i4 += (int64_t)gridDim.x * 256) {
      float z[4] = {0.f, 0.f, 0.f, 0.f};
      if (OP == OP_NOISE) philox_normal4(seed + (uint64_t)r * 0x9E3779B97F4A7C15ull, (uint64_t)i4, z);
      const int64_t i0 = i4 * 4;
      const int cnt = (int)((n - i0) < 4 ? (n - i0) : 4);
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (vec && cnt == 4) { const float4 f = *reinterpret_cast<const float4*>(xr + i0); v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
      else { for (int k = 0; k < cnt; ++k) v[k] = xr[i0 + k]; }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (OP == OP_MUL) v[k] = v[k] * a;
        else if (OP == OP_ADD) v[k] = v[k] + a;
        else if (OP == OP_GAMMA_POW) v[k] = powf((v[k] - st.mn) / rng, a) * rng + st.mn;        // :131
        else if (OP == OP_RENORM) v[k] = (v[k] - rn_mean) / rn_std * rn_std0 + rn_mean0;
        else if (OP == OP_CONTRAST) { v[k] = (v[k] - mean) * a + mean; if (b != 0.f) v[k] = fminf(fmaxf(v[k], st.mn), st.mx); }   // :163-166
        else if (OP == OP_NOISE) v[k] = v[k] + z[k] * a + b;                                       // :14-16
        if (k < cnt) { mn = fminf(mn, v[k]); mx = fmaxf(mx, v[k]); sm += v[k]; sq += (double)v[k] * v[k]; }
      }
      if (yr) {
        if (vec && cnt == 4) *reinterpret_cast<float4*>(yr + i0) = make_float4(v[0], v[1], v[2], v[3]);
        else { for (int k = 0; k < cnt; ++k) yr[i0 + k] = v[k]; }
      }
    }
    if (sout) block_stats_commit(mn, mx, sm, sq, sout + r);
  }
}

// ---- separable Gaussian blur, one pass over HBM ------------------------------------------------------------------
constexpr int BT_Z = 8, BT_Y = 8, BT_X = 32, BR_MAX = 3;      // output tile, maximum radius (k = 7)
struct BlurW { float w[2 * BR_MAX + 1]; };

// DEPTH = false is the 2-D blur of a [C][1][H][W] image (F.conv2d with the k x k kernel): tiles one plane deep and
// no z pass, since the normalised 2-D kernel is the outer product of the two normalised 1-D ones.
template <bool DEPTH>
__global__ void __launch_bounds__(256) aug_blur_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int D, int H, int W, int R,
                                                       BlurW kw, StatRow* __restrict__ sout, int stats_rows) {
  extern __shared__ float sm[];
  constexpr int TZ = DEPTH ? BT_Z : 1;
  const int RZ = DEPTH ? R : 0;
  const int EZ = TZ + 2 * RZ, EY = BT_Y + 2 * R, EX = BT_X + 2 * R;
  float* s_in = sm;                          // [EZ][EY][EX]
  float* s_x = sm + EZ * EY * EX;            // [EZ][EY][BT_X]   after the x pass
  float* s_y = s_x + EZ * EY * BT_X;         // [EZ][BT_Y][BT_X] after the y pass
  const int tx = (W + BT_X - 1) / BT_X, ty = (H + BT_Y - 1) / BT_Y, tz = (D + TZ - 1) / TZ;
  const int64_t tiles = (int64_t)C * tz * ty * tx, V = (int64_t)D * H * W;
  float mn = INFINITY, mx = -INFINITY; double ssum = 0.0, ssq = 0.0;
  int cur_c = -1;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    int64_t q = t;
    const int bx = (int)(q % tx); q /= tx; const int by = (int)(q % ty); q /= ty; const int bz = (int)(q % tz); const int c = (int)(q / tz);
    if (sout && stats_rows > 1 && c != cur_c) {
      if (cur_c >= 0) block_stats_commit(mn, mx, ssum, ssq, sout + cur_c);
      mn = INFINITY; mx = -INFINITY; ssum = 0.0; ssq = 0.0;
    }
    cur_c = c;
    const float* xc = x + c * V;
    const int z0 = bz * TZ - RZ, y0 = by * BT_Y - R, x0 = bx * BT_X - R;
    for (int i = threadIdx.x; i < EZ * EY * EX; i += 256) {
      const int lx = i % EX, ly = (i / EX) % EY, lz = i / (EX * EY);
      const int gz = z0 + lz, gy = y0 + ly, gx = x0 + lx;
      float v = 0.f;                         // F.conv3d zero padding
      if ((unsigned)gz < (unsigned)D && (unsigned)gy < (unsigned)H && (unsigned)gx < (unsigned)W) v = xc[((int64_t)gz * H + gy) * W + gx];
      s_in[i] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < EZ * EY * BT_X; i += 256) {
      const int lx = i % BT_X, r = i / BT_X;
      const float* p = s_in + r * EX + lx;
      float a = 0.f;
      for (int k = 0; k <= 2 * R; ++k) a = fmaf(p[k], kw.w[k], a);
      s_x[i] = a;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < EZ * BT_Y * BT_X; i += 256) {
      const int lx = i % BT_X, ly = (i / BT_X) % BT_Y, lz = i / (BT_X * BT_Y);
      const float* p = s_x + (lz * EY + ly) * BT_X + lx;
      float a = 0.f;
      for (int k = 0; k <= 2 * R; ++k) a = fmaf(p[k * BT_X], kw.w[k], a);
      s_y[i] = a;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < TZ * BT_Y * BT_X; i += 256) {
      const int lx = i % BT_X, ly = (i / BT_X) % BT_Y, lz = i / (BT_X * BT_Y);
      const int gz = bz * TZ + lz, gy = by * BT_Y + ly, gx = bx * BT_X + lx;
      if (gz < D && gy < H && gx < W) {
        const float* p = s_y + (lz * BT_Y + ly) * BT_X + lx;
        float a = 0.f;
        if (DEPTH) { for (int k = 0; k <= 2 * R; ++k) a = fmaf(p[k * BT_Y * BT_X], kw.w[k], a); }
        else a = p[0];
        y[c * V + ((int64_t)gz * H + gy) * W + gx] = a;
        mn = fminf(mn, a); mx = fmaxf(mx, a); ssum += a; ssq += (double)a * a;
      }
    }
    __syncthreads();
  }
  if (sout) {
    // every block owns tiles of increasing channel index; with one row, or the last channel of several, commit what is left
    if (stats_rows > 1) { if (cur_c >= 0) block_stats_commit(mn, mx, ssum, ssq, sout + cur_c); }
    else block_stats_commit(mn, mx, ssum, ssq, sout);
  }
}

// ---- the batched 2-D training branch (training/dataset/dim2/dataset_acdc.py:128-142) ------------------------------
// gaussian_noise -> brightness_additive -> gamma(retain_stats) -> random_scale_rotate_translate_2d -> crop_2d(random)
// for B ragged slices in three launches.  y1 = x + std*n + beta is recomputed from x wherever it is needed (the noise
// is counter-based), so no intermediate slice exists in HBM:
//   aug2d_stats1: per-chunk {min, max, sum, sumsq} of y1;
//   aug2d_stats2: per-chunk {sum, sumsq} of y2 = ((y1 - min)/rng)^gamma * rng + min;
//   aug2d_gather: for each pixel of the h x w crop, the bilinear / nearest taps of the affine grid over the whole slice,
//                 each tap's y3 = (y2 - mean2)/std2 * std1 + mean1 recomputed from x.
// Every slice is cut into chunks of AUG2D_CHUNK elements; each block reduces its chunk in a fixed tree and writes one
// partial, and the next launch folds a slice's partials in a fixed order (no atomics), so a plan always gives the same
// bits, whatever the batch it runs in.
constexpr int AUG2D_THREADS = 256, AUG2D_GROUPS = 4, AUG2D_CHUNK = AUG2D_THREADS * AUG2D_GROUPS * 4;
static_assert(sizeof(b200seg_aug2d_row) == 88, "b200seg_aug2d_row layout is part of the ABI");

struct Aug2dPart { double s, q; float mn, mx; float pad[2]; };

__device__ __forceinline__ int aug2d_chunks(int64_t n) { return (int)((n + AUG2D_CHUNK - 1) / AUG2D_CHUNK); }

// y1 with the exact expressions of OP_NOISE (mean 0) and OP_ADD, so the chain of per-function calls gives the same bits
__device__ __forceinline__ float aug2d_y1(float x, float z, float std, float beta) {
  const float zero = 0.f;
  float v = x + z * std + zero;
  return v + beta;
}

// the normal of element idx (component idx % 4 of Philox block idx / 4), as aug_pointwise_kernel<OP_NOISE> draws it
__device__ __forceinline__ float aug2d_normal(uint64_t key, int64_t idx) {
  float z[4];
  philox_normal4(key, (uint64_t)(idx >> 2), z);
  const int k = (int)(idx & 3);
  return k == 0 ? z[0] : (k == 1 ? z[1] : (k == 2 ? z[2] : z[3]));
}

// block-wide fixed-order merge (256 threads) -> thread 0 holds the result
__device__ __forceinline__ void aug2d_block_merge(float& mn, float& mx, double& s, double& q) {
  __shared__ float s_mn[AUG2D_THREADS / 32], s_mx[AUG2D_THREADS / 32];
  __shared__ double s_s[AUG2D_THREADS / 32], s_q[AUG2D_THREADS / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  s = warp_sum_d(s); q = warp_sum_d(q);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_mn[w] = mn; s_mx[w] = mx; s_s[w] = s; s_q[w] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < AUG2D_THREADS / 32; ++i) { mn = fminf(mn, s_mn[i]); mx = fmaxf(mx, s_mx[i]); s += s_s[i]; q += s_q[i]; }
  }
}

// fold a slice's partials in a fixed order (warp 0: lane-strided serial sums, then a fixed xor tree); every lane of
// warp 0 ends with the same values
__device__ __forceinline__ void aug2d_fold(const Aug2dPart* p, int n, float& mn, float& mx, double& s, double& q) {
  mn = INFINITY; mx = -INFINITY; s = 0.0; q = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) { const Aug2dPart a = p[i]; mn = fminf(mn, a.mn); mx = fmaxf(mx, a.mx); s += a.s; q += a.q; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  s = warp_sum_d(s); q = warp_sum_d(q);
}

// mean and unbiased std as read_stats computes them from the sums
__device__ __forceinline__ void aug2d_moments(double s, double q, double n, double& mean, double& std) {
  mean = s / n;
  const double var = (q - n * mean * mean) / (n > 1.0 ? n - 1.0 : 1.0);
  std = sqrt(var > 0.0 ? var : 0.0);
}

// the per-slice constants of the intensity chain, folded from the partials by warp 0 and broadcast through shared memory
struct Aug2dConsts { float mn1, rng1, mean2, std2, std1, mean1; };

template <bool SECOND>
__device__ __forceinline__ void aug2d_consts(const Aug2dPart* p1, const Aug2dPart* p2, int nch, double n, Aug2dConsts& out) {
  __shared__ Aug2dConsts sc;
  if (threadIdx.x < 32) {
    float mn, mx; double s, q;
    aug2d_fold(p1, nch, mn, mx, s, q);
    double m1, sd1; aug2d_moments(s, q, n, m1, sd1);
    Aug2dConsts c = {mn, mx - mn, 0.f, 0.f, (float)sd1, (float)m1};
    if (SECOND) {
      aug2d_fold(p2, nch, mn, mx, s, q);
      double m2, sd2; aug2d_moments(s, q, n, m2, sd2);
      c.mean2 = (float)m2; c.std2 = (float)sd2;
    }
    if (threadIdx.x == 0) sc = c;
  }
  __syncthreads();
  out = sc;
}

// PASS 1: partials of y1 (and, when the row asks for it, y1 itself); PASS 2: partials of y2
template <int PASS>
__global__ void __launch_bounds__(AUG2D_THREADS) aug2d_stats_kernel(const b200seg_aug2d_row* __restrict__ rows, int max_chunks,
                                                                   Aug2dPart* __restrict__ part1, Aug2dPart* __restrict__ part2) {
  const int b = blockIdx.y, c = blockIdx.x;
  const b200seg_aug2d_row r = rows[b];
  const int64_t n = (int64_t)r.H * r.W;
  const int nch = aug2d_chunks(n);
  if (c >= nch || nch > max_chunks) return;
  Aug2dConsts k = {};
  if (PASS == 2) aug2d_consts<false>(part1 + (int64_t)b * max_chunks, nullptr, nch, (double)n, k);
  const float* x = r.img;
  float* y1out = PASS == 1 ? r.y1 : nullptr;
  const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y1out)) & 15) == 0;
  float mn = INFINITY, mx = -INFINITY; double sm = 0.0, sq = 0.0;
#pragma unroll
  for (int gi = 0; gi < AUG2D_GROUPS; ++gi) {
    const int64_t g = (int64_t)c * (AUG2D_CHUNK / 4) + gi * AUG2D_THREADS + threadIdx.x;
    const int64_t i0 = g * 4;
    if (i0 >= n) break;
    const int cnt = (int)((n - i0) < 4 ? (n - i0) : 4);
    float v[4] = {0.f, 0.f, 0.f, 0.f}, z[4] = {0.f, 0.f, 0.f, 0.f};
    if (vec && cnt == 4) { const float4 f = *reinterpret_cast<const float4*>(x + i0); v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w; }
    else {
#pragma unroll
      for (int e = 0; e < 4; ++e) if (e < cnt) v[e] = x[i0 + e];
    }
    if (r.noise_std != 0.f) philox_normal4(r.noise_key, (uint64_t)g, z);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[e] = aug2d_y1(v[e], z[e], r.noise_std, r.beta);
      if (PASS == 2) v[e] = powf((v[e] - k.mn1) / k.rng1, r.gamma) * k.rng1 + k.mn1;
      if (e < cnt) { mn = fminf(mn, v[e]); mx = fmaxf(mx, v[e]); sm += v[e]; sq += (double)v[e] * v[e]; }
    }
    if (y1out) {
      if (vec && cnt == 4) *reinterpret_cast<float4*>(y1out + i0) = make_float4(v[0], v[1], v[2], v[3]);
      else {
#pragma unroll
        for (int e = 0; e < 4; ++e) if (e < cnt) y1out[i0 + e] = v[e];
      }
    }
  }
  aug2d_block_merge(mn, mx, sm, sq);
  if (threadIdx.x == 0) {
    Aug2dPart o = {sm, sq, mn, mx, {0.f, 0.f}};
    (PASS == 1 ? part1 : part2)[(int64_t)b * max_chunks + c] = o;
  }
}

// y3 of element idx of slice r
__device__ __forceinline__ float aug2d_y3(const b200seg_aug2d_row& r, int64_t idx, const Aug2dConsts& k) {
  const float z = r.noise_std != 0.f ? aug2d_normal(r.noise_key, idx) : 0.f;
  const float y1 = aug2d_y1(r.img[idx], z, r.noise_std, r.beta);
  const float y2 = powf((y1 - k.mn1) / k.rng1, r.gamma) * k.rng1 + k.mn1;
  return (y2 - k.mean2) / k.std2 * k.std1 + k.mean1;
}

// one thread = one pixel of slice blockIdx.y's h x w crop; the affine grid is defined on the whole H x W slice, exactly
// as aug_resample_kernel<AFFINE> computes it for D = 1 with theta [[a, b, 0, tx], [c, d, 0, ty], [0, 0, 1, 0]]
template <typename TL>
__global__ void __launch_bounds__(AUG2D_THREADS) aug2d_gather_kernel(const b200seg_aug2d_row* __restrict__ rows, int max_chunks,
                                                                    const Aug2dPart* __restrict__ part1, const Aug2dPart* __restrict__ part2,
                                                                    int h, int w, float* __restrict__ oimg, int64_t* __restrict__ olab) {
  const int b = blockIdx.y;
  const b200seg_aug2d_row r = rows[b];
  const int64_t n = (int64_t)r.H * r.W;
  const int nch = aug2d_chunks(n);
  if (nch > max_chunks) {           // statistics were never computed for this slice: make that visible, never guess
    for (int64_t i = (int64_t)blockIdx.x * AUG2D_THREADS + threadIdx.x; i < (int64_t)h * w; i += (int64_t)gridDim.x * AUG2D_THREADS) {
      oimg[(int64_t)b * h * w + i] = __int_as_float(0x7fc00000); olab[(int64_t)b * h * w + i] = 0;
    }
    return;
  }
  Aug2dConsts k;
  aug2d_consts<true>(part1 + (int64_t)b * max_chunks, part2 + (int64_t)b * max_chunks, nch, (double)n, k);
  const TL* lab = reinterpret_cast<const TL*>(r.lab);
  const int64_t HW = (int64_t)h * w;
  for (int64_t i = (int64_t)blockIdx.x * AUG2D_THREADS + threadIdx.x; i < HW; i += (int64_t)gridDim.x * AUG2D_THREADS) {
    const int sw = (int)(i % w) + r.crop_x, sh = (int)(i / w) + r.crop_y;
    const float bx = r.W > 1 ? (2.f * sw) / (float)(r.W - 1) - 1.f : 0.f;
    const float by = r.H > 1 ? (2.f * sh) / (float)(r.H - 1) - 1.f : 0.f;
    const float gx = fmaf(bx, r.theta[0], fmaf(by, r.theta[1], fmaf(0.f, 0.f, r.theta[2])));
    const float gy = fmaf(bx, r.theta[3], fmaf(by, r.theta[4], fmaf(0.f, 0.f, r.theta[5])));
    const float ix = (gx + 1.f) * 0.5f * (float)(r.W - 1);
    const float iy = (gy + 1.f) * 0.5f * (float)(r.H - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x_0 = (int)fx, y_0 = (int)fy;
    const float tx = ix - fx, ty = iy - fy;
    const bool vx0 = (unsigned)x_0 < (unsigned)r.W, vx1 = (unsigned)(x_0 + 1) < (unsigned)r.W;
    const bool vy0 = (unsigned)y_0 < (unsigned)r.H, vy1 = (unsigned)(y_0 + 1) < (unsigned)r.H;
    const int64_t base = (int64_t)y_0 * r.W + x_0;
    const float w00 = (1.f - tx) * (1.f - ty), w01 = tx * (1.f - ty), w10 = (1.f - tx) * ty, w11 = tx * ty;
    float v = 0.f;
    if (vy0 && vx0) v += aug2d_y3(r, base, k) * w00;
    if (vy0 && vx1) v += aug2d_y3(r, base + 1, k) * w01;
    if (vy1 && vx0) v += aug2d_y3(r, base + r.W, k) * w10;
    if (vy1 && vx1) v += aug2d_y3(r, base + r.W + 1, k) * w11;
    oimg[(int64_t)b * HW + i] = v;
    // mode='nearest': round half to even, zeros outside
    const int nx = (int)nearbyintf(ix), ny = (int)nearbyintf(iy);
    int64_t l = 0;
    if ((unsigned)nx < (unsigned)r.W && (unsigned)ny < (unsigned)r.H) l = (int64_t)lab[(int64_t)ny * r.W + nx];
    olab[(int64_t)b * HW + i] = l;
  }
}

inline int grid_for(int64_t n, int th) {
  int64_t g = (n + th - 1) / th;
  const int64_t cap = (int64_t)B200SEG_NUM_SMS * 8;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

template <typename TL, typename TLO>
int launch_resample(const float* img, const void* lab, int C, const Geom& g, bool affine, float* oimg, void* olab, StatRow* stats,
                    int stats_rows, cudaStream_t st) {
  const int grid = grid_for((int64_t)g.Do * g.Ho * g.Wo, 256);
  if (affine) aug_resample_kernel<TL, TLO, true><<<grid, 256, 0, st>>>(img, (const TL*)lab, C, g, oimg, (TLO*)olab, stats, stats_rows);
  else aug_resample_kernel<TL, TLO, false><<<grid, 256, 0, st>>>(img, (const TL*)lab, C, g, oimg, (TLO*)olab, stats, stats_rows);
  B200_CHECK_LAUNCH("aug_resample_kernel");
  return B200SEG_OK;
}

}  // namespace

extern "C" int b200seg_aug_resample(const float* img, const void* lab, int lab_bytes, int C, const int* src_dims, const int* sub_origin,
                                    const int* sub_dims, const float* theta, const int* out_origin, const int* out_dims, int flip_mask,
                                    float* out_img, void* out_lab, int out_lab_bytes, void* stats, int stats_rows, void* stream) {
  if (!src_dims || !sub_origin || !sub_dims || !out_origin || !out_dims || C < 0) return B200SEG_EINVAL;
  if ((lab == nullptr) != (out_lab == nullptr) || (img == nullptr) != (out_img == nullptr)) return B200SEG_EINVAL;
  if ((C == 0) != (img == nullptr) || (!img && !lab)) return B200SEG_EINVAL;          // C == 0: label map only
  if (!img && stats) return B200SEG_EINVAL;
  if (stats && stats_rows != 1 && stats_rows != C) return B200SEG_EINVAL;
  Geom g;
  g.D = src_dims[0]; g.H = src_dims[1]; g.W = src_dims[2];
  g.z0 = sub_origin[0]; g.y0 = sub_origin[1]; g.x0 = sub_origin[2];
  g.Ds = sub_dims[0]; g.Hs = sub_dims[1]; g.Ws = sub_dims[2];
  g.oz = out_origin[0]; g.oy = out_origin[1]; g.ox = out_origin[2];
  g.Do = out_dims[0]; g.Ho = out_dims[1]; g.Wo = out_dims[2];
  g.flip = flip_mask & 7;
  if (g.D <= 0 || g.H <= 0 || g.W <= 0 || g.Ds <= 0 || g.Hs <= 0 || g.Ws <= 0 || g.Do <= 0 || g.Ho <= 0 || g.Wo <= 0) return B200SEG_EINVAL;
  // the sub-volume lies inside the source, the output patch inside the sub-volume (Python slicing would clamp silently;
  // the reference's callers never rely on that, and an out-of-range gather must not happen)
  if (g.z0 < 0 || g.y0 < 0 || g.x0 < 0 || g.z0 + g.Ds > g.D || g.y0 + g.Hs > g.H || g.x0 + g.Ws > g.W) return B200SEG_EINVAL;
  if (g.oz < 0 || g.oy < 0 || g.ox < 0 || g.oz + g.Do > g.Ds || g.oy + g.Ho > g.Hs || g.ox + g.Wo > g.Ws) return B200SEG_EINVAL;
  for (int i = 0; i < 12; ++i) g.th[i] = theta ? theta[i] : 0.f;
  const bool affine = theta != nullptr;
  cudaStream_t st = as_stream(stream);
  StatRow* sr = (StatRow*)stats;
  if (!lab) return launch_resample<uint8_t, uint8_t>(img, nullptr, C, g, affine, out_img, nullptr, sr, stats_rows, st);
  if (lab_bytes == 1 && out_lab_bytes == 1) return launch_resample<uint8_t, uint8_t>(img, lab, C, g, affine, out_img, out_lab, sr, stats_rows, st);
  if (lab_bytes == 1 && out_lab_bytes == 8) return launch_resample<uint8_t, int64_t>(img, lab, C, g, affine, out_img, out_lab, sr, stats_rows, st);
  if (lab_bytes == 8 && out_lab_bytes == 8) return launch_resample<int64_t, int64_t>(img, lab, C, g, affine, out_img, out_lab, sr, stats_rows, st);
  if (lab_bytes == 8 && out_lab_bytes == 1) return launch_resample<int64_t, uint8_t>(img, lab, C, g, affine, out_img, out_lab, sr, stats_rows, st);
  return B200SEG_EINVAL;
}

extern "C" int b200seg_aug_pointwise(const float* x, float* y, int rows, int64_t n, int op, const float* a, const float* b,
                                     const void* stats_in, const void* stats_in2, void* stats_out, uint64_t seed, void* stream) {
  if (!x || rows <= 0 || n <= 0) return B200SEG_EINVAL;
  if (rows > 8) return B200SEG_EUNSUPPORTED;
  if (op != OP_STATS && !y) return B200SEG_EINVAL;
  if ((op == OP_GAMMA_POW || op == OP_RENORM || op == OP_CONTRAST) && !stats_in) return B200SEG_EINVAL;
  if (op == OP_RENORM && !stats_in2) return B200SEG_EINVAL;
  if (op == OP_STATS && !stats_out) return B200SEG_EINVAL;
  PwParams p;
  for (int i = 0; i < 8; ++i) { p.a[i] = (a && i < rows) ? a[i] : 0.f; p.b[i] = (b && i < rows) ? b[i] : 0.f; }
  cudaStream_t st = as_stream(stream);
  const int grid = grid_for((n + 3) / 4, 256);
  const StatRow* si = (const StatRow*)stats_in; const StatRow* si2 = (const StatRow*)stats_in2; StatRow* so = (StatRow*)stats_out;
#define PW(OP) aug_pointwise_kernel<OP><<<grid, 256, 0, st>>>(x, y, rows, n, p, si, si2, so, seed)
  switch (op) {
    case OP_MUL: PW(OP_MUL); break;
    case OP_ADD: PW(OP_ADD); break;
    case OP_GAMMA_POW: PW(OP_GAMMA_POW); break;
    case OP_RENORM: PW(OP_RENORM); break;
    case OP_CONTRAST: PW(OP_CONTRAST); break;
    case OP_NOISE: PW(OP_NOISE); break;
    case OP_STATS: PW(OP_STATS); break;
    default: return B200SEG_EINVAL;
  }
#undef PW
  B200_CHECK_LAUNCH("aug_pointwise_kernel");
  return B200SEG_OK;
}

namespace {
int launch_blur(bool depth, const float* x, float* y, int C, int D, int H, int W, const float* weights, int ksize,
                void* stats_out, int stats_rows, void* stream) {
  if (!x || !y || !weights || C <= 0 || D <= 0 || H <= 0 || W <= 0 || x == y) return B200SEG_EINVAL;
  if (ksize < 1 || (ksize & 1) == 0) return B200SEG_EINVAL;
  const int R = ksize / 2;
  if (R > BR_MAX) return B200SEG_EUNSUPPORTED;       // sigma_range [0.5, 1.0] gives k = 5 or 7 (augmentation.py:50-51)
  if (stats_out && stats_rows != 1 && stats_rows != C) return B200SEG_EINVAL;
  BlurW kw;
  for (int i = 0; i < 2 * BR_MAX + 1; ++i) kw.w[i] = i < ksize ? weights[i] : 0.f;
  const int TZ = depth ? BT_Z : 1, RZ = depth ? R : 0;
  const int EZ = TZ + 2 * RZ, EY = BT_Y + 2 * R, EX = BT_X + 2 * R;
  const size_t smem = sizeof(float) * ((size_t)EZ * EY * EX + (size_t)EZ * EY * BT_X + (size_t)EZ * BT_Y * BT_X);
  static bool attr_set = false;
  if (!attr_set) {
    B200_CUDA(cudaFuncSetAttribute(aug_blur_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr_set = true;
  }
  const int64_t tiles = (int64_t)C * ((D + TZ - 1) / TZ) * ((H + BT_Y - 1) / BT_Y) * ((W + BT_X - 1) / BT_X);
  const int64_t cap = (int64_t)B200SEG_NUM_SMS * 3;
  const int grid = (int)(tiles < cap ? tiles : cap);
  if (depth) aug_blur_kernel<true><<<grid, 256, smem, as_stream(stream)>>>(x, y, C, D, H, W, R, kw, (StatRow*)stats_out, stats_rows);
  else aug_blur_kernel<false><<<grid, 256, smem, as_stream(stream)>>>(x, y, C, D, H, W, R, kw, (StatRow*)stats_out, stats_rows);
  B200_CHECK_LAUNCH("aug_blur_kernel");
  return B200SEG_OK;
}
}  // namespace

extern "C" int b200seg_aug_gaussian_blur(const float* x, float* y, int C, int D, int H, int W, const float* weights, int ksize,
                                         void* stats_out, int stats_rows, void* stream) {
  return launch_blur(true, x, y, C, D, H, W, weights, ksize, stats_out, stats_rows, stream);
}

extern "C" int b200seg_aug_gaussian_blur2d(const float* x, float* y, int C, int H, int W, const float* weights, int ksize,
                                           void* stats_out, int stats_rows, void* stream) {
  return launch_blur(false, x, y, C, 1, H, W, weights, ksize, stats_out, stats_rows, stream);
}

extern "C" size_t b200seg_aug2d_workspace(int B, int64_t max_elems) {
  if (B <= 0 || max_elems <= 0) return 0;
  return (size_t)2 * B * (size_t)((max_elems + AUG2D_CHUNK - 1) / AUG2D_CHUNK) * sizeof(Aug2dPart);
}

extern "C" int b200seg_aug2d_train(const void* rows, int B, int64_t max_elems, int lab_bytes, int h, int w, float* out_img,
                                   int64_t* out_lab, void* workspace, size_t workspace_bytes, void* stream) {
  if (!rows || !out_img || !out_lab || !workspace || B <= 0 || max_elems <= 0 || h <= 0 || w <= 0) return B200SEG_EINVAL;
  if (B > 65535) return B200SEG_EUNSUPPORTED;
  if (lab_bytes != 1 && lab_bytes != 8) return B200SEG_EINVAL;
  if (workspace_bytes < b200seg_aug2d_workspace(B, max_elems)) return B200SEG_EINVAL;
  const int max_chunks = (int)((max_elems + AUG2D_CHUNK - 1) / AUG2D_CHUNK);
  const b200seg_aug2d_row* r = (const b200seg_aug2d_row*)rows;
  Aug2dPart* p1 = (Aug2dPart*)workspace;
  Aug2dPart* p2 = p1 + (size_t)B * max_chunks;
  cudaStream_t st = as_stream(stream);
  const dim3 gs(max_chunks, B);
  aug2d_stats_kernel<1><<<gs, AUG2D_THREADS, 0, st>>>(r, max_chunks, p1, p2);
  B200_CHECK_LAUNCH("aug2d_stats_kernel<1>");
  aug2d_stats_kernel<2><<<gs, AUG2D_THREADS, 0, st>>>(r, max_chunks, p1, p2);
  B200_CHECK_LAUNCH("aug2d_stats_kernel<2>");
  const int64_t per = ((int64_t)h * w + AUG2D_THREADS - 1) / AUG2D_THREADS;
  const dim3 gg((unsigned)(per < 65535 ? per : 65535), B);
  if (lab_bytes == 1) aug2d_gather_kernel<uint8_t><<<gg, AUG2D_THREADS, 0, st>>>(r, max_chunks, p1, p2, h, w, out_img, out_lab);
  else aug2d_gather_kernel<int64_t><<<gg, AUG2D_THREADS, 0, st>>>(r, max_chunks, p1, p2, h, w, out_img, out_lab);
  B200_CHECK_LAUNCH("aug2d_gather_kernel");
  return B200SEG_OK;
}
