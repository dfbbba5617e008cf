// surface.cu — validation surface distances, metric/utils.py:8-28 (calculate_distance): per foreground class the
// area-weighted average surface distance (ASD) and the percentile Hausdorff distance (HD) between the
// surfaces of label_true == c and label_pred == c, with the semantics of metric/metrics.py:265-720.
//
// Per class, on its bounding box of (gt | pred) extended by one voxel at the high end (DESIGN.md §3.10):
//   codes     2x2x2 neighbour code of both masks (ENCODE_NEIGHBOURHOOD_3D_KERNEL weights), border = code not 0 / 255
//   edt_rows  nearest border along axis 2 (two scans per row)
//   edt_cols  lower envelope of parabolas along axis 1 (Felzenszwalb-Huttenlocher), carrying the feature column
//   edt_depth same along axis 0; at every border position of the other mask the distance to the nearest border is
//             sqrt(((Δ0·s0)² + (Δ1·s1)²) + (Δ2·s2)²) from the integer feature offset — scipy's formula — and
//             (distance, area rank) is appended to that direction's segment
//   two stable segmented radix sorts (area rank, then distance) = numpy's sort by (distance, area)
//   reduce    Σa and Σd·a as numpy's pairwise sums, the percentile index as numpy's sequential cumsum + searchsorted
// fp64 throughout, every product / sum rounded on its own (no FMA contraction) so that values are numpy's.
#include <cub/device/device_segmented_radix_sort.cuh>

#include <climits>
#include <vector>

#include "common.cuh"

namespace {

constexpr int kMaxClasses = 256;
constexpr int kReduceThreads = 256;
constexpr int kTile = 4096;            // doubles staged per step of the sequential cumsum

struct Box {
  int lo[3];
  int n[3];                            // extent incl. the padding voxel
};

__device__ __forceinline__ bool is_border(uint8_t code) { return code != 0 && code != 255; }

// fl(fl(x*s)^2)
__device__ __forceinline__ double sq_scaled(int x, double s) {
  const double t = __dmul_rn((double)x, s);
  return __dmul_rn(t, t);
}

// boxes [C][6] = {min0, min1, min2, max0, max1, max2}; rank[code] orders the codes by area (ties share a rank);
// outputs start as the values of a class absent from both maps (ASD nan, HD inf)
__global__ void surface_init_kernel(int* boxes, int C, const double* __restrict__ table, uint8_t* rank,
                                    double* area_by_rank, double* asd, double* hd) {
  const int t = threadIdx.x;
  for (int i = t; i < C * 6; i += blockDim.x) boxes[i] = (i % 6) < 3 ? INT_MAX : -1;
  for (int i = t; i < C - 1; i += blockDim.x) { asd[i] = __longlong_as_double(0x7ff8000000000000LL); hd[i] = INFINITY; }
  if (t < 256) {
    const double a = table[t];
    int r = 0;
    for (int j = 0; j < 256; ++j) r += table[j] < a;
    rank[t] = (uint8_t)r;
    area_by_rank[r] = a;               // tied codes write the same value
  }
}

template <typename TP, typename TT>
__global__ void __launch_bounds__(256) surface_bbox_kernel(const TP* __restrict__ pred, const TT* __restrict__ gt,
                                                           int D, int H, int W, int C, int* boxes) {
  __shared__ int sb[kMaxClasses * 6];
  for (int i = threadIdx.x; i < C * 6; i += blockDim.x) sb[i] = (i % 6) < 3 ? INT_MAX : -1;
  __syncthreads();
  const int64_t N = (int64_t)D * H * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l0 = (int64_t)pred[i], l1 = (int64_t)gt[i];
    if ((l0 < 1 || l0 >= C) && (l1 < 1 || l1 >= C)) continue;
    const int w = (int)(i % W), h = (int)((i / W) % H), d = (int)(i / ((int64_t)W * H));
    for (int k = 0; k < 2; ++k) {
      const int64_t l = k ? l1 : l0;
      if (l < 1 || l >= C || (k && l1 == l0)) continue;
      int* b = sb + l * 6;
      atomicMin(b + 0, d); atomicMin(b + 1, h); atomicMin(b + 2, w);
      atomicMax(b + 3, d); atomicMax(b + 4, h); atomicMax(b + 5, w);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C * 6; i += blockDim.x) {
    if (sb[i - i % 6 + 3] < 0) continue;
    if ((i % 6) < 3) atomicMin(boxes + i, sb[i]); else atomicMax(boxes + i, sb[i]);
  }
}

// codes[0][V] of gt == c, codes[1][V] of pred == c over the extended box; resets both segments
template <typename TP, typename TT>
__global__ void __launch_bounds__(256) surface_codes_kernel(const TP* __restrict__ pred, const TT* __restrict__ gt,
                                                            int D, int H, int W, int c, Box b, uint8_t* __restrict__ codes,
                                                            int* seg_begin, int* seg_end) {
  const int64_t V = (int64_t)b.n[0] * b.n[1] * b.n[2];
  if (blockIdx.x == 0 && threadIdx.x == 0) { seg_begin[0] = 0; seg_begin[1] = (int)V; seg_end[0] = 0; seg_end[1] = (int)V; }
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < V; q += (int64_t)gridDim.x * blockDim.x) {
    const int q2 = (int)(q % b.n[2]), q1 = (int)((q / b.n[2]) % b.n[1]), q0 = (int)(q / ((int64_t)b.n[2] * b.n[1]));
    const int p0 = b.lo[0] + q0, p1 = b.lo[1] + q1, p2 = b.lo[2] + q2;
    unsigned cg = 0, cp = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int x0 = p0 - 1 + (k >> 2), x1 = p1 - 1 + ((k >> 1) & 1), x2 = p2 - 1 + (k & 1);
      if (x0 < 0 || x1 < 0 || x2 < 0 || x0 >= D || x1 >= H || x2 >= W) continue;
      const int64_t i = ((int64_t)x0 * H + x1) * W + x2;
      const unsigned bit = 1u << (7 - k);
      if ((int64_t)gt[i] == c) cg |= bit;
      if ((int64_t)pred[i] == c) cp |= bit;
    }
    codes[q] = (uint8_t)cg;
    codes[V + q] = (uint8_t)cp;
  }
}

// f1[job][q0][q1][q2] = column of the nearest border in the row (q0, q1), -1 when the row has none
__global__ void __launch_bounds__(128) surface_edt_rows_kernel(const uint8_t* __restrict__ codes, int* __restrict__ f1, Box b) {
  const int64_t rows = 2LL * b.n[0] * b.n[1];
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int n = b.n[2];
  const uint8_t* cr = codes + r * n;
  int* fr = f1 + r * n;
  int last = -1;
  for (int x = 0; x < n; ++x) { if (is_border(cr[x])) last = x; fr[x] = last; }
  int next = -1;
  for (int x = n - 1; x >= 0; --x) {
    if (is_border(cr[x])) next = x;
    if (next >= 0 && (fr[x] < 0 || next - x < x - fr[x])) fr[x] = next;
  }
}

// Lower envelope of the parabolas ((x - q)·s)² + g(q) over the sites q of one line of n positions
// (Felzenszwalb & Huttenlocher 2012); v / z: per-line scratch, element k at [k * stride].
// site(q, &g) says whether q is a site and gives g; out(x, q) receives the winning site (or -1).
template <typename Site, typename Out>
__device__ __forceinline__ void lower_envelope(int n, double s, Site site, Out out, int* v, double* z, int64_t stride) {
  const double s2 = __dmul_rn(s, s);
  int k = -1;
  for (int q = 0; q < n; ++q) {
    double gq;
    if (!site(q, gq)) continue;
    const double fq = __dadd_rn(gq, sq_scaled(q, s));
    double x = -INFINITY;
    while (k >= 0) {
      const int r = v[k * stride];
      double gr;
      site(r, gr);
      x = __ddiv_rn(__dsub_rn(fq, __dadd_rn(gr, sq_scaled(r, s))), __dmul_rn(2.0 * (q - r), s2));
      if (x <= z[k * stride]) --k; else break;
    }
    ++k;
    v[k * stride] = q;
    z[k * stride] = k == 0 ? -INFINITY : x;
  }
  if (k < 0) { for (int x = 0; x < n; ++x) out(x, -1); return; }
  int j = 0;
  for (int x = 0; x < n; ++x) {
    while (j < k && z[(j + 1) * stride] < (double)x) ++j;
    out(x, v[j * stride]);
  }
}

// f2[job][q0][x][q2] = row of the nearest border in the slice q0 (its column is f1 at that row), -1 if none
__global__ void __launch_bounds__(128) surface_edt_cols_kernel(const int* __restrict__ f1, int* __restrict__ f2, int n0, int n1,
                                                               int n2, double s1, double s2, int* vs, double* zs) {
  const int64_t lines = 2LL * n0 * n2;
  const int64_t line = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= lines) return;
  const int q2 = (int)(line % n2);
  const int64_t base = (line / n2) * n1 * n2 + q2;              // (job, q0) slice, column q2
  lower_envelope(n1, s1,
      [=](int q, double& g) { const int c = f1[base + (int64_t)q * n2]; if (c < 0) return false; g = sq_scaled(c - q2, s2); return true; },
      [=](int x, int q) { f2[base + (int64_t)x * n2] = q; }, vs + line, zs + line, lines);
}

// Along axis 0: for each border position of the OTHER mask, the distance to this job's nearest border, appended
// with the other mask's area rank to segment (1 - job): segment 0 holds gt -> pred, segment 1 pred -> gt.
__global__ void __launch_bounds__(128) surface_edt_depth_kernel(const uint8_t* __restrict__ codes, const int* __restrict__ f1,
                                                                const int* __restrict__ f2, Box b, double s0, double s1, double s2,
                                                                const uint8_t* __restrict__ rank, int* vs, double* zs,
                                                                int* seg_end, double* dist, uint8_t* arank) {
  const int n0 = b.n[0], n1 = b.n[1], n2 = b.n[2];
  const int64_t plane = (int64_t)n1 * n2, V = plane * n0;
  const int64_t lines = 2 * plane;
  const int64_t line = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (line >= lines) return;
  const int job = (int)(line / plane);
  const int64_t hw = line % plane;
  const int q1 = (int)(hw / n2), q2 = (int)(hw % n2);
  const int* g1 = f1 + job * V;
  const int* g2 = f2 + job * V;
  const uint8_t* other = codes + (1 - job) * V;
  lower_envelope(n0, s0,
      [=](int q, double& g) {
        const int h = g2[q * plane + hw];
        if (h < 0) return false;
        const int w = g1[q * plane + (int64_t)h * n2 + q2];
        g = __dadd_rn(sq_scaled(h - q1, s1), sq_scaled(w - q2, s2));
        return true;
      },
      [=](int x, int q) {
        const uint8_t code = other[x * plane + hw];
        if (!is_border(code)) return;
        double d = INFINITY;           // this mask has no border at all
        if (q >= 0) {
          const int h = g2[q * plane + hw];
          const int w = g1[q * plane + (int64_t)h * n2 + q2];
          d = __dsqrt_rn(__dadd_rn(__dadd_rn(sq_scaled(q - x, s0), sq_scaled(h - q1, s1)), sq_scaled(w - q2, s2)));
        }
        const int slot = atomicAdd(seg_end + (1 - job), 1);
        dist[slot] = d;
        arank[slot] = rank[code];
      },
      vs + line, zs + line, lines);
}

// numpy's pairwise_sum leaf (n <= 128): 8 interleaved partial sums, or a plain loop below 8 elements
template <bool kProduct>
__device__ double pairwise_leaf(const double* __restrict__ d, const uint8_t* __restrict__ r, const double* __restrict__ area, int64_t n) {
  auto x = [&](int64_t i) { const double a = area[r[i]]; return kProduct ? __dmul_rn(d[i], a) : a; };
  if (n < 8) {
    double res = 0.0;
    for (int64_t i = 0; i < n; ++i) res = __dadd_rn(res, x(i));
    return res;
  }
  double p[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) p[k] = x(k);
  int64_t i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] = __dadd_rn(p[k], x(i + k));
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(p[0], p[1]), __dadd_rn(p[2], p[3])), __dadd_rn(__dadd_rn(p[4], p[5]), __dadd_rn(p[6], p[7])));
  for (; i < n; ++i) res = __dadd_rn(res, x(i));
  return res;
}

// numpy's recursive split of pairwise_sum: n > 128 -> (n2, n - n2) with n2 = n/2 rounded down to a multiple of 8
__device__ __forceinline__ int64_t pairwise_split(int64_t n) { const int64_t h = n / 2; return h - h % 8; }

// Per segment (one block each): ASD_dir = Σd·a / Σa and HD_dir = d[min(searchsorted(cumsum(a) / Σa, p), n - 1)]
// over the (distance, area)-sorted surfels, with numpy's summation orders; leaves: scratch of n/8 + 1 doubles x 2.
__global__ void __launch_bounds__(kReduceThreads) surface_reduce_kernel(const double* __restrict__ dist, const uint8_t* __restrict__ arank,
                                                                        const double* __restrict__ area_by_rank, const int* __restrict__ seg_begin,
                                                                        const int* __restrict__ seg_end, double p, int64_t* leaf_pos,
                                                                        double* leaf_sum, int64_t leaf_cap, double* dir) {
  __shared__ double tile[kTile];
  __shared__ int64_t s_nleaf, s_idx;
  __shared__ double s_sum, s_prod;
  const int seg = blockIdx.x;
  const int64_t b = seg_begin[seg], n = seg_end[seg] - b;
  const double* d = dist + b;
  const uint8_t* r = arank + b;
  int64_t* lpos = leaf_pos + seg * leaf_cap;
  double* lsum = leaf_sum + seg * 2 * leaf_cap;
  if (n == 0) {                        // the reference's empty list: 0/0 and np.Inf
    if (threadIdx.x == 0) { dir[seg] = __longlong_as_double(0x7ff8000000000000LL); dir[2 + seg] = INFINITY; }
    return;
  }
  // 1. the leaves of numpy's pairwise recursion, in order (thread 0), then their sums (all threads)
  if (threadIdx.x == 0) {
    int64_t stack[64];
    int top = 0, nl = 0;
    int64_t start = 0;
    stack[top++] = n;
    while (top > 0) {
      const int64_t m = stack[--top];
      if (m <= 128) { lpos[nl++] = start; start += m; continue; }
      const int64_t h = pairwise_split(m);
      stack[top++] = m - h;
      stack[top++] = h;
    }
    lpos[nl] = n;
    s_nleaf = nl;
  }
  __syncthreads();
  const int64_t nl = s_nleaf;
  for (int64_t j = threadIdx.x; j < nl; j += blockDim.x) {
    const int64_t s = lpos[j], m = lpos[j + 1] - s;
    lsum[2 * j] = pairwise_leaf<false>(d + s, r + s, area_by_rank, m);
    lsum[2 * j + 1] = pairwise_leaf<true>(d + s, r + s, area_by_rank, m);
  }
  __syncthreads();
  // 2. combine the leaves in the recursion's order (post-order walk with an explicit stack)
  if (threadIdx.x == 0) {
    int64_t size[64];
    double left[64][2];
    int stage[64];
    int top = 0;
    int64_t next = 0;
    double val[2] = {0.0, 0.0};
    size[0] = n; stage[0] = 0; top = 1;
    bool have = false;
    while (top > 0) {
      const int t = top - 1;
      if (!have) {
        if (size[t] <= 128) { val[0] = lsum[2 * next]; val[1] = lsum[2 * next + 1]; ++next; have = true; --top; continue; }
        const int64_t h = pairwise_split(size[t]);
        if (stage[t] == 0) { size[top] = h; stage[top] = 0; ++top; continue; }
        size[top] = size[t] - h; stage[top] = 0; ++top; continue;
      }
      // a child finished with val
      if (stage[t] == 0) { left[t][0] = val[0]; left[t][1] = val[1]; stage[t] = 1; have = false; continue; }
      val[0] = __dadd_rn(left[t][0], val[0]);
      val[1] = __dadd_rn(left[t][1], val[1]);
      --top;
    }
    s_sum = val[0];
    s_prod = val[1];
  }
  __syncthreads();
  const double T = s_sum;
  // 3. the first k with fl(S_k / T) >= p, S_k the sequential cumsum; fl(S / T) is monotone in S, so compare S_k with
  //    the least double S* satisfying it
  int64_t idx = 0;
  if (p > 0.0) {
    double sstar = 0.0;
    if (threadIdx.x == 0) {
      sstar = __dmul_rn(p, T);
      while (sstar > 0.0 && __ddiv_rn(sstar, T) >= p) sstar = __longlong_as_double(__double_as_longlong(sstar) - 1);   // next double down (sstar > 0)
      while (__ddiv_rn(sstar, T) < p && sstar < INFINITY) sstar = __longlong_as_double(__double_as_longlong(sstar) + 1);
      s_idx = -1;
    }
    double S = 0.0;
    __syncthreads();
    for (int64_t t0 = 0; t0 < n; t0 += kTile) {
      const int m = (int)min((int64_t)kTile, n - t0);
      for (int i = threadIdx.x; i < m; i += blockDim.x) tile[i] = area_by_rank[r[t0 + i]];
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int i = 0; i < m; ++i) {
          S = __dadd_rn(S, tile[i]);
          if (S >= sstar) { s_idx = t0 + i; break; }
        }
      }
      __syncthreads();
      if (s_idx >= 0) break;
    }
    idx = s_idx < 0 ? n - 1 : s_idx;
  }
  if (threadIdx.x == 0) {
    dir[seg] = __ddiv_rn(s_prod, T);
    dir[2 + seg] = d[idx];
  }
}

__global__ void surface_combine_kernel(const double* __restrict__ dir, double* asd, double* hd) {
  asd[0] = __dmul_rn(__dadd_rn(dir[0], dir[1]), 0.5);
  hd[0] = dir[3] > dir[2] ? dir[3] : dir[2];      // Python's max(gt_to_pred, pred_to_gt)
}

inline int grid_for(int64_t n, int th) {
  int64_t g = (n + th - 1) / th;
  const int64_t cap = (int64_t)B200SEG_NUM_SMS * 16;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Workspace carve-up for an extended box of at most V voxels (both jobs / segments).
struct Layout {
  size_t boxes, rank, area, seg, dir, codes, f1, f2, vs, zs, dist, dist_alt, rk, rk_alt, lpos, lsum, cub, total;
  size_t cub_bytes;
};

size_t cub_bytes_for(int64_t V) {
  size_t a = 0, b = 0;
  cub::DoubleBuffer<uint8_t> k8(nullptr, nullptr);
  cub::DoubleBuffer<double> vd(nullptr, nullptr);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, a, k8, vd, (int)(2 * V), 2, (const int*)nullptr, (const int*)nullptr, 0, 8);
  cub::DeviceSegmentedRadixSort::SortPairs(nullptr, b, vd, k8, (int)(2 * V), 2, (const int*)nullptr, (const int*)nullptr);
  return a > b ? a : b;
}

Layout layout(int64_t V, int C, size_t cub_bytes) {
  Layout L{};
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o = align256(o + bytes); return at; };
  const int64_t leaf_cap = V / 8 + 2;                  // leaves per segment: >= 8 elements each except possibly one
  L.boxes = take(sizeof(int) * 6 * (size_t)C);
  L.rank = take(256);
  L.area = take(sizeof(double) * 256);
  L.seg = take(sizeof(int) * 4);
  L.dir = take(sizeof(double) * 4);
  L.codes = take(2 * (size_t)V);
  L.f1 = take(sizeof(int) * 2 * (size_t)V);
  L.f2 = take(sizeof(int) * 2 * (size_t)V);
  L.vs = take(sizeof(int) * 3 * (size_t)V);            // lines x (n + 1) <= 1.5 x 2V
  L.zs = take(sizeof(double) * 3 * (size_t)V);
  L.dist = take(sizeof(double) * 2 * (size_t)V);
  L.dist_alt = take(sizeof(double) * 2 * (size_t)V);
  L.rk = take(2 * (size_t)V);
  L.rk_alt = take(2 * (size_t)V);
  L.lpos = take(sizeof(int64_t) * 2 * (size_t)leaf_cap);
  L.lsum = take(sizeof(double) * 4 * (size_t)leaf_cap);
  L.cub_bytes = cub_bytes;
  L.cub = take(cub_bytes);
  L.total = o;
  return L;
}

template <typename TP, typename TT>
int run(const void* pred_v, const void* gt_v, int D, int H, int W, int C, double s0, double s1, double s2, double percent,
        const double* table, double* asd, double* hd, uint8_t* ws, size_t ws_bytes, cudaStream_t st) {
  const TP* pred = (const TP*)pred_v;
  const TT* gt = (const TT*)gt_v;
  const int64_t Vmax = (int64_t)(D + 1) * (H + 1) * (W + 1);
  const Layout L = layout(Vmax, C, cub_bytes_for(Vmax));
  if (ws_bytes < L.total) return B200SEG_EINVAL;
  int* boxes = (int*)(ws + L.boxes);
  uint8_t* rank = ws + L.rank;
  double* area = (double*)(ws + L.area);
  int* seg_begin = (int*)(ws + L.seg);
  int* seg_end = seg_begin + 2;
  double* dir = (double*)(ws + L.dir);
  uint8_t* codes = ws + L.codes;
  int* f1 = (int*)(ws + L.f1);
  int* f2 = (int*)(ws + L.f2);
  int* vs = (int*)(ws + L.vs);
  double* zs = (double*)(ws + L.zs);

  surface_init_kernel<<<1, 256, 0, st>>>(boxes, C, table, rank, area, asd, hd);
  B200_CHECK_LAUNCH("surface_init_kernel");
  surface_bbox_kernel<TP, TT><<<grid_for((int64_t)D * H * W, 256), 256, 0, st>>>(pred, gt, D, H, W, C, boxes);
  B200_CHECK_LAUNCH("surface_bbox_kernel");
  std::vector<int> hb(6 * (size_t)C);
  B200_CUDA(cudaMemcpyAsync(hb.data(), boxes, sizeof(int) * hb.size(), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));               // the one planning copy: the per-class boxes

  for (int c = 1; c < C; ++c) {
    const int* bx = hb.data() + 6 * c;
    if (bx[3] < 0) continue;                          // absent from both maps: stays nan / inf
    Box b;
    for (int a = 0; a < 3; ++a) { b.lo[a] = bx[a]; b.n[a] = bx[3 + a] - bx[a] + 2; }
    const int64_t V = (int64_t)b.n[0] * b.n[1] * b.n[2];
    surface_codes_kernel<TP, TT><<<grid_for(V, 256), 256, 0, st>>>(pred, gt, D, H, W, c, b, codes, seg_begin, seg_end);
    B200_CHECK_LAUNCH("surface_codes_kernel");
    const int64_t rows = 2LL * b.n[0] * b.n[1], cols = 2LL * b.n[0] * b.n[2], depth = 2LL * b.n[1] * b.n[2];
    surface_edt_rows_kernel<<<ceil_div(rows, 128), 128, 0, st>>>(codes, f1, b);
    B200_CHECK_LAUNCH("surface_edt_rows_kernel");
    surface_edt_cols_kernel<<<ceil_div(cols, 128), 128, 0, st>>>(f1, f2, b.n[0], b.n[1], b.n[2], s1, s2, vs, zs);
    B200_CHECK_LAUNCH("surface_edt_cols_kernel");
    cub::DoubleBuffer<double> kd((double*)(ws + L.dist), (double*)(ws + L.dist_alt));
    cub::DoubleBuffer<uint8_t> kr(ws + L.rk, ws + L.rk_alt);
    surface_edt_depth_kernel<<<ceil_div(depth, 128), 128, 0, st>>>(codes, f1, f2, b, s0, s1, s2, rank, vs, zs, seg_end,
                                                                  kd.Current(), kr.Current());
    B200_CHECK_LAUNCH("surface_edt_depth_kernel");
    // (distance, area) order: stable sort by area rank, then stable sort by distance
    size_t cub_bytes = L.cub_bytes;
    B200_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kr, kd, (int)(2 * V), 2, seg_begin, seg_end, 0, 8, st));
    cub_bytes = L.cub_bytes;
    B200_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(ws + L.cub, cub_bytes, kd, kr, (int)(2 * V), 2, seg_begin, seg_end, 0, 64, st));
    surface_reduce_kernel<<<2, kReduceThreads, 0, st>>>(kd.Current(), kr.Current(), area, seg_begin, seg_end, percent / 100.0,
                                                        (int64_t*)(ws + L.lpos), (double*)(ws + L.lsum), Vmax / 8 + 2, dir);
    B200_CHECK_LAUNCH("surface_reduce_kernel");
    surface_combine_kernel<<<1, 1, 0, st>>>(dir, asd + (c - 1), hd + (c - 1));
    B200_CHECK_LAUNCH("surface_combine_kernel");
  }
  return B200SEG_OK;
}

}  // namespace

extern "C" size_t b200seg_surface_distance_workspace(int D, int H, int W, int C) {
  if (D <= 0 || H <= 0 || W <= 0 || C <= 0 || C > kMaxClasses) return 0;
  const int64_t V = (int64_t)(D + 1) * (H + 1) * (W + 1);
  if (2 * V > INT_MAX) return 0;
  return layout(V, C, cub_bytes_for(V)).total;
}

extern "C" int b200seg_surface_distance(const void* pred, int pred_bytes, const void* gt, int gt_bytes, int D, int H, int W, int C,
                                        double s0, double s1, double s2, double percent, const double* table, double* asd,
                                        double* hd, void* workspace, size_t workspace_bytes, void* stream) {
  if (!pred || !gt || !table || !asd || !hd || !workspace || D <= 0 || H <= 0 || W <= 0 || C < 2) return B200SEG_EINVAL;
  if (!(s0 > 0.0) || !(s1 > 0.0) || !(s2 > 0.0) || !(percent == percent)) return B200SEG_EINVAL;
  if (C > kMaxClasses || 2 * (int64_t)(D + 1) * (H + 1) * (W + 1) > INT_MAX) return B200SEG_EUNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  uint8_t* ws = (uint8_t*)workspace;
#define SD(TP, TT) run<TP, TT>(pred, gt, D, H, W, C, s0, s1, s2, percent, table, asd, hd, ws, workspace_bytes, st)
  if (pred_bytes == 1 && gt_bytes == 1) return SD(uint8_t, uint8_t);
  if (pred_bytes == 1 && gt_bytes == 8) return SD(uint8_t, int64_t);
  if (pred_bytes == 8 && gt_bytes == 1) return SD(int64_t, uint8_t);
  if (pred_bytes == 8 && gt_bytes == 8) return SD(int64_t, int64_t);
#undef SD
  return B200SEG_EINVAL;
}
