// wgrad_tc.cu — conv3d weight gradient as wgmma GEMMs (sm_90a), fp16 operands, fp32 accumulation in registers.
// Replaces cuDNN wgrad behind autograd of nn.Conv3d (train_ddp.py:193/208); what it writes is the fp32
// parameter-gradient tensor DDP all-reduces.
//
//   dW[co][ci][tap] = sum_voxels dy[v][co] * a[v + tap][ci],      a = act(IN(x))
//
// GEMM view per CTA: D_tap[128 co][N ci] += dy^T[128 co x 128 voxels] * a_tap[128 voxels x N ci] for a GROUP of
// in-plane taps of one depth offset zd; K = voxels, accumulated over every voxel tile the CTA owns, so the
// accumulators stay in registers for the CTA's whole life (G*N <= 192 columns) and there is ONE epilogue.
//   * both operands are staged as [channel/8][voxel][8 ch] — the same image conv_tc.cu uses — and read by
//     wgmma as MN-major no-swizzle matrices (core matrix = 8 voxels x 8 channels, 128 B):
//     A = dy tile (16x8 voxels), B = halo tile of `a` ((16+kh-1)x(8+kw-1) voxels); a tap is a shifted
//     B descriptor, exactly like the forward kernel.
//   * `a` is never materialised by a separate pass: the loader warps stage RAW x with cp.async (up to three stages in
//     flight) and apply InstanceNorm-normalise + ReLU in place in shared memory once a stage has landed (zero-filled
//     padding voxels stay zero), exactly like conv_tc.cu's forward loader.
//   * only the REAL output channels of the M tile are staged (Cout = 32 stages 4 of the 8 planes a warpgroup reads); the
//     rows computed from whatever follows are never read back.
//   * split-K over voxel tiles fills the machine: grid = jobs x S.  With S > 1 every CTA stores its partial D tiles
//     into its own slice of a caller-provided buffer and a second kernel adds the S slices into dW in split order, so
//     dW is the same bit for bit on every run.
// Warp roles (512 threads, 1 CTA/SM): warps 0-7 = two MMA warpgroups (output channels 64g .. 64g+63 of the M tile)
// that also run the epilogue, warps 8-15 loaders.
#include "common.cuh"
#include "conv_args.h"
#include "tc_common.cuh"
#include "wgmma.cuh"
#include <string.h>

namespace {

using namespace tc;

constexpr int TH = 16, TW = 8;
constexpr int kConsumerWGs = 2;
constexpr int kLoadWarp0 = 8;
constexpr int kLoadThreads = 256;           // all loader warps cooperate on every stage
constexpr int kThreads = 16 * 32;   // 512
constexpr int MT = 128;                    // output-channel tile (GEMM M)
constexpr int kMaxCols = 192;              // accumulator columns per job (taps x Cin tile): 96 fp32 registers per thread
// Registers per thread after the role dispatch, inside the CTA's pool of 512 x 128: the consumer warpgroups hold up to
// 96 accumulators plus descriptors and epilogue addresses, the loaders' cp.async + transform loop needs far fewer.
constexpr int kRegsLaunch = 128, kRegsConsumer = 152, kRegsLoad = 104;
static_assert(2 * 128 * kRegsConsumer + 2 * 128 * kRegsLoad <= kThreads * kRegsLaunch, "register split exceeds the CTA pool");

struct WgParams {
  const __half* x; int x_ld, x_coff;       // raw input; normalised + activated on the fly when x_stats / act
  const double* x_stats; float eps; int act;
  const __half* dy; int dy_ld, dy_coff;
  float* dw;
  float* part;                             // S > 1: split-K partials [S][Cout][Cin][taps], summed in split order
  int B, D, H, W, Cin, Cout, kd, kh, kw;
  int NTC, ci_tiles, co_tiles, ngroups, gbase, grem, S;
  int HALO_H, HALO_W, nvox_h, a_plane, dy_plane, a_bytes, dy_bytes, stage_bytes, NS, prefetch;
  int tiles_h, tiles_w, nvt;
  int smem_bar_off, smem_norm_off;
};

// barrier block layout (uint64 each): full[NS] (stage staged and transformed) empty[NS] (stage read by both consumers)
struct Bars {
  uint32_t bar0; const WgParams& p;
  __device__ __forceinline__ uint32_t full(int i) const { return bar0 + 8u * (uint32_t)i; }
  __device__ __forceinline__ uint32_t empty(int i) const { return bar0 + 8u * (uint32_t)(p.NS + i); }
};

struct Job { int co_tile, ci_tile, zd, grp, tap0, ntaps, s; };
__device__ __forceinline__ Job decode_job(const WgParams& p, int bid) {
  Job j;
  j.s = bid % p.S; int q = bid / p.S;
  j.grp = q % p.ngroups; q /= p.ngroups;
  j.zd = q % p.kd; q /= p.kd;
  j.ci_tile = q % p.ci_tiles; j.co_tile = q / p.ci_tiles;
  if (j.grp < p.grem) { j.ntaps = p.gbase + 1; j.tap0 = j.grp * (p.gbase + 1); }
  else { j.ntaps = p.gbase; j.tap0 = p.grem * (p.gbase + 1) + (j.grp - p.grem) * p.gbase; }
  return j;
}

// voxel tiles this CTA owns: vt = s, s+S, ... ; those whose input depth slice lies outside the volume are skipped.
// The walk is a mixed-radix counter (w-tile, h-tile, d, b) advanced by the digits of S: no divisions per tile.
struct VtWalk {
  int s0, s1, s2, s3;               // digits of the stride S
  int r0, r1, r2;                   // radices: tiles_w, tiles_h, D
  __device__ __forceinline__ void init(const WgParams& p) {
    r0 = p.tiles_w; r1 = p.tiles_h; r2 = p.D;
    int x = p.S;
    s0 = x % r0; x /= r0; s1 = x % r1; x /= r1; s2 = x % r2; s3 = x / r2;
  }
};
struct VtCursor {
  int vt, wi, hi, d, b, din;
  __device__ __forceinline__ void step(const VtWalk& k, const WgParams& p) {
    vt += p.S;
    int c;
    wi += k.s0; c = wi >= k.r0; if (c) wi -= k.r0;
    hi += k.s1 + c; c = hi >= k.r1; if (c) hi -= k.r1;
    d += k.s2 + c; c = d >= k.r2; if (c) d -= k.r2;
    b += k.s3 + c;
  }
  __device__ __forceinline__ void seek(const VtWalk& k, const WgParams& p, int zoff) {      // first valid tile at or after vt
    while (vt < p.nvt) { din = d + zoff; if ((unsigned)din < (unsigned)p.D) return; step(k, p); }
  }
  __device__ __forceinline__ void init(const VtWalk& k, const WgParams& p, int s, int zoff) {
    vt = s;
    int t = s;
    wi = t % k.r0; t /= k.r0; hi = t % k.r1; t /= k.r1; d = t % k.r2; b = t / k.r2;
    seek(k, p, zoff);
  }
  __device__ __forceinline__ bool valid(const WgParams& p) const { return vt < p.nvt; }
  __device__ __forceinline__ void next(const VtWalk& k, const WgParams& p, int zoff) { step(k, p); seek(k, p, zoff); }
  __device__ __forceinline__ int h0() const { return hi * TH; }
  __device__ __forceinline__ int w0() const { return wi * TW; }
};

template <int P>
__device__ __forceinline__ void wg_loader(const WgParams& p, const Job& job, uint8_t* smem, const float2* s_norm, const Bars& bars) {
  const int lt = threadIdx.x - kLoadWarp0 * 32;
  const int ph = p.kh / 2, pw = p.kw / 2, zoff = job.zd - p.kd / 2;
  const int co0 = job.co_tile * MT;
  const int co_real = min(MT, p.Cout - co0);
  const int ci0 = job.ci_tile * p.NTC;
  // dy tile: thread owns plane (lt % cpv) and walks voxels v0, v0+vstep, ...
  const int cpv_d = co_real / 8;
  const int vstep_d = kLoadThreads / cpv_d;
  const bool act_d = lt < vstep_d * cpv_d;
  const int c8_d = lt % cpv_d, v0_d = lt / cpv_d;
  const int cpv_a = p.NTC / 8;
  const int vstep_a = kLoadThreads / cpv_a;
  const bool act_a = lt < vstep_a * cpv_a;
  const int c8_a = lt % cpv_a, v0_a = lt / cpv_a;
  const int sh_a = vstep_a / p.HALO_W, sw_a = vstep_a % p.HALO_W;
  const int hh0 = v0_a / p.HALO_W, ww0 = v0_a % p.HALO_W;
  const bool xform = (p.x_stats != nullptr) || (p.act != 0);
  const bool relu = p.act == B200SEG_ACT_RELU;
  const float slope = act_slope(p.act);
  VtWalk vw; vw.init(p);
  VtCursor ci, cd;
  ci.init(vw, p, job.s, zoff); cd.init(vw, p, job.s, zoff);
  Ring ri, rd; ri.init(p.NS); rd.init(p.NS);

  auto issue = [&]() {
    mbar_wait(bars.empty(ri.idx), ri.phase ^ 1);
    const uint32_t sdy = smem_u32(smem + ri.idx * p.stage_bytes);
    const uint32_t sa = sdy + (uint32_t)p.dy_bytes;
    if (act_d) {
      const __half* src = p.dy + ((int64_t)(ci.b * p.D + ci.d) * p.H * p.W) * p.dy_ld + p.dy_coff + co0 + c8_d * 8;
      const uint32_t dst = sdy + (uint32_t)(c8_d * p.dy_plane);
#pragma unroll 4
      for (int v = v0_d; v < TH * TW; v += vstep_d) {
        const int h = ci.h0() + (v >> 3), w = ci.w0() + (v & 7);
        const bool ok = h < p.H && w < p.W;
        cp_async16(dst + (uint32_t)v * 16u, ok ? (const void*)(src + ((int64_t)h * p.W + w) * p.dy_ld) : (const void*)p.dy, ok ? 16u : 0u);
      }
    }
    if (act_a) {
      const __half* src = p.x + ((int64_t)(ci.b * p.D + ci.din) * p.H * p.W) * p.x_ld + p.x_coff + ci0 + c8_a * 8;
      const uint32_t dst = sa + (uint32_t)(c8_a * p.a_plane);
      int hh = hh0, ww = ww0;
#pragma unroll 4
      for (int v = v0_a; v < p.nvox_h; v += vstep_a) {
        const int h = ci.h0() - ph + hh, w = ci.w0() - pw + ww;
        const bool ok = (unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W;
        cp_async16(dst + (uint32_t)v * 16u, ok ? (const void*)(src + ((int64_t)h * p.W + w) * p.x_ld) : (const void*)p.x, ok ? 16u : 0u);
        hh += sh_a; ww += sw_a;
        if (ww >= p.HALO_W) { ww -= p.HALO_W; ++hh; }
      }
    }
    ri.advance(); ci.next(vw, p, zoff);
  };

#pragma unroll
  for (int i = 0; i < P; ++i) { if (ci.valid(p)) issue(); cp_async_commit(); }
  while (cd.valid(p)) {
    cp_async_wait<P - 1>();
    if (xform && act_a) {
      uint8_t* sp = smem + rd.idx * p.stage_bytes + p.dy_bytes + c8_a * p.a_plane;
      float sc[8], sf[8];                          // x*sc + sf == (x - mean) * rstd
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 mr = s_norm[cd.b * p.NTC + c8_a * 8 + j];
        sc[j] = mr.y; sf[j] = -mr.x * mr.y;
      }
      int hh = hh0, ww = ww0;
#pragma unroll 2
      for (int v = v0_a; v < p.nvox_h; v += vstep_a) {
        const int h = cd.h0() - ph + hh, w = cd.w0() - pw + ww;
        if ((unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W) {      // padding voxels stay zero
          uint4* chunk = reinterpret_cast<uint4*>(sp + v * 16);
          *chunk = relu ? norm_act8<true>(*chunk, sc, sf, slope) : norm_act8<false>(*chunk, sc, sf, slope);
        }
        hh += sh_a; ww += sw_a;
        if (ww >= p.HALO_W) { ww -= p.HALO_W; ++hh; }
      }
    }
    fence_proxy_async();
    mbar_arrive(bars.full(rd.idx));
    rd.advance(); cd.next(vw, p, zoff);
    if (ci.valid(p)) issue();
    cp_async_commit();
  }
  cp_async_wait<0>();
}

// most taps one job's group can have at Cin tile NTC (fill_params: G = min(kMaxCols / NTC, kh * kw), kh, kw <= 3)
__host__ __device__ constexpr int max_taps(int ntc) { return kMaxCols / ntc < 9 ? kMaxCols / ntc : 9; }

// Calls f(std::integral_constant<int, G>{}) for the job's run-time tap count n, G0 <= n <= GMAX.
template <int G, int GMAX, class F>
__device__ __forceinline__ void dispatch_taps(int n, F&& f) {
  if constexpr (G < GMAX) {
    if (n != G) { dispatch_taps<G + 1, GMAX>(n, f); return; }
  }
  f(std::integral_constant<int, G>{});
}

// ---- a consumer warpgroup whose 64 rows of the M tile hold no real output channel (Cout <= 64): it issues no MMA and
// holds no accumulator, it only hands each stage back once it has been staged.
__device__ __forceinline__ void idle_consumer_role(const WgParams& p, const Job& job, int tid, const Bars& bars) {
  const int zoff = job.zd - p.kd / 2;
  VtWalk vw; vw.init(p);
  VtCursor c; c.init(vw, p, job.s, zoff);
  Ring r; r.init(p.NS);
  for (; c.valid(p); c.next(vw, p, zoff)) {
    mbar_wait(bars.full(r.idx), r.phase);
    if (tid == 0) mbar_arrive(bars.empty(r.idx));
    r.advance();
  }
}

// ---- MMA warpgroup g: output channels co0 + 64g .. +63 of the M tile, the NTAPS taps of the job's group.  Per voxel
// tile one wgmma group (NTAPS x 8 instructions m64 x NTC x 16) is committed; the stage the group before it read is then
// handed back.  After the last tile the accumulators are added into dW (thread: rows 16w + l/4 (+8), column pairs
// 8j + 2(l%4)).  NTAPS is a template argument and the group has no branch: a run-time tap count made ptxas retire every
// group before the next one could issue (C7517), which undid the one-group-in-flight pipelining.
template <int NTC, int NTAPS>
__device__ __forceinline__ void consumer_role(const WgParams& p, const Job& job, int wg, int tid, uint8_t* smem, const Bars& bars) {
  const int zoff = job.zd - p.kd / 2;
  const int co0 = job.co_tile * MT, co_real = min(MT, p.Cout - co0), ci0 = job.ci_tile * NTC;
  // dy^T as the A operand: MN-major (lbo = next 8 voxels, sbo = next channel plane); x halo tile as the B operand:
  // MN-major (lbo = next halo row of voxels, sbo = next channel plane), a tap = start shifted by whole voxel slots
  const uint64_t dy_tmpl = make_desc(0, 128u, (uint32_t)p.dy_plane);
  const uint64_t a_tmpl = make_desc(0, (uint32_t)p.HALO_W * 16u, (uint32_t)p.a_plane);
  const uint32_t dy_kstep = 16u;                                       // 16 voxels = 256 B
  const uint32_t a_kstep = 2u * (uint32_t)p.HALO_W;                    // two halo rows of voxels per K=16 step
  const uint32_t stage16 = (uint32_t)p.stage_bytes >> 4, dy16 = (uint32_t)p.dy_bytes >> 4;
  const uint32_t smem16 = smem_u32(smem) >> 4;
  const uint32_t dy_wg16 = (uint32_t)(wg * 8 * p.dy_plane) >> 4;
  // start of each tap's B operand in the staged halo tile, in 16-byte voxel slots: taps run along w, then wrap to the
  // next halo row
  uint32_t tap_off[NTAPS];
#pragma unroll
  for (int g = 0; g < NTAPS; ++g) {
    const int t = job.tap0 + g;
    tap_off[g] = (uint32_t)((t / p.kw) * p.HALO_W + t % p.kw);
  }
  float acc[NTAPS][NTC / 2];
  VtWalk vw; vw.init(p);
  VtCursor c; c.init(vw, p, job.s, zoff);
  const bool any = c.valid(p);
  Ring r; r.init(p.NS);
  int pend = -1;
  uint32_t accumulate = 0;
  for (; c.valid(p); c.next(vw, p, zoff)) {
    mbar_wait(bars.full(r.idx), r.phase);
    const uint64_t da0 = dy_tmpl + (uint64_t)(smem16 + (uint32_t)r.idx * stage16 + dy_wg16);
    const uint64_t db0 = a_tmpl + (uint64_t)(smem16 + (uint32_t)r.idx * stage16 + dy16);
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) wgmma_fence_operands(acc[g]);
    wgmma_fence();
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) {
      uint64_t db = db0 + (uint64_t)tap_off[g];
      // opaque per stage: otherwise ptxas hoists all NTAPS x 8 loop-invariant B offsets into registers and spills
      asm volatile("" : "+l"(db));
#pragma unroll
      for (int j = 0; j < (TH * TW) / 16; ++j)
        Wgmma<NTC, 1, 1>::mma(acc[g], da0 + (uint64_t)((uint32_t)j * dy_kstep), db + (uint64_t)((uint32_t)j * a_kstep),
                              accumulate | (uint32_t)(j > 0));
    }
    wgmma_commit();
    wgmma_wait<1>();                               // the group before this one has retired: its stage is free
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) wgmma_fence_operands(acc[g]);
    if (pend >= 0 && tid == 0) mbar_arrive(bars.empty(pend));
    pend = r.idx;
    accumulate = 1;
    r.advance();
  }
  wgmma_wait<0>();
#pragma unroll
  for (int g = 0; g < NTAPS; ++g) wgmma_fence_operands(acc[g]);
  if (pend >= 0 && tid == 0) mbar_arrive(bars.empty(pend));
  // S == 1: this CTA is the only contributor of its dW elements, one add each.  S > 1: the partial tile goes to its own
  // slice of the split-K buffer (zeros when the CTA owned no voxel tile) and add_slices sums the slices in order,
  // so dW does not depend on which CTA finishes first.
  const int warp = tid >> 5, lane = tid & 31;
  const int taps = p.kd * p.kh * p.kw, tap_base = job.zd * p.kh * p.kw + job.tap0;
  const int64_t nw = (int64_t)p.Cout * p.Cin * taps;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wg * 64 + 16 * warp + (lane >> 2) + 8 * i;
    if (row >= co_real) continue;
    const int64_t off = ((int64_t)(co0 + row) * p.Cin + ci0) * taps + tap_base;
    float* drow = p.S > 1 ? p.part + (int64_t)job.s * nw + off : p.dw + off;
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) {
#pragma unroll
      for (int j = 0; j < NTC / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        const float v0 = any ? acc[g][4 * j + 2 * i] : 0.f, v1 = any ? acc[g][4 * j + 2 * i + 1] : 0.f;
        if (p.S > 1) { drow[(int64_t)col * taps + g] = v0; drow[(int64_t)(col + 1) * taps + g] = v1; }
        else if (any) { drow[(int64_t)col * taps + g] += v0; drow[(int64_t)(col + 1) * taps + g] += v1; }
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1)
wgrad_tc_kernel(const __grid_constant__ WgParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int ci0 = decode_job(p, blockIdx.x).ci_tile * p.NTC;

  const Bars bars{smem_u32(smem + p.smem_bar_off), p};
  float2* s_norm = reinterpret_cast<float2*>(smem + p.smem_norm_off);     // [B][NTC] {mean, rstd} of this job's channels

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.NS; ++i) { mbar_init(bars.full(i), kLoadThreads); mbar_init(bars.empty(i), kConsumerWGs); }
    fence_barrier_init();
  }
  {
    const double n = (double)p.D * p.H * p.W;
    for (int i = threadIdx.x; i < p.B * p.NTC; i += kThreads) {
      float m = 0.f, r = 1.f;
      const int b = i / p.NTC, c = i % p.NTC;
      if (p.x_stats) stats_to_mean_rstd(p.x_stats + ((int64_t)b * p.Cin + ci0 + c) * 2, n, p.eps, m, r);
      s_norm[i] = make_float2(m, r);
    }
  }
  __syncthreads();

  if (warp >= kLoadWarp0) {
    // =========================== LOADERS ===========================
    setmaxnreg_dec<kRegsLoad>();
    // each role decodes the job after its setmaxnreg: a value live across the register split is spilled
    const Job job = decode_job(p, blockIdx.x);
    if (p.prefetch >= 3) wg_loader<3>(p, job, smem, s_norm, bars);
    else if (p.prefetch == 2) wg_loader<2>(p, job, smem, s_norm, bars);
    else wg_loader<1>(p, job, smem, s_norm, bars);
  } else {
    // =========================== MMA + EPILOGUE ===========================
    setmaxnreg_inc<kRegsConsumer>();
    const Job job = decode_job(p, blockIdx.x);
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    // warpgroup-uniform, and uniform over the CTA's one job: whether this half of the M tile holds real channels,
    // and how many taps the job's group has
    if (wg * 64 >= min(MT, p.Cout - job.co_tile * MT)) {
      idle_consumer_role(p, job, tid, bars);
    } else {
      dispatch_n(p.NTC, [&](auto ntc) {
        constexpr int NTC = decltype(ntc)::value;
        dispatch_taps<1, max_taps(NTC)>(job.ntaps, [&](auto nt) { consumer_role<NTC, decltype(nt)::value>(p, job, wg, tid, smem, bars); });
      });
    }
  }
}

// Cin tile (GEMM N): 64 when Cin is a multiple of 128 (three taps share one staged tile, twice the jobs of a 128-wide
// tile), else the whole Cin up to 128, else the largest of 128 / 96 / 64 / 48 / 32 / 16 dividing it.
int pick_ntc(int Cin) {
  if (Cin % 16) return 0;
  if (Cin % 128 == 0) return 64;
  if (Cin <= 128) return Cin;
  const int c[] = {128, 96, 64, 48, 32, 16};
  for (int v : c) if (Cin % v == 0) return v;
  return 0;
}

bool fill_params(const WgradArgs& a, WgParams& p) {
  memset(&p, 0, sizeof(p));
  p.B = a.B; p.D = a.D; p.H = a.H; p.W = a.W; p.Cin = a.Cin; p.Cout = a.Cout; p.kd = a.kd; p.kh = a.kh; p.kw = a.kw;
  p.NTC = pick_ntc(a.Cin);
  if (!p.NTC || a.Cout % 8) return false;
  if (a.B * p.NTC > 2048) return false;
  p.ci_tiles = a.Cin / p.NTC;
  p.co_tiles = (a.Cout + MT - 1) / MT;
  const int taps_hw = a.kh * a.kw;
  int G = kMaxCols / p.NTC; if (G > taps_hw) G = taps_hw;
  p.ngroups = (taps_hw + G - 1) / G;
  p.gbase = taps_hw / p.ngroups; p.grem = taps_hw % p.ngroups;
  p.HALO_H = TH + a.kh - 1; p.HALO_W = TW + a.kw - 1; p.nvox_h = p.HALO_H * p.HALO_W;
  int slots = p.nvox_h; if ((slots & 1) == 0) ++slots;
  p.a_plane = slots * 16;
  p.dy_plane = (TH * TW + 1) * 16;
  p.a_bytes = (p.NTC / 8) * p.a_plane; p.a_bytes = (p.a_bytes + 127) / 128 * 128;
  // only the real output-channel planes of the widest M tile are staged; the descriptors' 8-plane footprint beyond
  // them falls on the `a` tile / the next stage / the tail slack (allocated below), whose values feed rows never read
  const int co_max = a.Cout < MT ? a.Cout : MT;
  p.dy_bytes = (co_max / 8) * p.dy_plane; p.dy_bytes = (p.dy_bytes + 127) / 128 * 128;
  p.stage_bytes = p.a_bytes + p.dy_bytes;
  const int norm_bytes = a.B * p.NTC * 8;
  const int budget = 227 * 1024 - 2048 - 16 * p.dy_plane - norm_bytes;
  p.NS = budget / p.stage_bytes; if (p.NS > 6) p.NS = 6;
  if (p.NS < 2) return false;
  p.prefetch = p.NS - 1 < 3 ? p.NS - 1 : 3;
  p.tiles_h = (a.H + TH - 1) / TH; p.tiles_w = (a.W + TW - 1) / TW;
  const int64_t nvt = (int64_t)a.B * a.D * p.tiles_h * p.tiles_w;
  if (nvt > 0x7fffffff) return false;
  p.nvt = (int)nvt;
  const int64_t jobs = (int64_t)p.co_tiles * p.ci_tiles * a.kd * p.ngroups;
  int S = (int)(B200SEG_NUM_SMS / jobs); if (S < 1) S = 1;
  if (S > p.nvt) S = p.nvt;
  p.S = S;
  int off = p.NS * p.stage_bytes + 16 * p.dy_plane;       // + slack for the 16-plane descriptor footprint
  off = (off + 15) / 16 * 16;
  p.smem_bar_off = off; off += 2 * p.NS * 8;
  off = (off + 15) / 16 * 16;
  p.smem_norm_off = off;
  return true;
}

}  // namespace

bool conv3d_wgrad_tc_supported(const WgradArgs& a, int dtype) {
  if (dtype != B200SEG_F16) return false;
  if (a.kd > 3 || a.kh > 3 || a.kw > 3) return false;
  if ((a.x_ld % 8) || (a.x_coff % 8) || (a.dy_ld % 8) || (a.dy_coff % 8)) return false;
  if ((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.dy)) & 15) return false;
  if (a.dbias) return false;
  WgParams p;
  return fill_params(a, p);
}

// split-K partial buffer: S slices of dW (none when one CTA covers every voxel tile of its job)
size_t conv3d_wgrad_tc_workspace(const WgradArgs& a) {
  WgParams p;
  if (!fill_params(a, p) || p.S == 1) return 0;
  return (size_t)p.S * a.Cout * a.Cin * a.kd * a.kh * a.kw * sizeof(float);
}

// dw must be zero-initialised (or hold a gradient to accumulate into): the result is ADDED to it.
int conv3d_wgrad_tc(const WgradArgs& a, int dtype, void* workspace, size_t ws_bytes, cudaStream_t st) {
  if (!conv3d_wgrad_tc_supported(a, dtype)) return B200SEG_EUNSUPPORTED;
  const size_t need = conv3d_wgrad_tc_workspace(a);
  if (need && (!workspace || ws_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15))) return B200SEG_EINVAL;
  WgParams p;
  fill_params(a, p);
  p.x = reinterpret_cast<const __half*>(a.x); p.x_ld = a.x_ld; p.x_coff = a.x_coff;
  p.x_stats = a.x_stats; p.eps = a.eps; p.act = a.act;
  p.dy = reinterpret_cast<const __half*>(a.dy); p.dy_ld = a.dy_ld; p.dy_coff = a.dy_coff;
  p.dw = a.dw;
  const int64_t jobs = (int64_t)p.co_tiles * p.ci_tiles * a.kd * p.ngroups;
  const int smem_bytes = p.smem_norm_off + a.B * p.NTC * 8 + 64;
  static thread_local bool attr_set = false;
  if (!attr_set) {
    B200_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  const int grid = (int)(jobs * p.S);
  p.part = reinterpret_cast<float*>(workspace);
  wgrad_tc_kernel<<<grid, kThreads, smem_bytes, st>>>(p);
  B200_CHECK_LAUNCH("wgrad_tc_kernel");
  if (p.S > 1) {
    const int64_t n = (int64_t)a.Cout * a.Cin * a.kd * a.kh * a.kw;
    return add_slices(p.part, n, p.S, a.dw, n, st);
  }
  return B200SEG_OK;
}
