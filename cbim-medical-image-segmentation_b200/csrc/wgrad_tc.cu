// wgrad_tc.cu — conv3d weight gradient as wgmma GEMMs (sm_90a), fp16 operands, fp32 accumulation in registers.
// Replaces cuDNN wgrad behind autograd of nn.Conv3d (train_ddp.py:193/208); what it writes is the fp32
// parameter-gradient tensor DDP all-reduces.
//
//   dW[co][ci][tap] = sum_voxels dy[v][co] * a[v + tap][ci],      a = act(IN(x))
//
// GEMM view per CTA: D_tap[128 co][N ci] += dy^T[128 co x 128 voxels] * a_tap[128 voxels x N ci] for a GROUP of
// in-plane taps of one depth offset zd; K = voxels, accumulated over every voxel tile the CTA owns, so the
// accumulators stay in registers for the CTA's whole life (G*N <= 192 columns) and there is ONE epilogue.
//   * A = dy tile (16x8 voxels), B = halo tile of `a` ((16+kh-1)x(8+kw-1) voxels), both read by wgmma as MN-major
//     matrices; a tap is a B descriptor shifted by whole voxels.  Each operand is staged in one of two images:
//       rows   — one 64- or 128-byte row of 32 / 64 channels per voxel, [group][voxel][32 or 64 ch], stored
//                SWIZZLE_64B / SWIZZLE_128B (tmap.h) and read through swizzled descriptors (SBO = 8 voxel rows).
//                Used for dy when min(Cout, 128) is 32, 64 or 128 (Cout a multiple of 64 above 64) and for x when the
//                Cin tile is 32, 64 or 96 (three 32-channel groups);
//       planes — [channel/8][voxel][8 ch], the image conv_tc.cu uses, read through no-swizzle descriptors (core matrix
//                = 8 voxels x 8 channels, 128 B), for every other width.
//     A row image moves a voxel's channels as one 64- or 128-byte TMA line instead of 4 or 8 16-byte ones.  Either way
//     the MMAs, their operands and their K order are the same, so dW does not depend on the image.
//   * both operands arrive by tensor TMA: per stage one elected thread issues one box for the dy tile and one for the
//     x halo tile (three at a Cin tile of 96; tmap.h; out-of-volume voxels are zero-filled by the TMA unit) onto the
//     stage's LAND barrier, as soon as the consumers hand the slot back, so every free slot of the ring is in flight.
//   * `a` is never materialised by a separate pass: when x needs InstanceNorm-normalise + activation, the other loader
//     warps apply it in place in shared memory once a stage has landed (zero-filled padding voxels stay zero, as in
//     conv_tc.cu's forward loader) and publish FULL; raw x is consumed straight off LAND.
//   * only the REAL output channels of the M tile are staged (Cout = 32 stages 4 of the 8 planes a warpgroup reads); the
//     rows computed from whatever follows are never read back.
//   * the ring holds as many stages as fit (up to 6).  Where fewer than 4 whole 16x8 tiles fit (Cout 128 with a Cin
//     tile of 80 or more), each tile is staged as two 8-row halves and a stage carries K steps 0-3 or 4-7 of the tile:
//     the same MMAs in the same order, so dW is the same bit for bit either way.
//   * split-K over voxel tiles fills the machine: grid = jobs x S.  With S > 1 every CTA stores its partial D tiles
//     into its own slice of a caller-provided buffer and a second kernel adds the S slices into dW in split order, so
//     dW is the same bit for bit on every run.
// Warp roles (512 threads, 1 CTA/SM): warps 0-7 = two MMA warpgroups (output channels 64g .. 64g+63 of the M tile)
// that also run the epilogue, warp 8 = TMA producer (one thread), warps 9-15 = in-place transform.
#include "common.cuh"
#include "conv_args.h"
#include "tc_common.cuh"
#include "tmap.h"
#include "wgmma.cuh"
#include <string.h>

namespace {

using namespace tc;

constexpr int TH = 16, TW = 8;
constexpr int kConsumerWGs = 2;
constexpr int kLoadWarp0 = 8;               // TMA producer warp; the transform warps follow it
constexpr int kXformThreads = 7 * 32;       // warps 9-15 transform every stage together
constexpr int kMaxStages = 6;
constexpr int kThreads = 16 * 32;   // 512
constexpr int MT = 128;                    // output-channel tile (GEMM M)
constexpr int kMaxCols = 192;              // accumulator columns per job (taps x Cin tile): 96 fp32 registers per thread
// Registers per thread after the role dispatch, inside the CTA's pool of 512 x 128: the consumer warpgroups hold up to
// 96 accumulators plus descriptors and epilogue addresses, the loaders' TMA issue and transform loops need far fewer.
constexpr int kRegsLaunch = 128, kRegsConsumer = 152, kRegsLoad = 104;
static_assert(2 * 128 * kRegsConsumer + 2 * 128 * kRegsLoad <= kThreads * kRegsLaunch, "register split exceeds the CTA pool");

struct WgParams {
  alignas(64) CUtensorMap tm_dy;           // dy as {g ch, w, h, group, b*D+d}, box {dy_ch, TW, TS, min(Cout, MT)/dy_ch}
  alignas(64) CUtensorMap tm_x;            // x likewise: planes {8, HALO_W, HALO_H, NTC/8}, rows x_boxes x {x_ch, .., 1}
  uint64_t dy_desc, x_desc;                // wgmma descriptor templates (layout, LBO, SBO) of the two staged images
  const double* x_stats; float eps; int act;   // x is normalised + activated in shared memory when x_stats / act
  const float* x_affine; int per_channel;      // or transformed per channel (conv_args.h); the table is then [NTC]
  float* dw;
  float* part;                             // S > 1: split-K partials [S][Cout][Cin][taps], summed in split order
  int B, D, H, W, Cin, Cout, kd, kh, kw;
  int NTC, ci_tiles, co_tiles, ngroups, gbase, grem, S;
  int TS, halves;                          // voxel rows per stage: TH (whole tiles) or TH/2 (two stages per tile)
  int dy_ch, x_ch, x_boxes;                // channels per staged group (8 = planes, 32 / 64 = rows); x boxes per stage
  int HALO_H, HALO_W, nvox_h, a_plane, dy_plane, a_bytes, dy_bytes, stage_bytes, NS;   // *_plane: group stride
  int tiles_h, tiles_w, nvt;
  int smem_bar_off, smem_norm_off;
};

// barrier block layout (uint64 each): full[NS] (stage transformed) empty[NS] (stage read by both consumers)
// land[NS] (both TMA boxes of the stage have landed)
struct Bars {
  uint32_t bar0; const WgParams& p;
  __device__ __forceinline__ uint32_t full(int i) const { return bar0 + 8u * (uint32_t)i; }
  __device__ __forceinline__ uint32_t empty(int i) const { return bar0 + 8u * (uint32_t)(p.NS + i); }
  __device__ __forceinline__ uint32_t land(int i) const { return bar0 + 8u * (uint32_t)(2 * p.NS + i); }
  // what the consumers wait on: the transformed stage, or the raw stage straight off the TMA
  __device__ __forceinline__ uint32_t ready(int i) const { return (p.x_stats || p.x_affine || p.act) ? full(i) : land(i); }
};

// blockIdx.x read afresh: a job decoded again after the register split, or after the MMA loop, is not merged with an
// earlier decode (whose fields would otherwise stay live, and spill, across it)
__device__ __forceinline__ int cta_id() {
  int v;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(v));
  return v;
}

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
// A cursor visits the stages of the CTA's tiles in order: every half of a tile (p.halves of them) before the next tile.
struct VtCursor {
  int vt, wi, hi, d, b, din, half;
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
    vt = s; half = 0;
    int t = s;
    wi = t % k.r0; t /= k.r0; hi = t % k.r1; t /= k.r1; d = t % k.r2; b = t / k.r2;
    seek(k, p, zoff);
  }
  __device__ __forceinline__ bool valid(const WgParams& p) const { return vt < p.nvt; }
  __device__ __forceinline__ void next(const VtWalk& k, const WgParams& p, int zoff) {
    if (++half < p.halves) return;
    half = 0; step(k, p); seek(k, p, zoff);
  }
  __device__ __forceinline__ int h0(const WgParams& p) const { return hi * TH + half * p.TS; }     // first row of the stage
  __device__ __forceinline__ int w0() const { return wi * TW; }
};

// ---- TMA producer (one thread): per stage, once both consumers have handed the slot back, one box of dy
// {dy_ch, TW, TS, co_max/dy_ch groups} and the x halo as one box {8 ch, HALO_W, HALO_H, NTC/8 planes} (planes) or
// x_boxes boxes {x_ch, HALO_W, HALO_H, 1} a_plane apart (rows), all completing on LAND.  Out-of-volume voxels and output
// channels past Cout are zero-filled and counted in the transaction bytes like any other.
__device__ __forceinline__ void tma_producer(const WgParams& p, const Job& job, uint8_t* smem, const Bars& bars) {
  const int ph = p.kh / 2, pw = p.kw / 2, zoff = job.zd - p.kd / 2;
  const int co_g0 = job.co_tile * (MT / p.dy_ch), ci_g0 = job.ci_tile * (p.NTC / p.x_ch);
  const int x_box_groups = p.NTC / p.x_ch / p.x_boxes;
  const uint32_t stage_tx = (uint32_t)(p.dy_bytes + p.NTC * p.nvox_h * 2);
  VtWalk vw; vw.init(p);
  VtCursor c; c.init(vw, p, job.s, zoff);
  Ring r; r.init(p.NS);
  for (; c.valid(p); c.next(vw, p, zoff)) {
    mbar_wait(bars.empty(r.idx), r.phase ^ 1);
    const uint32_t sdy = smem_u32(smem + r.idx * p.stage_bytes);
    mbar_arrive_expect_tx(bars.land(r.idx), stage_tx);
    tma_load_5d(sdy, &p.tm_dy, bars.land(r.idx), 0, c.w0(), c.h0(p), co_g0, c.b * p.D + c.d);
    for (int i = 0; i < p.x_boxes; ++i)
      tma_load_5d(sdy + (uint32_t)(p.dy_bytes + i * p.a_plane), &p.tm_x, bars.land(r.idx), 0, c.w0() - pw, c.h0(p) - ph,
                  ci_g0 + i * x_box_groups, c.b * p.D + c.din);
    r.advance();
  }
}

// ---- in-place InstanceNorm-normalise + activation of each landed x halo tile (only when x needs it).  Thread owns
// the 8-channel chunk c8 = xt % cpv of the halo voxels v0, v0 + vstep, ...; zero-filled padding voxels stay zero.  In a
// row image the chunk sits in group c8 / (x_ch/8) at position j ^ phase(row), j = c8 % (x_ch/8), where the phase is
// the row's shared-address bits 7.. (the TMA swizzle; the stage and every group start are aligned to its repeat); in
// the plane image it is plane c8 and the phase mask is 0.
__device__ __forceinline__ void transform_role(const WgParams& p, const Job& job, uint8_t* smem, const float2* s_norm, const Bars& bars) {
  const int xt = threadIdx.x - (kLoadWarp0 + 1) * 32;
  const int ph = p.kh / 2, pw = p.kw / 2, zoff = job.zd - p.kd / 2;
  const int cpv = p.NTC / 8;
  const int vstep = kXformThreads / cpv;
  const bool active = xt < vstep * cpv;
  const int c8 = xt % cpv, v0 = xt / cpv;
  const int gch = p.x_ch / 8, row_bytes = p.x_ch * 2;
  const uint32_t chunk = (uint32_t)(c8 % gch), phase_mask = p.x_ch == 64 ? 7u : p.x_ch == 32 ? 3u : 0u;
  const uint32_t group_off = (uint32_t)(p.dy_bytes + (c8 / gch) * p.a_plane);
  const int sh = vstep / p.HALO_W, sw = vstep % p.HALO_W;
  const int hh0 = v0 / p.HALO_W, ww0 = v0 % p.HALO_W;
  const bool relu = p.act == B200SEG_ACT_RELU;
  const float slope = act_slope(p.act);
  VtWalk vw; vw.init(p);
  VtCursor c; c.init(vw, p, job.s, zoff);
  Ring r; r.init(p.NS);
  for (; c.valid(p); c.next(vw, p, zoff)) {
    mbar_wait(bars.land(r.idx), r.phase);
    if (active) {
      uint32_t off = (uint32_t)(r.idx * p.stage_bytes) + group_off + (uint32_t)(v0 * row_bytes);
      float sc[8], sf[8];                          // x*sc + sf: (x - mean) * rstd, or the per-channel transform
      const float2* tb = s_norm + (p.per_channel ? 0 : c.b * p.NTC) + c8 * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 st = tb[j];
        sc[j] = st.x; sf[j] = st.y;
      }
      const int hb = c.h0(p) - ph, wb = c.w0() - pw;
      int hh = hh0, ww = ww0;
#pragma unroll 2
      for (int v = v0; v < p.nvox_h; v += vstep) {
        const int h = hb + hh, w = wb + ww;
        if ((unsigned)h < (unsigned)p.H && (unsigned)w < (unsigned)p.W) {      // padding voxels stay zero
          uint4* q = reinterpret_cast<uint4*>(smem + off + ((chunk ^ ((off >> 7) & phase_mask)) << 4));
          *q = relu ? norm_act8<true>(*q, sc, sf, slope) : norm_act8<false>(*q, sc, sf, slope);
        }
        off += (uint32_t)(vstep * row_bytes);
        hh += sh; ww += sw;
        if (ww >= p.HALO_W) { ww -= p.HALO_W; ++hh; }
      }
    }
    fence_proxy_async();                           // generic-proxy writes -> visible to the tensor core (async proxy)
    mbar_arrive(bars.full(r.idx));
    r.advance();
  }
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
    mbar_wait(bars.ready(r.idx), r.phase);
    if (tid == 0) mbar_arrive(bars.empty(r.idx));
    r.advance();
  }
}

// ---- MMA warpgroup g: output channels co0 + 64g .. +63 of the M tile, the NTAPS taps of the job's group.  Per stage
// one wgmma group (NTAPS x KS instructions m64 x NTC x 16; KS = 8 for a whole 16x8 tile, 4 for a half) is committed;
// the stage the group before it read is then handed back.  Each accumulator sees K steps 0-7 of every tile in order,
// whether a tile arrives in one stage or two.  After the last tile the accumulators are added into dW (thread: rows
// 16w + l/4 (+8), column pairs 8j + 2(l%4)).  NTAPS and KS are template arguments and the group has no branch: a
// run-time tap count made ptxas retire every group before the next one could issue (C7517), which undid the
// one-group-in-flight pipelining.
template <int NTC, int NTAPS, int KS>
__device__ __forceinline__ void consumer_role(const WgParams& p, const Job& job, int wg, int tid, uint8_t* smem, const Bars& bars) {
  const int zoff = job.zd - p.kd / 2;
  // dy^T as the A operand, the x halo tile as the B operand, both MN-major (fill_params builds the descriptor
  // templates); every shift below is a whole number of voxels, one voxel = x_ch / 8 (or dy_ch / 8) 16-byte units
  const uint32_t dy_vox16 = (uint32_t)p.dy_ch >> 3, x_vox16 = (uint32_t)p.x_ch >> 3;
  const uint32_t dy_kstep = 16u * dy_vox16;                            // 16 voxels per K=16 step
  const uint32_t a_kstep = 2u * (uint32_t)p.HALO_W * x_vox16;          // two halo rows of voxels per K=16 step
  const uint32_t stage16 = (uint32_t)p.stage_bytes >> 4, dy16 = (uint32_t)p.dy_bytes >> 4;
  const uint32_t smem16 = smem_u32(smem) >> 4;
  const uint32_t dy_wg16 = (uint32_t)(wg * (64 / p.dy_ch) * p.dy_plane) >> 4;     // the warpgroup's 64 output channels
  // start of each tap's B operand in the staged halo tile: taps run along w, then wrap to the next halo row
  uint32_t tap_off[NTAPS];
#pragma unroll
  for (int g = 0; g < NTAPS; ++g) {
    const int t = job.tap0 + g;
    tap_off[g] = (uint32_t)((t / p.kw) * p.HALO_W + t % p.kw) * x_vox16;
  }
  float acc[NTAPS][NTC / 2];
  VtWalk vw; vw.init(p);
  VtCursor c; c.init(vw, p, job.s, zoff);
  const bool any = c.valid(p);
  Ring r; r.init(p.NS);
  int pend = -1;
  uint32_t accumulate = 0;
  for (; c.valid(p); c.next(vw, p, zoff)) {
    mbar_wait(bars.ready(r.idx), r.phase);
    const uint64_t da0 = p.dy_desc + (uint64_t)(smem16 + (uint32_t)r.idx * stage16 + dy_wg16);
    const uint64_t db0 = p.x_desc + (uint64_t)(smem16 + (uint32_t)r.idx * stage16 + dy16);
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) wgmma_fence_operands(acc[g]);
    wgmma_fence();
#pragma unroll
    for (int g = 0; g < NTAPS; ++g) {
      uint64_t db = db0 + (uint64_t)tap_off[g], da = da0;
#pragma unroll
      for (int j = 0; j < KS; ++j) {
        // opaque per step: otherwise ptxas hoists all NTAPS x KS loop-invariant offsets into registers and spills
        asm volatile("" : "+l"(da), "+l"(db));
        Wgmma<NTC, 1, 1>::mma(acc[g], da, db, accumulate | (uint32_t)(j > 0));
        da += dy_kstep; db += a_kstep;
      }
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
  const Job e = decode_job(p, cta_id());
  const int co0 = e.co_tile * MT, co_real = min(MT, p.Cout - co0), ci0 = e.ci_tile * NTC;
  const int warp = tid >> 5, lane = tid & 31;
  const int taps = p.kd * p.kh * p.kw, tap_base = e.zd * p.kh * p.kw + e.tap0;
  const int64_t nw = (int64_t)p.Cout * p.Cin * taps;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = wg * 64 + 16 * warp + (lane >> 2) + 8 * i;
    if (row >= co_real) continue;
    const int64_t off = ((int64_t)(co0 + row) * p.Cin + ci0) * taps + tap_base;
    float* drow = p.S > 1 ? p.part + (int64_t)e.s * nw + off : p.dw + off;
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
  float2* s_norm = reinterpret_cast<float2*>(smem + p.smem_norm_off);     // [B or 1][NTC] {scale, shift} of this job's channels

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.NS; ++i) {
      mbar_init(bars.full(i), kXformThreads); mbar_init(bars.empty(i), kConsumerWGs); mbar_init(bars.land(i), 1);
    }
    fence_barrier_init();
  }
  {
    const double n = (double)p.D * p.H * p.W;
    for (int i = threadIdx.x; i < (p.per_channel ? 1 : p.B) * p.NTC; i += kThreads) {
      const int b = i / p.NTC, c = i % p.NTC;
      if (p.x_affine) {
        s_norm[i] = make_float2(p.x_affine[2 * (ci0 + c)], p.x_affine[2 * (ci0 + c) + 1]);
      } else {
        float m = 0.f, r = 1.f;
        if (p.x_stats) stats_to_mean_rstd(p.x_stats + ((int64_t)b * p.Cin + ci0 + c) * 2, n, p.eps, m, r);
        s_norm[i] = make_float2(r, -m * r);
      }
    }
  }
  __syncthreads();

  if (warp >= kLoadWarp0) {
    // =========================== LOADERS ===========================
    setmaxnreg_dec<kRegsLoad>();
    // each role decodes the job after its setmaxnreg: a value live across the register split is spilled
    const Job job = decode_job(p, cta_id());
    if (warp == kLoadWarp0) {
      if ((threadIdx.x & 31) == 0) tma_producer(p, job, smem, bars);
    } else if (p.x_stats || p.x_affine || p.act) {
      transform_role(p, job, smem, s_norm, bars);
    }
  } else {
    // =========================== MMA + EPILOGUE ===========================
    setmaxnreg_inc<kRegsConsumer>();
    const Job job = decode_job(p, cta_id());
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    // warpgroup-uniform, and uniform over the CTA's one job: whether this half of the M tile holds real channels,
    // and how many taps the job's group has
    if (wg * 64 >= min(MT, p.Cout - job.co_tile * MT)) {
      idle_consumer_role(p, job, tid, bars);
    } else {
      dispatch_n(p.NTC, [&](auto ntc) {
        constexpr int NTC = decltype(ntc)::value;
        dispatch_taps<1, max_taps(NTC)>(job.ntaps, [&](auto nt) {
          constexpr int NTAPS = decltype(nt)::value;
          if (p.halves == 2) consumer_role<NTC, NTAPS, TH / 4>(p, job, wg, tid, smem, bars);
          else consumer_role<NTC, NTAPS, TH / 2>(p, job, wg, tid, smem, bars);
        });
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
  const int nb = a.per_channel ? 1 : a.B;           // samples with their own row in the transform table
  if (nb * p.NTC > 2048) return false;
  p.ci_tiles = a.Cin / p.NTC;
  p.co_tiles = (a.Cout + MT - 1) / MT;
  const int taps_hw = a.kh * a.kw;
  int G = kMaxCols / p.NTC; if (G > taps_hw) G = taps_hw;
  p.ngroups = (taps_hw + G - 1) / G;
  p.gbase = taps_hw / p.ngroups; p.grem = taps_hw % p.ngroups;
  p.HALO_W = TW + a.kw - 1;
  // only the real output-channel planes of the widest M tile are staged; a consumer warpgroup's A descriptor spans 8
  // whole planes, so with Cout not a multiple of 64 the last live warpgroup reads past them into the `a` tile, the
  // next stage or, from the last slot, the tail (rows computed from those values are never read back)
  const int co_max = a.Cout < MT ? a.Cout : MT;
  const int norm_bytes = nb * p.NTC * 8;
  int tail = 0;
  auto size_ring = [&](int ts) {
    p.TS = ts; p.halves = TH / ts;
    p.HALO_H = ts + a.kh - 1; p.nvox_h = p.HALO_H * p.HALO_W;
    // TMA boxes land with dense groups; a 32-channel row group starts on the 512-byte SWIZZLE_64B repeat
    p.a_plane = p.nvox_h * p.x_ch * 2;
    if (p.x_ch == 32) p.a_plane = (p.a_plane + 511) / 512 * 512;
    p.dy_plane = ts * TW * p.dy_ch * 2;
    // a multiple of 1024 (co_max >= 8, ts >= 8): the `a` box starts 1024-byte aligned.  With a row image in the stage
    // every stage starts on the 1024-byte SWIZZLE_128B repeat as well.
    p.dy_bytes = (co_max / p.dy_ch) * p.dy_plane;
    const int align = p.dy_ch != 8 || p.x_ch != 8 ? 1024 : 128;
    p.a_bytes = (p.NTC / p.x_ch) * p.a_plane; p.a_bytes = (p.a_bytes + align - 1) / align * align;
    p.stage_bytes = p.a_bytes + p.dy_bytes;
    // a plane-image A descriptor spans 8 whole planes per warpgroup and may read past the staged ones; a row image's
    // descriptor stays inside them (Cout 32: its second 32-channel atom is the first one again, LBO = 0)
    const int span = p.dy_ch == 8 ? (co_max + 63) / 64 * 8 * p.dy_plane : 0;
    tail = span > p.stage_bytes ? span - p.stage_bytes : 0;
    p.NS = (227 * 1024 - 2048 - tail - norm_bytes) / p.stage_bytes;
    if (p.NS > kMaxStages) p.NS = kMaxStages;
  };
  // whole 16x8 tiles, or two 8-row halves per tile where fewer than 4 whole tiles fit
  auto size = [&](int dy_ch, int x_ch) {
    p.dy_ch = dy_ch; p.x_ch = x_ch; p.x_boxes = x_ch == 8 ? 1 : p.NTC / x_ch;
    size_ring(TH);
    if (p.NS < 4) size_ring(TH / 2);
  };
  // row images: dy where the M tile is whole 32- or 64-channel groups of real channels, x at Cin tiles of 32, 64, 96 —
  // unless aligning the stages to the swizzle repeat would cost the ring a stage (a row image next to a plane image)
  size(8, 8);
  const int ns_planes = p.NS, ts_planes = p.TS;
  const int dy_ch = co_max == 32 ? 32 : (co_max == 64 || (co_max == MT && a.Cout % 64 == 0)) ? 64 : 8;
  const int x_ch = p.NTC == 64 ? 64 : (p.NTC == 32 || p.NTC == 96) ? 32 : 8;
  if (dy_ch != 8 || x_ch != 8) {
    size(dy_ch, x_ch);
    if (p.NS != ns_planes || p.TS != ts_planes) size(8, 8);
  }
  if (p.NS < 2) return false;
  p.tiles_h = (a.H + TH - 1) / TH; p.tiles_w = (a.W + TW - 1) / TW;
  const int64_t nvt = (int64_t)a.B * a.D * p.tiles_h * p.tiles_w;
  if (nvt > 0x7fffffff) return false;
  p.nvt = (int)nvt;
  const int64_t jobs = (int64_t)p.co_tiles * p.ci_tiles * a.kd * p.ngroups;
  int S = (int)(B200SEG_NUM_SMS / jobs); if (S < 1) S = 1;
  if (S > p.nvt) S = p.nvt;
  p.S = S;
  // wgmma descriptor templates: the layout type in bits 62-63 (0 none, 1 SWIZZLE_128B, 2 SWIZZLE_64B), LBO and SBO.
  // MN-major no swizzle: LBO = next 8 voxels (K), SBO = next 8-channel plane (M / N).  MN-major swizzled: LBO = next
  // channel group (M / N), SBO = next 8 voxel rows (K).  The base-offset field stays 0 although a tap or K step starts
  // an operand mid-way through the 8-row swizzle atom: the tensor core XORs each row's chunks with bits 7.. of the row's
  // own shared address, as the TMA unit does when it stores them, so the start address alone places every row (checked
  // bit for bit against the plane image on H100; setting the field to the start's phase corrupts dW).
  auto layout = [](int ch) { return (uint64_t)(ch == 64 ? 1 : ch == 32 ? 2 : 0) << 62; };
  auto desc = [](uint32_t lbo, uint32_t sbo) {
    return (uint64_t)((lbo >> 4) & 0x3FFF) << 16 | (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  };
  p.dy_desc = layout(p.dy_ch) | (p.dy_ch == 8 ? desc(128u, (uint32_t)p.dy_plane) : desc(0u, 8u * 2u * p.dy_ch));
  // B: the next 8 voxels of a K step lie one halo row on
  p.x_desc = layout(p.x_ch) | (p.x_ch == 8 ? desc((uint32_t)p.HALO_W * 16u, (uint32_t)p.a_plane)
                                            : desc((uint32_t)p.a_plane, (uint32_t)p.HALO_W * 2u * p.x_ch));
  int off = p.NS * p.stage_bytes + tail;
  off = (off + 15) / 16 * 16;
  p.smem_bar_off = off; off += 3 * p.NS * 8;
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
  // the alignment conditions of conv3d_wgrad_tc_supported are the ones TMA needs; only a missing driver entry point
  // can make this fail
  if (!b200seg_make_act_tmap(&p.tm_dy, a.dy, a.dy_ld, a.dy_coff, a.Cout, a.B * a.D, a.H, a.W, TW, p.TS,
                             (a.Cout < MT ? a.Cout : MT) / p.dy_ch, p.dy_ch) ||
      !b200seg_make_act_tmap(&p.tm_x, a.x, a.x_ld, a.x_coff, a.Cin, a.B * a.D, a.H, a.W, p.HALO_W, p.HALO_H,
                             p.NTC / p.x_ch / p.x_boxes, p.x_ch))
    return B200SEG_ECUDA;
  p.x_stats = a.x_stats; p.eps = a.eps; p.act = a.act;
  p.x_affine = a.x_affine; p.per_channel = a.per_channel;
  p.dw = a.dw;
  const int64_t jobs = (int64_t)p.co_tiles * p.ci_tiles * a.kd * p.ngroups;
  const int smem_bytes = p.smem_norm_off + (a.per_channel ? 1 : a.B) * p.NTC * 8 + 64;
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
