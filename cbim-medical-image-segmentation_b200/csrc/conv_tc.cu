// conv_tc.cu — conv3d forward / data-gradient as a wgmma implicit GEMM (sm_90a), fp16 operands, fp32 accumulation
// in registers.  Replaces cuDNN fprop/dgrad behind nn.Conv3d (conv_layers.py:29-38) and fuses the surrounding
// InstanceNorm+ReLU (conv_layers.py:40-43), residual add (:92) and the next layer's InstanceNorm reduction.
//
// GEMM view (per CTA tile):  D[128 voxels][NT cout] += A[128 voxels][KC cin] * B[KC cin][NT cout]
// for every filter tap and every KC-chunk of Cin.
//   * M tile  = 16(h) x 8(w) output voxels of one depth slice; GEMM row r = hl*8 + wl.
//   * A operand = a HALO tile (16+kh-1)x(8+kw-1) voxels x KC channels of ONE input depth slice, staged
//     once in shared memory as [KC/8][halo voxel][8 ch] (K-major, no-swizzle core matrices:
//     8 consecutive w-voxels x 16 B).  Every (kh,kw) tap reads the SAME staged tile through a shifted
//     matrix descriptor (start += (zh*HALO_W + zw)*16 B, SBO = HALO_W*16 B) — im2col is never formed.
//   * Staging: raw inputs (every data-gradient launch) arrive as one tensor-TMA box per stage; inputs that need
//     InstanceNorm / activation are copied by the loader warps (TMA box or 16-byte cp.async, up to three stages
//     ahead), normalised + activated IN PLACE in shared memory and then published to the MMA warpgroups.  The
//     normalised activation tensor never exists in HBM.
//   * B operand = weights pre-packed on device into the exact shared-memory image per (ntile,tap,kchunk)
//     ([KC/8][NT][8] fp16): resident for the CTA's lifetime when the layer's weights fit (<=112 KB), else streamed
//     by 1-D bulk TMA (cp.async.bulk) through an mbarrier ring.
//   * D lives in the registers of two consumer warpgroups (64 rows each, wgmma m64 x NT x 16), which also run the
//     epilogue: bias / residual / dgrad ReLU-mask, fp16 store, InstanceNorm sums of the stored tile.  The epilogue's
//     side operand (residual, or the pre-norm input of the dgrad mask) is one tensor-TMA box per tile in shared memory,
//     issued a tile or more ahead, so no epilogue waits on a global load.
// Warp roles (640 threads = 5 warpgroups, 1 CTA/SM, persistent over tiles; `setmaxnreg` moves registers from the
// loader / weight warpgroups to the two consumer warpgroups, whose accumulators need them):
//   warps 0-7  MMA + epilogue (warpgroup g = GEMM rows 64g .. 64g+63)
//   warps 8-15 A loaders (cp.async / TMA + in-place transform; all 256 threads share every stage)
//   warp  16   weight producer (bulk TMA); warp 17 side-operand producer (tensor TMA); warps 18-19 only complete the
//              warpgroup
#include "common.cuh"
#include "conv_args.h"
#include "tc_common.cuh"
#include "tmap.h"
#include "wgmma.cuh"
#include <string.h>

namespace {

using namespace tc;

constexpr int TH = 16, TW = 8;            // output tile (h, w); M = 128
constexpr int kConsumerWGs = 2;           // MMA + epilogue warpgroups (warps 0-7)
constexpr int kLoadWarp0 = 8;
constexpr int kLoadThreads = 256;
constexpr int kWgtWarp = 16;
constexpr int kThreads = 20 * 32;   // 640: five complete warpgroups (setmaxnreg is a warpgroup-wide instruction);
                                    // warps 18-19 only take part in the block-wide barriers
// Registers per thread after the role dispatch.  setmaxnreg trades registers inside the CTA's OWN pool — what the
// launch allotted: 640 threads x 96 = 61440, not the SM's 65536 (an over-subscribed split makes setmaxnreg.inc wait
// forever).  Split: 2 consumer warpgroups x 136 (NT/2 <= 64 accumulators + epilogue) + 2 loader warpgroups x 80 (three
// transform chains interleaved) + {weights, 3 idle} x 40 = 60416.
constexpr int kRegsLaunch = 96, kRegsConsumer = 136, kRegsLoad = 80, kRegsWgt = 40;
static_assert(2 * 128 * kRegsConsumer + 2 * 128 * kRegsLoad + 128 * kRegsWgt <= kThreads * kRegsLaunch, "register split exceeds the CTA pool");

struct TcParams {
  ConvArgs a;
  const void* wimg;        // weight image [ntile][tap][kchunk][KC/8][NT][8]
  int KC, NKC, NT, NTILES;
  int HALO_H, HALO_W, nvox_h, plane_stride;   // plane_stride in bytes (odd multiple of 16)
  int a_stage_bytes, b_stage_bytes, SA, SB;
  int tiles_h, tiles_w, n_tiles;
  int w_resident;          // all weights of the layer live in shared memory for the CTA's lifetime (no B ring)
  int prefetch;            // A stages the loaders keep in flight (1..3, < SA)
  int use_tma;             // halo tiles are staged by ONE tensor-TMA box per stage (else 16-byte cp.async copies)
  int SS, side_stage_bytes; // side-operand slots (residual / dgrad_x tile, [NT/8 planes][128 voxels][8 ch]); 0 = none
  int smem_a_off, smem_b_off, smem_side_off, smem_bar_off, smem_norm_off, smem_gnorm_off;
  int norm_bstride;        // entries per sample in the {scale, shift} table: Cin, or 0 for a per-channel table
  alignas(64) CUtensorMap tm_x;      // x as {8 ch, w, h, channel plane, b*D + d}
  alignas(64) CUtensorMap tm_side;   // res or gx (Cout channels), same dims; box {8, TW, TH, NT/8}
};

// barrier block layout (uint64 each): a_full[SA] a_empty[SA] b_full[SB] b_empty[SB] a_land[SA] side_full[SS]
// side_empty[SS].  SA / SB / SS are read from the kernel parameters, not copied: copies would hold registers in every
// role (measured: more loader spills).
struct Bars {
  uint32_t bar0; const TcParams& p;
  __device__ __forceinline__ uint32_t a_full(int i) const { return bar0 + 8u * (uint32_t)i; }
  __device__ __forceinline__ uint32_t a_empty(int i) const { return bar0 + 8u * (uint32_t)(p.SA + i); }
  __device__ __forceinline__ uint32_t b_full(int i) const { return bar0 + 8u * (uint32_t)(2 * p.SA + i); }
  __device__ __forceinline__ uint32_t b_empty(int i) const { return bar0 + 8u * (uint32_t)(2 * p.SA + p.SB + i); }
  __device__ __forceinline__ uint32_t a_land(int i) const { return bar0 + 8u * (uint32_t)(2 * p.SA + 2 * p.SB + i); }   // TMA: the stage's box has landed
  __device__ __forceinline__ uint32_t side_full(int i) const { return bar0 + 8u * (uint32_t)(3 * p.SA + 2 * p.SB + i); }
  __device__ __forceinline__ uint32_t side_empty(int i) const { return bar0 + 8u * (uint32_t)(3 * p.SA + 2 * p.SB + p.SS + i); }
};

struct TileCoord { int b, d, h0, w0, ntile; };
// Persistent tile walk t = blockIdx.x, +gridDim.x, ... as a mixed-radix counter (ntile, w-tile, h-tile, d, b):
// one set of divisions per kernel instead of four per tile per warp role (~1000 cycles/tile measured).
// TileWalk = the constants of the walk (radices, digits of the stride); TileIter = one position on it.
struct TileWalk {
  int s0, s1, s2, s3, s4;           // digits of the stride
  int r0, r1, r2, r3;               // radices
  int n_tiles, stride;
  __device__ __forceinline__ void init(const TcParams& p) {
    r0 = p.NTILES; r1 = p.tiles_w; r2 = p.tiles_h; r3 = p.a.D;
    n_tiles = p.n_tiles; stride = gridDim.x;
    int x = stride;
    s0 = x % r0; x /= r0; s1 = x % r1; x /= r1; s2 = x % r2; x /= r2; s3 = x % r3; s4 = x / r3;
  }
};
struct TileIter {
  int ntile, wi, hi, d, b, t;       // current digits, linear index
  __device__ __forceinline__ void init(const TileWalk& k) {
    t = blockIdx.x;
    int x = t;
    ntile = x % k.r0; x /= k.r0; wi = x % k.r1; x /= k.r1; hi = x % k.r2; x /= k.r2; d = x % k.r3; b = x / k.r3;
  }
  __device__ __forceinline__ bool valid(const TileWalk& k) const { return t < k.n_tiles; }
  __device__ __forceinline__ TileCoord coord() const { TileCoord c; c.b = b; c.d = d; c.h0 = hi * TH; c.w0 = wi * TW; c.ntile = ntile; return c; }
  __device__ __forceinline__ void next(const TileWalk& k) {
    t += k.stride;
    int c;
    ntile += k.s0; c = ntile >= k.r0; if (c) ntile -= k.r0;
    wi += k.s1 + c; c = wi >= k.r1; if (c) wi -= k.r1;
    hi += k.s2 + c; c = hi >= k.r2; if (c) hi -= k.r2;
    d += k.s3 + c; c = d >= k.r3; if (c) d -= k.r3;
    b += k.s4 + c;
  }
};

// One A stage = (tile, K chunk, depth tap) with an in-volume input slice; the loaders walk them in exactly the order
// the MMA warpgroups consume them: for tile { for kc { for zd { skip if din outside the volume } } }.
struct StageCursor {
  TileIter ti; int kc, zd, din;
  __device__ __forceinline__ void init(const TileWalk& k, const TcParams& p) {
    ti.init(k); kc = 0; zd = -1;
    if (ti.valid(k)) next(k, p);
  }
  __device__ __forceinline__ bool valid(const TileWalk& k) const { return ti.valid(k); }
  __device__ __forceinline__ void next(const TileWalk& k, const TcParams& p) {
    for (;;) {
      if (++zd == p.a.kd) { zd = 0; if (++kc == p.NKC) { kc = 0; ti.next(k); if (!ti.valid(k)) return; } }
      din = ti.d + zd - p.a.kd / 2;
      if ((unsigned)din < (unsigned)p.a.D) return;
    }
  }
};

// ------------------------------------------------------------------ A loaders
// cp.async (LDGSTS) prefetch of P stages + in-place InstanceNorm/ReLU once a stage has landed.  Each thread owns ONE
// 8-channel plane and a fixed set of (at most kMaxChunks) halo voxels of it, copies exactly those 16-byte chunks and
// later transforms exactly those chunks, so no cross-thread synchronisation is needed between copy and transform.
// Everything that does not depend on the tile (voxel slot, offset from the tile origin, halo row / column) is computed
// once per thread; per stage the work is one pointer add per chunk, and the bounds tests vanish for interior tiles.
constexpr int kMaxChunks = 6;
// the chunk table covers every halo tile: kh, kw <= 3 (conv3d_tc_shape_ok) and KC <= 64 (tc_pick_kc), so at most
// 18 x 10 halo voxels over at least 256 / 8 threads per plane
static_assert(kMaxChunks * (kLoadThreads / (64 / 8)) >= (TH + 2) * (TW + 2), "loader chunk table smaller than the largest halo tile");

template <int P, bool TMA>
__device__ __forceinline__ void loader_role(const TcParams& p, uint8_t* smem, const float2* s_norm, const Bars& bars) {
  const ConvArgs& a = p.a;
  const int lt = threadIdx.x - kLoadWarp0 * 32;
  const int cpv = p.KC / 8;
  const int vstep = kLoadThreads / cpv;
  const bool active = lt < vstep * cpv;
  const int c8 = lt % cpv, v0 = lt / cpv;
  const int ph = a.kh / 2, pw = a.kw / 2;
  const bool xform = (a.x_stats != nullptr) || (a.x_affine != nullptr) || (a.act != 0);
  const int act = a.act;
  const __half* xbase = reinterpret_cast<const __half*>(a.x);
  const uint32_t smem_a = smem_u32(smem + p.smem_a_off) + (uint32_t)(c8 * p.plane_stride);
  uint8_t* smem_a_gen = smem + p.smem_a_off + c8 * p.plane_stride;
  // TMA mode: thread 0 stages the halo tile with ONE tensor-TMA box per stage; every thread then transforms exactly
  // the chunks it would have copied (same table, same code) once the box has landed.  Nobody but thread 0 walks the
  // issue cursor.
  const uint32_t stage_tx = (uint32_t)(cpv * p.nvox_h * 16);

  // per-thread chunk table
  int rel[kMaxChunks];            // element offset of the chunk's voxel from the (possibly out-of-volume) tile origin
  uint32_t hw[kMaxChunks];        // halo row << 16 | halo column ; 0xffffffff = no such chunk
#pragma unroll
  for (int i = 0; i < kMaxChunks; ++i) {
    const int v = v0 + i * vstep;
    const bool have = active && v < p.nvox_h;
    const int hh = v / p.HALO_W, ww = v % p.HALO_W;
    if constexpr (TMA) {
      rel[i] = c8 * p.plane_stride + v * 16;      // byte offset of the chunk inside a stage: plane image [c8][v][8 ch]
    } else {
      rel[i] = (hh * a.W + ww) * a.x_ld;
    }
    hw[i] = have ? ((uint32_t)hh << 16) | (uint32_t)ww : 0xffffffffu;
  }

  const int nch = (p.nvox_h + vstep - 1) / vstep;       // chunks per thread actually present (warp-uniform loop bound)

  TileWalk tw; tw.init(p);
  StageCursor ci, cd;
  ci.init(tw, p); cd.init(tw, p);
  Ring ri, rd; ri.init(p.SA); rd.init(p.SA);

  auto issue = [&]() {
    if constexpr (TMA) {
      if (lt == 0) {
        mbar_wait(bars.a_empty(ri.idx), ri.phase ^ 1);
        mbar_arrive_expect_tx(bars.a_land(ri.idx), stage_tx);
        const uint32_t dst = smem_u32(smem + p.smem_a_off) + (uint32_t)(ri.idx * p.a_stage_bytes);
        tma_load_5d(dst, &p.tm_x, bars.a_land(ri.idx), 0, ci.ti.wi * TW - pw, ci.ti.hi * TH - ph, ci.kc * cpv, ci.ti.b * a.D + ci.din);
        ri.advance(); ci.next(tw, p);
      }
    } else {
    mbar_wait(bars.a_empty(ri.idx), ri.phase ^ 1);
    const uint32_t dst = smem_a + (uint32_t)(ri.idx * p.a_stage_bytes) + (uint32_t)v0 * 16u;
    const int hb = ci.ti.hi * TH - ph, wb = ci.ti.wi * TW - pw;
    const bool interior = hb >= 0 && wb >= 0 && hb + p.HALO_H <= a.H && wb + p.HALO_W <= a.W;
    const __half* xs = xbase + (((int64_t)(ci.ti.b * a.D + ci.din) * a.H + hb) * a.W + wb) * a.x_ld + a.x_coff + ci.kc * p.KC + c8 * 8;
#pragma unroll
    for (int i = 0; i < kMaxChunks; ++i) {
      if (i < nch && hw[i] != 0xffffffffu) {
        const bool ok = interior || (((unsigned)(hb + (int)(hw[i] >> 16)) < (unsigned)a.H) && ((unsigned)(wb + (int)(hw[i] & 0xffffu)) < (unsigned)a.W));
        cp_async16(dst + (uint32_t)(i * vstep) * 16u, ok ? (const void*)(xs + rel[i]) : (const void*)xbase, ok ? 16u : 0u);
      }
    }
    ri.advance(); ci.next(tw, p);
    }
  };

  const float slope = act_slope(act);
  const bool relu = act == B200SEG_ACT_RELU;
  float sc[8], sf[8];                              // x*sc + sf: (x - mean) * rstd, or the per-channel affine transform
  int norm_key = -1;                               // (b, kc) the constants belong to
#pragma unroll
  for (int i = 0; i < P; ++i) { if (ci.valid(tw)) issue(); if constexpr (!TMA) cp_async_commit(); }
  while (cd.valid(tw)) {
    if constexpr (TMA) mbar_wait(bars.a_land(rd.idx), rd.phase);
    else cp_async_wait<P - 1>();      // this thread's copies of the oldest stage have landed
    if (xform && active) {
      const int key = cd.ti.b * p.NKC + cd.kc;
      if (key != norm_key) {
        norm_key = key;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 st = s_norm[cd.ti.b * p.norm_bstride + cd.kc * p.KC + c8 * 8 + j];
          sc[j] = st.x; sf[j] = st.y;
        }
      }
      uint8_t* sp = TMA ? smem + p.smem_a_off + rd.idx * p.a_stage_bytes : smem_a_gen + rd.idx * p.a_stage_bytes + v0 * 16;
      auto chunk = [&](int i) { return TMA ? sp + rel[i] : sp + (i * vstep) * 16; };
      const int hb = cd.ti.hi * TH - ph, wb = cd.ti.wi * TW - pw;
      const bool interior = hb >= 0 && wb >= 0 && hb + p.HALO_H <= a.H && wb + p.HALO_W <= a.W;
      // two batches of three chunks: all loads of a batch are issued before the first use (ILP for the one loader
      // warp each scheduler has), zero-filled padding voxels are left untouched (the conv pads the NORMALISED tensor)
#pragma unroll
      for (int i0 = 0; i0 < kMaxChunks; i0 += 3) {
        if (i0 >= nch) break;
        uint4 raw[3]; bool ok[3];
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          const int i = i0 + u;
          ok[u] = i < nch && hw[i] != 0xffffffffu &&
                  (interior || (((unsigned)(hb + (int)(hw[i] >> 16)) < (unsigned)a.H) && ((unsigned)(wb + (int)(hw[i] & 0xffffu)) < (unsigned)a.W)));
          if constexpr (TMA) raw[u] = make_uint4(0, 0, 0, 0);
          if (ok[u]) raw[u] = *reinterpret_cast<const uint4*>(chunk(i));
        }
        if constexpr (TMA) {      // one branch per batch: the three chunks' dependency chains interleave
          if (relu) {
#pragma unroll
            for (int u = 0; u < 3; ++u) raw[u] = norm_act8<true>(raw[u], sc, sf, slope);
          } else {
#pragma unroll
            for (int u = 0; u < 3; ++u) raw[u] = norm_act8<false>(raw[u], sc, sf, slope);
          }
#pragma unroll
          for (int u = 0; u < 3; ++u)
            if (ok[u]) *reinterpret_cast<uint4*>(chunk(i0 + u)) = raw[u];
        } else {      // 64 registers: one chunk at a time
#pragma unroll
          for (int u = 0; u < 3; ++u) {
            if (!ok[u]) continue;
            raw[u] = relu ? norm_act8<true>(raw[u], sc, sf, slope) : norm_act8<false>(raw[u], sc, sf, slope);
            *reinterpret_cast<uint4*>(chunk(i0 + u)) = raw[u];
          }
        }
      }
    }
    fence_proxy_async();          // generic-proxy / cp.async writes -> visible to the tensor core (async proxy)
    mbar_arrive(bars.a_full(rd.idx));
    rd.advance(); cd.next(tw, p);
    if (ci.valid(tw)) issue();
    if constexpr (!TMA) cp_async_commit();
  }
  if constexpr (!TMA) cp_async_wait<0>();
}

// ---- TMA staging of RAW inputs (every data-gradient launch): one elected loader thread issues ONE tensor-TMA box
// {8 ch, HALO_W, HALO_H, KC/8 planes} per stage — the TMA unit writes the [plane][halo voxel][8 ch] image and zero-fills
// conv padding / ragged tiles — and the MMA warpgroups consume the stage straight off the TMA's transaction barrier: no
// loader instruction touches the data.  (Inputs that need InstanceNorm / activation go through loader_role<P>, whose TMA
// mode lands the same box and then transforms it in place with the cp.async path's per-thread chunk table.)
__device__ __forceinline__ void loader_role_tma(const TcParams& p, uint8_t* smem, const Bars& bars) {
  const ConvArgs& a = p.a;
  const int lt = threadIdx.x - kLoadWarp0 * 32;
  const int ph = a.kh / 2, pw = a.kw / 2;
  const uint32_t smem_a = smem_u32(smem + p.smem_a_off);
  TileWalk tw; tw.init(p);
  const uint32_t stage_tx = (uint32_t)((p.KC / 8) * p.nvox_h * 16);
  auto issue = [&](const StageCursor& c, int slot) {
    mbar_arrive_expect_tx(bars.a_land(slot), stage_tx);
    tma_load_5d(smem_a + (uint32_t)(slot * p.a_stage_bytes), &p.tm_x, bars.a_land(slot), 0, c.ti.wi * TW - pw, c.ti.hi * TH - ph,
                  c.kc * (p.KC / 8), c.ti.b * a.D + c.din);
  };
  if (lt == 0) {
    StageCursor c; c.init(tw, p);
    Ring r; r.init(p.SA);
    for (; c.valid(tw); c.next(tw, p)) {
      mbar_wait(bars.a_empty(r.idx), r.phase ^ 1);
      issue(c, r.idx);
      r.advance();
    }
  }
}

// ------------------------------------------------------------------ MMA + epilogue (two consumer warpgroups)
// Warpgroup g owns GEMM rows 64g .. 64g+63 (tile rows hl = 8g .. 8g+7): its A descriptor starts 8g halo rows into the
// staged tile.  Per filter tap one wgmma group (KC/16 instructions m64 x NT x 16) is committed; the group before it is
// then waited for and the shared-memory slots only it read (its B slot when the weights stream, the A stage after its
// last tap) are handed back, so one group is always in flight while the next tap's operands are checked.
// Epilogue straight from the accumulator registers: thread (warp w, lane l) holds rows r0 = 64g + 16w + l/4 and r0 + 8
// (same w, next h) and column pairs 8j + 2(l%4).  InstanceNorm sums are reduced over the 8 lanes sharing a column pair
// and kept in registers (lane l keeps the groups j with j % 8 == l / 4) while consecutive tiles share a (batch, N tile);
// then each warp adds them to y_stats with one fp64 atomic per value.  Every addition before the atomic happens in a
// fixed order; the order of the fp64 atomics can move only the last fp64 bits of the statistics.
// KSTEPS = KC / 16 is a template argument so that a tap's group is straight-line code: with a run-time trip count the
// unrolled loop and its remainder made ptxas move accumulators between the MMAs and serialise them (C7519).
template <int NT, int KSTEPS>
__device__ __forceinline__ void consumer_role(const TcParams& p, int wg, int tid, uint8_t* smem, const Bars& bars, const float2* s_gnorm) {
  const ConvArgs& a = p.a;
  // A stage ready: published by the loaders, or (raw input staged by TMA) the TMA's own transaction barrier
  const uint32_t a_ready0 = (p.use_tma && !(a.x_stats || a.x_affine || a.act)) ? bars.a_land(0) : bars.a_full(0);
  const int warp = tid >> 5, lane = tid & 31;
  const bool signaller = tid == 0;
  const int r0 = 64 * wg + 16 * warp + (lane >> 2);
  const int hl0 = r0 >> 3, wl = r0 & 7;
  const int taps_hw = a.kh * a.kw, pd = a.kd / 2;
  // A: plane image = K-major no-swizzle core matrices (LBO = plane, SBO = one halo row of 16-byte slots)
  const uint64_t a_tmpl = make_desc(0, (uint32_t)p.plane_stride, (uint32_t)p.HALO_W * 16u);
  const uint64_t b_tmpl = make_desc(0, (uint32_t)NT * 16u, 128u);
  const uint32_t a_kstep = (2u * (uint32_t)p.plane_stride) >> 4, b_kstep = (2u * (uint32_t)NT * 16u) >> 4;
  const uint32_t a_stage16 = (uint32_t)p.a_stage_bytes >> 4, b_stage16 = (uint32_t)p.b_stage_bytes >> 4;
  const uint32_t smem_a16 = (smem_u32(smem + p.smem_a_off) >> 4) + (uint32_t)(wg * 8 * p.HALO_W);
  const uint32_t smem_b16 = smem_u32(smem + p.smem_b_off) >> 4;
  const uint32_t a_rowstep = (uint32_t)p.HALO_W;                      // next tap row, in 16-byte units
  const int resident = p.w_resident;
  const int taps_all = a.kd * taps_hw;
  const uint32_t res_step = (uint32_t)p.NKC * b_stage16;
  const bool dgrad = a.gx != nullptr, want_stats = a.y_stats != nullptr, has_side = dgrad || a.res != nullptr;
  const float gslope = act_slope(a.g_act);
  constexpr int KEEP = (NT / 8 + 7) / 8;                               // column groups whose sums this lane keeps
  float ks[KEEP][4];                                                   // {sum c, sum c+1, second c, second c+1}
#pragma unroll
  for (int k = 0; k < KEEP; ++k) ks[k][0] = ks[k][1] = ks[k][2] = ks[k][3] = 0.f;
  int stat_key = -1;                                                   // b * NTILES + ntile the kept sums belong to
  auto flush = [&]() {
    if (stat_key < 0) return;
    const int b = stat_key / p.NTILES, cb = (stat_key % p.NTILES) * NT;
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
      const int j = 8 * k + (lane >> 2);
      if (j < NT / 8) {
        double* st = a.y_stats + ((int64_t)b * a.Cout + cb + 8 * j + 2 * (lane & 3)) * 2;
        atomicAdd(st, (double)ks[k][0]); atomicAdd(st + 1, (double)ks[k][2]);
        atomicAdd(st + 2, (double)ks[k][1]); atomicAdd(st + 3, (double)ks[k][3]);
      }
      ks[k][0] = ks[k][1] = ks[k][2] = ks[k][3] = 0.f;
    }
  };
  if (resident) mbar_wait(bars.b_full(0), 0);
  Ring ra, rb, rs; ra.init(p.SA); rb.init(p.SB); rs.init(p.SS);
  int pend_a = -1, pend_b = -1;                                        // slots read only by the group in flight
  auto release = [&]() {
    if (signaller) {
      if (pend_b >= 0) mbar_arrive(bars.b_empty(pend_b));
      if (pend_a >= 0) mbar_arrive(bars.a_empty(pend_a));
    }
    pend_a = -1; pend_b = -1;
  };
  float acc[NT / 2];
  TileWalk tw; tw.init(p); TileIter ti; ti.init(tw);
  for (; ti.valid(tw); ti.next(tw)) {
    const TileCoord tc = ti.coord();
    uint32_t accumulate = 0;
    for (int kc = 0; kc < p.NKC; ++kc) {
      for (int zd = 0; zd < a.kd; ++zd) {
        const int din = tc.d + zd - pd;
        if ((unsigned)din >= (unsigned)a.D) continue;
        mbar_wait(a_ready0 + 8u * (uint32_t)ra.idx, ra.phase);
        uint64_t da_row = a_tmpl + (uint64_t)(smem_a16 + (uint32_t)ra.idx * a_stage16);
        uint64_t db_res = b_tmpl + (uint64_t)(smem_b16 + (uint32_t)((tc.ntile * taps_all + zd * taps_hw) * p.NKC + kc) * b_stage16);
        for (int zh = 0; zh < a.kh; ++zh) {
          for (int zw = 0; zw < a.kw; ++zw) {
            uint64_t db;
            int bslot = -1;
            if (resident) {
              db = db_res;
              db_res += (uint64_t)res_step;
            } else {
              mbar_wait(bars.b_full(rb.idx), rb.phase);
              db = b_tmpl + (uint64_t)(smem_b16 + (uint32_t)rb.idx * b_stage16);
              bslot = rb.idx;
              rb.advance();
            }
            const uint64_t da = da_row + (uint64_t)((uint32_t)zh * a_rowstep + (uint32_t)zw);
            wgmma_fence_operands(acc);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < KSTEPS; ++j)
              Wgmma<NT, 0, 0>::mma(acc, da + (uint64_t)((uint32_t)j * a_kstep), db + (uint64_t)((uint32_t)j * b_kstep), accumulate | (uint32_t)(j > 0));
            accumulate = 1;
            wgmma_commit();
            wgmma_wait<1>();                       // the previous group has retired: its slots are free
            wgmma_fence_operands(acc);
            release();
            pend_b = bslot;
            if (zh == a.kh - 1 && zw == a.kw - 1) pend_a = ra.idx;
          }
        }
        ra.advance();
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    release();

    // ---- epilogue: bias / residual / dgrad mask, fp16 rounding and store, InstanceNorm sums
    const int co_base = tc.ntile * NT;
    __half* yp[2];
    bool valid[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int h = tc.h0 + hl0 + i, w = tc.w0 + wl;
      valid[i] = h < a.H && w < a.W;
      const int64_t vox = ((int64_t)(tc.b * a.D + tc.d) * a.H + (valid[i] ? h : 0)) * a.W + (valid[i] ? w : 0);
      yp[i] = reinterpret_cast<__half*>(a.y) + vox * a.y_ld + a.y_coff + co_base;
    }
    // side tile [NT/8 planes][128 rows][8 ch]: rows r0, r0 + 8 of plane j; the 8 lanes sharing a plane read 128
    // consecutive bytes
    const uint8_t* side = smem + p.smem_side_off + rs.idx * p.side_stage_bytes + r0 * 16 + 4 * (lane & 3);
    if (has_side) mbar_wait(bars.side_full(rs.idx), rs.phase);
    const float2* gn = s_gnorm + tc.b * a.Cout + co_base;
    if (want_stats && tc.b * p.NTILES + tc.ntile != stat_key) { flush(); stat_key = tc.b * p.NTILES + tc.ntile; }
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      float2 bv = make_float2(0.f, 0.f);
      if (a.bias) bv = *reinterpret_cast<const float2*>(a.bias + co_base + c);
      float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!valid[i]) continue;                 // rows outside the volume: nothing stored, nothing counted
        float v0 = acc[4 * j + 2 * i] + bv.x, v1 = acc[4 * j + 2 * i + 1] + bv.y;
        float2 sv = make_float2(0.f, 0.f);
        if (has_side) sv = __half22float2(*reinterpret_cast<const __half2*>(side + j * (TH * TW * 16) + i * 128));
        if (dgrad) {
          const float4 mr = *reinterpret_cast<const float4*>(gn + c);      // {mean, rstd} of two channels
          const float h0 = (sv.x - mr.x) * mr.y, h1 = (sv.y - mr.z) * mr.w;
          v0 = __half2float(__float2half_rn(v0 * act_grad_s(h0, gslope)));
          v1 = __half2float(__float2half_rn(v1 * act_grad_s(h1, gslope)));
          s0 += v0; s1 += v1; q0 = fmaf(v0, h0, q0); q1 = fmaf(v1, h1, q1);
        } else {
          v0 = __half2float(__float2half_rn(v0)); v1 = __half2float(__float2half_rn(v1));
          if (has_side) { v0 = __half2float(__float2half_rn(v0 + sv.x)); v1 = __half2float(__float2half_rn(v1 + sv.y)); }
          s0 += v0; s1 += v1; q0 = fmaf(v0, v0, q0); q1 = fmaf(v1, v1, q1);
        }
        *reinterpret_cast<__half2*>(yp[i] + c) = __floats2half2_rn(v0, v1);
      }
      if (want_stats) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o);
          q0 += __shfl_xor_sync(0xffffffffu, q0, o); q1 += __shfl_xor_sync(0xffffffffu, q1, o);
        }
        if ((j & 7) == (lane >> 2)) { ks[j >> 3][0] += s0; ks[j >> 3][1] += s1; ks[j >> 3][2] += q0; ks[j >> 3][3] += q1; }
      }
    }
    if (has_side) { mbar_arrive(bars.side_empty(rs.idx)); rs.advance(); }   // every consumer thread: its reads are done
  }
  if (want_stats) flush();
}

// ------------------------------------------------------------------ the kernel
// One instantiation per (NT, KC / 16) that tc_pick_nt / tc_pick_kc can produce, so each gets its own register
// allocation instead of sharing the worst case of every tile width.
template <int NT, int KSTEPS>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const ConvArgs& a = p.a;
  // canonical warp index: the shuffle makes it provably warp-uniform, so the role branches below are uniform branches
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int taps_hw = a.kh * a.kw;
  const int pd = a.kd / 2;
  const Bars bars{smem_u32(smem + p.smem_bar_off), p};

  float2* s_norm = reinterpret_cast<float2*>(smem + p.smem_norm_off);   // [B or 1][Cin] {scale, shift} of x
  float2* s_gnorm = reinterpret_cast<float2*>(smem + p.smem_gnorm_off); // [B][Cout] {mean, rstd} of dgrad_x
  const uint32_t smem_b = smem_u32(smem + p.smem_b_off);

  // ---- one-time setup
  if (threadIdx.x == 0) {
    for (int i = 0; i < p.SA; ++i) { mbar_init(bars.a_full(i), kLoadThreads); mbar_init(bars.a_empty(i), kConsumerWGs); mbar_init(bars.a_land(i), 1); }
    for (int i = 0; i < p.SB; ++i) { mbar_init(bars.b_full(i), 1); mbar_init(bars.b_empty(i), kConsumerWGs); }
    for (int i = 0; i < p.SS; ++i) { mbar_init(bars.side_full(i), 1); mbar_init(bars.side_empty(i), kConsumerWGs * 128); }
    fence_barrier_init();
  }
  {
    const double n = (double)a.D * a.H * a.W;
    for (int i = threadIdx.x; i < (a.per_channel ? 1 : a.B) * a.Cin; i += kThreads) {
      if (a.x_affine) {
        s_norm[i] = make_float2(a.x_affine[2 * i], a.x_affine[2 * i + 1]);
      } else {
        float m = 0.f, r = 1.f;
        if (a.x_stats) stats_to_mean_rstd(a.x_stats + (int64_t)i * 2, n, a.eps, m, r);
        s_norm[i] = make_float2(r, -m * r);
      }
    }
    if (a.gx) {
      for (int i = threadIdx.x; i < a.B * a.Cout; i += kThreads) {
        float m, r;
        stats_to_mean_rstd(a.g_stats + (int64_t)i * 2, n, a.g_eps, m, r);
        s_gnorm[i] = make_float2(m, r);
      }
    }
  }
  __syncthreads();

  if (warp >= kLoadWarp0 && warp < kWgtWarp) {
    // =========================== A LOADERS ===========================
    setmaxnreg_dec<kRegsLoad>();
    if (p.use_tma && !(a.x_stats || a.x_affine || a.act)) loader_role_tma(p, smem, bars);
    else if (p.use_tma) loader_role<3, true>(p, smem, s_norm, bars);
    else if (p.prefetch >= 3) loader_role<3, false>(p, smem, s_norm, bars);
    else loader_role<1, false>(p, smem, s_norm, bars);
  } else if (warp >= kWgtWarp) {
    setmaxnreg_dec<kRegsWgt>();
    if (warp == kWgtWarp && lane == 0) {
      // =========================== WEIGHT PRODUCER (bulk TMA) ===========================
      const uint8_t* wimg = reinterpret_cast<const uint8_t*>(p.wimg);
      const int taps = a.kd * taps_hw;
      if (p.w_resident) {
        // small layers: the whole weight image is loaded once; the consumers index it directly
        const int nblobs = p.NTILES * taps * p.NKC;
        mbar_arrive_expect_tx(bars.b_full(0), (uint32_t)(nblobs * p.b_stage_bytes));
        for (int i = 0; i < nblobs; ++i)
          bulk_g2s(smem_b + i * p.b_stage_bytes, wimg + (int64_t)i * p.b_stage_bytes, (uint32_t)p.b_stage_bytes, bars.b_full(0));
      } else {
        Ring ring; ring.init(p.SB);
        TileWalk tw; tw.init(p); TileIter ti; ti.init(tw);
        for (; ti.valid(tw); ti.next(tw)) {
          const TileCoord tc = ti.coord();
          for (int kc = 0; kc < p.NKC; ++kc) {
            for (int zd = 0; zd < a.kd; ++zd) {
              const int din = tc.d + zd - pd;
              if ((unsigned)din >= (unsigned)a.D) continue;
              for (int thw = 0; thw < taps_hw; ++thw) {
                const int tap = zd * taps_hw + thw;
                mbar_wait(bars.b_empty(ring.idx), ring.phase ^ 1);
                mbar_arrive_expect_tx(bars.b_full(ring.idx), (uint32_t)p.b_stage_bytes);
                const uint8_t* src = wimg + ((int64_t)(tc.ntile * taps + tap) * p.NKC + kc) * p.b_stage_bytes;
                bulk_g2s(smem_b + ring.idx * p.b_stage_bytes, src, (uint32_t)p.b_stage_bytes, bars.b_full(ring.idx));
                ring.advance();
              }
            }
          }
        }
      }
    } else if (warp == kWgtWarp + 1 && lane == 0 && p.SS > 0) {
      // =========================== SIDE-OPERAND PRODUCER (tensor TMA) ===========================
      // the residual / dgrad_x tile of every output tile, in tile order, up to SS tiles ahead of the epilogue
      const uint32_t smem_side = smem_u32(smem + p.smem_side_off);
      Ring ring; ring.init(p.SS);
      TileWalk tw; tw.init(p); TileIter ti; ti.init(tw);
      for (; ti.valid(tw); ti.next(tw)) {
        mbar_wait(bars.side_empty(ring.idx), ring.phase ^ 1);
        mbar_arrive_expect_tx(bars.side_full(ring.idx), (uint32_t)p.side_stage_bytes);
        tma_load_5d(smem_side + (uint32_t)(ring.idx * p.side_stage_bytes), &p.tm_side, bars.side_full(ring.idx), 0, ti.wi * TW,
                    ti.hi * TH, ti.ntile * (p.NT / 8), ti.b * a.D + ti.d);
        ring.advance();
      }
    }
  } else {
    // =========================== MMA + EPILOGUE (warps 0-7) ===========================
    setmaxnreg_inc<kRegsConsumer>();
    const int wg = warp >> 2, tid = threadIdx.x & 127;
    consumer_role<NT, KSTEPS>(p, wg, tid, smem, bars, s_gnorm);
  }
}

// KC / 16 for KC in {16, 32, 48, 64} (tc_pick_kc) as a compile-time constant
template <class F>
void dispatch_ksteps(int ksteps, F&& f) {
  switch (ksteps) {
    case 1: f(std::integral_constant<int, 1>{}); break;
    case 2: f(std::integral_constant<int, 2>{}); break;
    case 3: f(std::integral_constant<int, 3>{}); break;
    default: f(std::integral_constant<int, 4>{}); break;
  }
}

template <int NT, int KSTEPS>
int launch_conv_tc(const TcParams& p, int grid, int smem_bytes, cudaStream_t st) {
  static thread_local bool attr_set = false;
  if (!attr_set) {
    B200_CUDA(cudaFuncSetAttribute(conv_tc_kernel<NT, KSTEPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  conv_tc_kernel<NT, KSTEPS><<<grid, kThreads, smem_bytes, st>>>(p);
  B200_CHECK_LAUNCH("conv_tc_kernel");
  return B200SEG_OK;
}

}  // namespace

bool conv3d_tc_shape_ok(int Cin, int Cout, int kd, int kh, int kw, int dtype) {
  if (dtype != B200SEG_F16) return false;
  if (tc_pick_nt(Cout) == 0 || tc_pick_kc(Cin) == 0) return false;
  if (kh > 3 || kw > 3 || kd > 3 || kd < 1 || kh < 1 || kw < 1) return false;
  return true;
}

bool conv3d_fwd_tc_supported(const ConvArgs& a, int dtype) {
  if (!conv3d_tc_shape_ok(a.Cin, a.Cout, a.kd, a.kh, a.kw, dtype)) return false;
  if ((a.x_ld % 8) || (a.x_coff % 8) || (a.y_ld % 8) || (a.y_coff % 8)) return false;
  if (a.res && ((a.r_ld % 8) || (a.r_coff % 8))) return false;
  if (a.gx && ((a.gx_ld % 8) || (a.gx_coff % 8))) return false;
  if ((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.y) | reinterpret_cast<uintptr_t>(a.w)) & 15) return false;
  // the residual / dgrad_x tile is a tensor-TMA box: 16-byte aligned base
  if ((reinterpret_cast<uintptr_t>(a.res) | reinterpret_cast<uintptr_t>(a.gx)) & 15) return false;
  // The transform table of x ([B][Cin], or [Cin] in per-channel mode, <= 32 KB) and, in dgrad mode, the {mean, rstd}
  // table of dgrad_x ([B][Cout], <= 64 KB) live in shared memory; within these limits the planner in conv3d_fwd_tc
  // still fits the side-operand slots and two A and two B stages of the largest tile.  (The InstanceNorm sums of y are
  // kept in registers and need no table.)
  const int nb = a.per_channel ? 1 : a.B;
  if (nb * a.Cin > 4096 || nb * a.Cout > 8192) return false;
  return true;
}

// `a.w` must be the TC weight IMAGE ([ntile][tap][kchunk][KC/8][NT][8], b200seg_pack_weight layout=TC).
int conv3d_fwd_tc(const ConvArgs& a, int dtype, cudaStream_t st) {
  if (!conv3d_fwd_tc_supported(a, dtype)) return B200SEG_EUNSUPPORTED;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.a = a;
  p.wimg = a.w;
  p.KC = tc_pick_kc(a.Cin); p.NKC = a.Cin / p.KC;
  p.NT = tc_pick_nt(a.Cout); p.NTILES = a.Cout / p.NT;
  p.HALO_H = TH + a.kh - 1; p.HALO_W = TW + a.kw - 1;
  p.nvox_h = p.HALO_H * p.HALO_W;
  int slots = p.nvox_h; if ((slots & 1) == 0) slots += 1;     // odd number of 16-B slots -> conflict-free plane stride
  // Operand staging, chosen from the shape alone: RAW inputs (every data-gradient launch) are staged by ONE tensor-TMA
  // box per stage and consumed by the MMA warpgroups straight off the TMA barrier; inputs that need InstanceNorm /
  // activation by a TMA box + in-place transform while Cin <= 64 and at least 4 A stages fit (below), by per-thread
  // cp.async copies + transform otherwise.  When the tensor map cannot be built every input takes the cp.async path.
  const bool raw_input = !a.x_stats && !a.x_affine && a.act == 0;
  p.use_tma = ((raw_input || a.Cin <= 64) &&
               b200seg_make_act_tmap(&p.tm_x, a.x, a.x_ld, a.x_coff, a.Cin, a.B * a.D, a.H, a.W, p.HALO_W, p.HALO_H, p.KC / 8)) ? 1 : 0;
  p.plane_stride = p.use_tma ? p.nvox_h * 16 : slots * 16;    // a TMA box is written densely
  p.a_stage_bytes = (p.KC / 8) * p.plane_stride;
  p.a_stage_bytes = (p.a_stage_bytes + 127) / 128 * 128;      // TMA destinations are 128-byte aligned
  p.b_stage_bytes = p.KC * p.NT * 2;
  p.tiles_h = (a.H + TH - 1) / TH; p.tiles_w = (a.W + TW - 1) / TW;
  int64_t nt = (int64_t)a.B * a.D * p.tiles_h * p.tiles_w * p.NTILES;
  if (nt > 0x7fffffff) return B200SEG_EUNSUPPORTED;
  p.n_tiles = (int)nt;
  // The epilogue's side operand (residual, or dgrad_x behind the activation mask) arrives as one tensor-TMA box
  // {8 ch, TW, TH, NT/8 planes} per tile, zero-filled past the volume edge, in a ring of SS slots.  Narrow tiles
  // (NT <= 64) take only a few hundred clocks of MMAs, so their box is issued two tiles ahead; wider tiles are long
  // enough for one slot.
  if (a.res || a.gx) {
    p.SS = p.NT <= 64 ? 2 : 1;
    p.side_stage_bytes = TH * TW * p.NT * 2;
    const bool ok = a.gx ? b200seg_make_act_tmap(&p.tm_side, a.gx, a.gx_ld, a.gx_coff, a.Cout, a.B * a.D, a.H, a.W, TW, TH, p.NT / 8)
                         : b200seg_make_act_tmap(&p.tm_side, a.res, a.r_ld, a.r_coff, a.Cout, a.B * a.D, a.H, a.W, TW, TH, p.NT / 8);
    if (!ok) return B200SEG_ECUDA;       // conv3d_fwd_tc_supported checked every other condition of the map
  }
  // shared memory carve-up
  p.norm_bstride = a.per_channel ? 0 : a.Cin;
  const int norm_bytes = (a.per_channel ? 1 : a.B) * a.Cin * 8;
  const int gnorm_bytes = a.gx ? a.B * a.Cout * 8 : 0;
  const int side_bytes = p.SS * p.side_stage_bytes;
  const int budget = 227 * 1024 - 1024 - norm_bytes - gnorm_bytes - side_bytes - 512;
  const int64_t w_total = (int64_t)a.kd * a.kh * a.kw * a.Cin * a.Cout * 2;
  int b_region;
  if (w_total <= 112 * 1024 && w_total + 2 * p.a_stage_bytes <= budget) {
    p.w_resident = 1; p.SB = 1;
    b_region = (int)w_total;
    p.SA = (budget - b_region) / p.a_stage_bytes; if (p.SA > 6) p.SA = 6;
  } else {
    p.w_resident = 0;
    p.SA = 4;
    while (p.SA > 2 && p.SA * p.a_stage_bytes + 3 * p.b_stage_bytes > budget) --p.SA;
    p.SB = (budget - p.SA * p.a_stage_bytes) / p.b_stage_bytes; if (p.SB > 8) p.SB = 8;
    if (p.SB < 2) return B200SEG_EUNSUPPORTED;
    b_region = p.SB * p.b_stage_bytes;
  }
  if (p.SA < 2) return B200SEG_EUNSUPPORTED;
  p.prefetch = p.SA - 1 < 3 ? p.SA - 1 : 3;
  if (p.use_tma && !raw_input && p.SA < 4) p.use_tma = 0;       // the TMA + transform loader runs three stages ahead
  int off = 0;
  p.smem_a_off = off; off += p.SA * p.a_stage_bytes;
  off = (off + 127) / 128 * 128;
  p.smem_b_off = off; off += b_region;
  off = (off + 127) / 128 * 128;
  p.smem_side_off = off; off += side_bytes;
  off = (off + 15) / 16 * 16;
  p.smem_bar_off = off; off += (3 * p.SA + 2 * p.SB + 2 * p.SS) * 8;
  off = (off + 15) / 16 * 16;
  p.smem_norm_off = off; off += norm_bytes;
  off = (off + 15) / 16 * 16;
  p.smem_gnorm_off = off; off += gnorm_bytes;
  const int smem_bytes = off + 1024;       // slack for the 1024-B alignment of the dynamic segment
  int grid = p.n_tiles < B200SEG_NUM_SMS ? p.n_tiles : B200SEG_NUM_SMS;
  int rc = B200SEG_OK;
  dispatch_n(p.NT, [&](auto nt) {
    dispatch_ksteps(p.KC / 16, [&](auto ks) { rc = launch_conv_tc<decltype(nt)::value, decltype(ks)::value>(p, grid, smem_bytes, st); });
  });
  return rc;
}
