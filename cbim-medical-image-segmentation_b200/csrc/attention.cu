// attention.cu — global multi-head self-attention, the core of monai 1.1.0's SABlock between its qkv and out_proj
// Linears (UNETR's ViT encoder):  out = softmax(q k^T * dh^-0.5) v  per (batch, head) over all L tokens, dh = 64.
//
// Layout: qkv [B][L][3*inner] with channel which*inner + h*64 + d (SABlock's "b h (qkv l d)" rearrange), out [B][L][inner]
// with channel h*64 + d (its "b h l d -> b l (h d)" rearrange), so both Linears read / write these buffers directly.
// lse and delta are fp32 [B][heads][L]: the row log-sum-exp the forward leaves for the backward, and rowsum(dO * O).
//
// Forward: a CTA owns kBQ = 32 query rows of one (batch, head), one 16-row tile per warp, and streams the keys through
// shared memory in tiles of kBK = 64 with an online softmax, so scores never leave registers and no [B, h, L, L] map
// exists.  Backward (FlashAttention-2 order, deterministic — every output element is written by exactly one thread,
// no atomics): a delta pre-pass, a dK/dV kernel whose CTA owns 32 keys and loops over query tiles, and a dQ kernel
// whose CTA owns 32 queries and loops over key tiles; both recompute P from lse.
//
// fp16 (AMP) path: S = QK^T, PV, dP = dO V^T, dV = P^T dO, dK = dS^T Q and dQ = dS K run as mma.sync m16n8k16 tiles
// (fp16 operands, fp32 accumulation).  The QK^T accumulators, after the fp32 softmax, are re-packed in registers as the
// A operand of the next MMA.  Why mma.sync and not wgmma: wgmma's smallest tile is 64 rows per warpgroup, which would
// make the query tile 64 rows; bcv at B = 2 (L = 216, 12 heads) would then launch 2*12*4 = 96 CTAs on 132 SMs, while
// 32-row tiles of two 16-row warps give 168.  The per-element softmax work between the two GEMMs also keeps each score
// tile in the registers of the warp that made it, which is the natural mma.sync data flow.
// Numerics: scores and softmax statistics are fp32; probabilities are rounded to fp16 before PV, as the reference's
// `einsum(att_mat, v)` does under autocast; the row sum l uses the unrounded values.
//
// fp32 path (no AMP): CUDA-core kernels with one thread per query (forward, dQ) or per key (dK/dV) and the other side
// streamed through shared memory in 64-row tiles; same algorithm, same determinism.
#include "common.cuh"
#include <math.h>

namespace {

constexpr int kDH = 64;                  // head dimension (the only one supported)
constexpr int kBQ = 32;                  // rows a CTA owns (queries: forward / dQ; keys: dK/dV)
constexpr int kBK = 64;                  // rows of the streamed side per shared-memory tile
constexpr int kThreads = 64;             // two warps, 16 rows each
constexpr int kRS = kDH + 8;             // row stride (halves) of row-major tiles: conflict-free fragment reads
constexpr int kTS = kBK + 8;             // row stride (halves) of transposed [dim][token] tiles
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// ------------------------------------------------------------------------------------------------ tensor-core helpers
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack2(float x, float y) {
  __half2 h = __floats2half2_rn(x, y);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t lds32(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t ldg32(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// A fragments (rows ra, rb = ra + 8; all 64 dims as 4 k-steps) straight from global memory; row i of the operand is
// at src + i*ld.  Rows at or past L are zero.
__device__ __forceinline__ void load_a_global(const __half* src, int64_t ld, int ra, int rb, int L, int t, uint32_t (&a)[4][4]) {
  const __half* pa = src + (int64_t)ra * ld + 2 * t;
  const __half* pb = src + (int64_t)rb * ld + 2 * t;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = ra < L ? ldg32(pa + ks * 16) : 0u;
    a[ks][1] = rb < L ? ldg32(pb + ks * 16) : 0u;
    a[ks][2] = ra < L ? ldg32(pa + ks * 16 + 8) : 0u;
    a[ks][3] = rb < L ? ldg32(pb + ks * 16 + 8) : 0u;
  }
}
// acc(16 x 8) += A(16 x 64) * tile[c0 .. c0+8)^T, tile row-major [kBK][kRS]
__device__ __forceinline__ void mma_rows(float (&acc)[4], const uint32_t (&a)[4][4], const __half* tile, int c0, int g, int t) {
  const __half* p = tile + (c0 + g) * kRS + 2 * t;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) mma16816(acc, a[ks], lds32(p + ks * 16), lds32(p + ks * 16 + 8));
}
// acc[nt](16 x 8) += P(16 x 16, packed accumulators) * X[k0 .. k0+16)(16 x 64), X given transposed [kDH][kTS]
__device__ __forceinline__ void mma_cols(float (&acc)[8][4], const uint32_t (&p)[4], const __half* tr, int k0, int g, int t) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const __half* q = tr + (nt * 8 + g) * kTS + k0 + 2 * t;
    mma16816(acc[nt], p, lds32(q), lds32(q + 8));
  }
}
// the 16 x 16 A operand formed by two adjacent 8-column accumulator blocks
__device__ __forceinline__ void pack_a(const float (&s0)[4], const float (&s1)[4], uint32_t (&p)[4]) {
  p[0] = pack2(s0[0], s0[1]); p[1] = pack2(s0[2], s0[3]); p[2] = pack2(s1[0], s1[1]); p[3] = pack2(s1[2], s1[3]);
}

// rows r0 .. r0+kBK of a token-major operand (row i at src + i*ld, 64 halves) -> row-major tile [kBK][kRS]; zero past L
__device__ __forceinline__ void stage_rows(__half* dst, const __half* src, int64_t ld, int r0, int L) {
  for (int c = threadIdx.x; c < kBK * 8; c += kThreads) {
    const int r = c >> 3, ch = c & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < L) v = *reinterpret_cast<const uint4*>(src + (int64_t)(r0 + r) * ld + ch * 8);
    *reinterpret_cast<uint4*>(dst + r * kRS + ch * 8) = v;
  }
}
// the same rows transposed -> [kDH][kTS] (token index fastest across the lanes: conflict-free 2-byte stores)
__device__ __forceinline__ void stage_cols(__half* dst, const __half* src, int64_t ld, int r0, int L) {
  for (int c = threadIdx.x; c < kBK * 8; c += kThreads) {
    const int r = c & (kBK - 1), ch = c / kBK;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < L) v = *reinterpret_cast<const uint4*>(src + (int64_t)(r0 + r) * ld + ch * 8);
    const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[(ch * 8 + i) * kTS + r] = h[i];
  }
}

struct Head {              // pointers of one (batch, head)
  int64_t C, C3;
  const void* q; const void* k; const void* v;     // token i of each at +i*C3
};
template <typename T>
__device__ __forceinline__ Head head_of(const T* qkv, int L, int heads) {
  Head hd;
  hd.C = (int64_t)heads * kDH; hd.C3 = 3 * hd.C;
  const T* base = qkv + (int64_t)blockIdx.z * L * hd.C3 + blockIdx.y * kDH;
  hd.q = base; hd.k = base + hd.C; hd.v = base + 2 * hd.C;
  return hd;
}

// ------------------------------------------------------------------------------------------------ fp16 forward
__global__ void __launch_bounds__(kThreads)
attn_fwd_mma_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, float* __restrict__ lse, int L, int heads, float sl2) {
  __shared__ __align__(16) __half sK[kBK * kRS];
  __shared__ __align__(16) __half sVt[kDH * kTS];
  const Head hd = head_of(qkv, L, heads);
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ra = blockIdx.x * kBQ + (threadIdx.x >> 5) * 16 + g, rb = ra + 8;
  uint32_t aq[4][4];
  load_a_global((const __half*)hd.q, hd.C3, ra, rb, L, t, aq);
  float ma = -INFINITY, mb = -INFINITY, la = 0.f, lb = 0.f;
  float o[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
  for (int k0 = 0; k0 < L; k0 += kBK) {
    __syncthreads();
    stage_rows(sK, (const __half*)hd.k, hd.C3, k0, L);
    stage_cols(sVt, (const __half*)hd.v, hd.C3, k0, L);
    __syncthreads();
    float sc[8][4];
    float mxa = -INFINITY, mxb = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
      mma_rows(sc[n], aq, sK, n * 8, g, t);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool ok = k0 + n * 8 + 2 * t + e < L;
        sc[n][e] = ok ? sc[n][e] * sl2 : -INFINITY;
        sc[n][2 + e] = ok ? sc[n][2 + e] * sl2 : -INFINITY;
        mxa = fmaxf(mxa, sc[n][e]); mxb = fmaxf(mxb, sc[n][2 + e]);
      }
    }
    // key k0 < L is in every tile, so the new maxima are finite
    const float mna = fmaxf(ma, quad_max(mxa)), mnb = fmaxf(mb, quad_max(mxb));
    const float ca = exp2f(ma - mna), cb = exp2f(mb - mnb);
    ma = mna; mb = mnb;
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        sc[n][e] = exp2f(sc[n][e] - mna); sc[n][2 + e] = exp2f(sc[n][2 + e] - mnb);
        sa += sc[n][e]; sb += sc[n][2 + e];
      }
    }
    la = la * ca + sa; lb = lb * cb + sb;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { o[nt][0] *= ca; o[nt][1] *= ca; o[nt][2] *= cb; o[nt][3] *= cb; }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t p[4];
      pack_a(sc[2 * kk], sc[2 * kk + 1], p);
      mma_cols(o, p, sVt, kk * 16, g, t);
    }
  }
  la = quad_sum(la); lb = quad_sum(lb);
  const int64_t ob = (int64_t)blockIdx.z * L;
  const int64_t lb0 = ((int64_t)blockIdx.z * heads + blockIdx.y) * L;
  if (ra < L) {
    const float ia = 1.f / la;
    __half* op = out + (ob + ra) * hd.C + blockIdx.y * kDH + 2 * t;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<__half2*>(op + nt * 8) = __floats2half2_rn(o[nt][0] * ia, o[nt][1] * ia);
    if (t == 0) lse[lb0 + ra] = (ma + log2f(la)) * kLn2;
  }
  if (rb < L) {
    const float ib = 1.f / lb;
    __half* op = out + (ob + rb) * hd.C + blockIdx.y * kDH + 2 * t;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<__half2*>(op + nt * 8) = __floats2half2_rn(o[nt][2] * ib, o[nt][3] * ib);
    if (t == 0) lse[lb0 + rb] = (mb + log2f(lb)) * kLn2;
  }
}

// ------------------------------------------------------------------------------------------------ backward pre-pass
// delta[b][h][i] = <dO_i, O_i> over the head's 64 channels (one thread per (token, head))
template <typename T>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const T* __restrict__ out, const T* __restrict__ dout, float* __restrict__ delta, int B, int L, int heads) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)B * L * heads) return;
  const int h = (int)(idx % heads);
  const int64_t row = idx / heads;
  const int64_t off = row * heads * kDH + h * kDH;
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < kDH / 8; ++c) {
    float o[8], d[8];
    ld8<T>(out + off + c * 8, o);
    ld8<T>(dout + off + c * 8, d);
#pragma unroll
    for (int i = 0; i < 8; ++i) s += o[i] * d[i];
  }
  const int64_t b = row / L, i = row % L;
  delta[(b * heads + h) * L + i] = s;
}

// ------------------------------------------------------------------------------------------------ fp16 dK / dV
// key-stationary: dV_j = sum_i P_ij dO_i, dK_j = scale * sum_i dS_ij q_i, dS = P (dP - delta), dP = dO V^T
__global__ void __launch_bounds__(kThreads)
attn_bwd_dkdv_mma_kernel(const __half* __restrict__ qkv, const __half* __restrict__ dout, const float* __restrict__ lse,
                         const float* __restrict__ delta, __half* __restrict__ dqkv, int L, int heads, float scale, float sl2) {
  __shared__ __align__(16) __half sQ[kBK * kRS];
  __shared__ __align__(16) __half sdO[kBK * kRS];
  __shared__ __align__(16) __half sQt[kDH * kTS];
  __shared__ __align__(16) __half sdOt[kDH * kTS];
  __shared__ float sL[kBK], sD[kBK];
  const Head hd = head_of(qkv, L, heads);
  const __half* dO = dout + (int64_t)blockIdx.z * L * hd.C + blockIdx.y * kDH;
  const int64_t s0 = ((int64_t)blockIdx.z * heads + blockIdx.y) * L;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ja = blockIdx.x * kBQ + (threadIdx.x >> 5) * 16 + g, jb = ja + 8;
  uint32_t ak[4][4], av[4][4];
  load_a_global((const __half*)hd.k, hd.C3, ja, jb, L, t, ak);
  load_a_global((const __half*)hd.v, hd.C3, ja, jb, L, t, av);
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    dk[nt][0] = dk[nt][1] = dk[nt][2] = dk[nt][3] = 0.f;
    dv[nt][0] = dv[nt][1] = dv[nt][2] = dv[nt][3] = 0.f;
  }
  for (int i0 = 0; i0 < L; i0 += kBK) {
    __syncthreads();
    stage_rows(sQ, (const __half*)hd.q, hd.C3, i0, L);
    stage_cols(sQt, (const __half*)hd.q, hd.C3, i0, L);
    stage_rows(sdO, dO, hd.C, i0, L);
    stage_cols(sdOt, dO, hd.C, i0, L);
    for (int r = threadIdx.x; r < kBK; r += kThreads) {
      const bool ok = i0 + r < L;
      sL[r] = ok ? lse[s0 + i0 + r] * kLog2e : INFINITY;      // a query past L gets P = 0
      sD[r] = ok ? delta[s0 + i0 + r] : 0.f;
    }
    __syncthreads();
#pragma unroll 1
    for (int kk = 0; kk < kBK; kk += 16) {                   // 16 queries
      float sc[2][4], dp[2][4], pr[2][4];
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
        dp[n][0] = dp[n][1] = dp[n][2] = dp[n][3] = 0.f;
        mma_rows(sc[n], ak, sQ, kk + n * 8, g, t);            // S^T = K Q^T
        mma_rows(dp[n], av, sdO, kk + n * 8, g, t);           // dP^T = V dO^T
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int r = kk + n * 8 + 2 * t + (e & 1);
          const float p = exp2f(sc[n][e] * sl2 - sL[r]);
          pr[n][e] = p;
          sc[n][e] = p * (dp[n][e] - sD[r]);
        }
      }
      uint32_t pp[4], ps[4];
      pack_a(pr[0], pr[1], pp);
      pack_a(sc[0], sc[1], ps);
      mma_cols(dv, pp, sdOt, kk, g, t);                       // dV += P^T dO
      mma_cols(dk, ps, sQt, kk, g, t);                        // dK += dS^T Q
    }
  }
  __half* base = dqkv + (int64_t)blockIdx.z * L * hd.C3 + blockIdx.y * kDH + 2 * t;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int j = half ? jb : ja;
    if (j >= L) continue;
    __half* p = base + (int64_t)j * hd.C3;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      *reinterpret_cast<__half2*>(p + hd.C + nt * 8) = __floats2half2_rn(dk[nt][2 * half] * scale, dk[nt][2 * half + 1] * scale);
      *reinterpret_cast<__half2*>(p + 2 * hd.C + nt * 8) = __floats2half2_rn(dv[nt][2 * half], dv[nt][2 * half + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ fp16 dQ
// query-stationary: dQ_i = scale * sum_j dS_ij k_j
__global__ void __launch_bounds__(kThreads)
attn_bwd_dq_mma_kernel(const __half* __restrict__ qkv, const __half* __restrict__ dout, const float* __restrict__ lse,
                       const float* __restrict__ delta, __half* __restrict__ dqkv, int L, int heads, float scale, float sl2) {
  __shared__ __align__(16) __half sK[kBK * kRS];
  __shared__ __align__(16) __half sV[kBK * kRS];
  __shared__ __align__(16) __half sKt[kDH * kTS];
  const Head hd = head_of(qkv, L, heads);
  const __half* dO = dout + (int64_t)blockIdx.z * L * hd.C + blockIdx.y * kDH;
  const int64_t s0 = ((int64_t)blockIdx.z * heads + blockIdx.y) * L;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int ra = blockIdx.x * kBQ + (threadIdx.x >> 5) * 16 + g, rb = ra + 8;
  uint32_t aq[4][4], ado[4][4];
  load_a_global((const __half*)hd.q, hd.C3, ra, rb, L, t, aq);
  load_a_global(dO, hd.C, ra, rb, L, t, ado);
  const float lsa = ra < L ? lse[s0 + ra] * kLog2e : INFINITY, lsb = rb < L ? lse[s0 + rb] * kLog2e : INFINITY;
  const float dla = ra < L ? delta[s0 + ra] : 0.f, dlb = rb < L ? delta[s0 + rb] : 0.f;
  float dq[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) dq[nt][0] = dq[nt][1] = dq[nt][2] = dq[nt][3] = 0.f;
  for (int j0 = 0; j0 < L; j0 += kBK) {
    __syncthreads();
    stage_rows(sK, (const __half*)hd.k, hd.C3, j0, L);
    stage_rows(sV, (const __half*)hd.v, hd.C3, j0, L);
    stage_cols(sKt, (const __half*)hd.k, hd.C3, j0, L);
    __syncthreads();
#pragma unroll 1
    for (int kk = 0; kk < kBK; kk += 16) {                   // 16 keys
      float sc[2][4], dp[2][4];
#pragma unroll
      for (int n = 0; n < 2; ++n) {
        sc[n][0] = sc[n][1] = sc[n][2] = sc[n][3] = 0.f;
        dp[n][0] = dp[n][1] = dp[n][2] = dp[n][3] = 0.f;
        mma_rows(sc[n], aq, sK, kk + n * 8, g, t);            // S = Q K^T
        mma_rows(dp[n], ado, sV, kk + n * 8, g, t);           // dP = dO V^T
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = j0 + kk + n * 8 + 2 * t + e < L;
          const float pa = ok ? exp2f(sc[n][e] * sl2 - lsa) : 0.f, pb = ok ? exp2f(sc[n][2 + e] * sl2 - lsb) : 0.f;
          sc[n][e] = pa * (dp[n][e] - dla);
          sc[n][2 + e] = pb * (dp[n][2 + e] - dlb);
        }
      }
      uint32_t ps[4];
      pack_a(sc[0], sc[1], ps);
      mma_cols(dq, ps, sKt, kk, g, t);                        // dQ += dS K
    }
  }
  __half* base = dqkv + (int64_t)blockIdx.z * L * hd.C3 + blockIdx.y * kDH + 2 * t;
  if (ra < L) {
    __half* p = base + (int64_t)ra * hd.C3;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<__half2*>(p + nt * 8) = __floats2half2_rn(dq[nt][0] * scale, dq[nt][1] * scale);
  }
  if (rb < L) {
    __half* p = base + (int64_t)rb * hd.C3;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) *reinterpret_cast<__half2*>(p + nt * 8) = __floats2half2_rn(dq[nt][2] * scale, dq[nt][3] * scale);
  }
}

// ------------------------------------------------------------------------------------------------ fp32 (CUDA cores)
constexpr int kOS = kDH + 1;             // padded row stride (floats) of the per-thread rows: conflict-free

// rows r0 .. r0+kBK of a token-major fp32 operand -> [kBK][ds] (zero past L)
__device__ __forceinline__ void stage_f32(float* dst, int ds, const float* src, int64_t ld, int r0, int L) {
  for (int c = threadIdx.x; c < kBK * (kDH / 4); c += kThreads) {
    const int r = c / (kDH / 4), ch = c % (kDH / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r0 + r < L) v = *reinterpret_cast<const float4*>(src + (int64_t)(r0 + r) * ld + ch * 4);
    float* d = dst + r * ds + ch * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
}

// one thread per query row; keys and values streamed through shared memory
__global__ void __launch_bounds__(kThreads)
attn_fwd_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, float* __restrict__ lse, int L, int heads, float sl2) {
  __shared__ __align__(16) float sK[kBK * kDH];
  __shared__ __align__(16) float sV[kBK * kDH];
  const Head hd = head_of(qkv, L, heads);
  const int i = blockIdx.x * kBK + threadIdx.x;
  float q[kDH], o[kDH];
#pragma unroll
  for (int d = 0; d < kDH; ++d) { q[d] = i < L ? ((const float*)hd.q)[(int64_t)i * hd.C3 + d] * sl2 : 0.f; o[d] = 0.f; }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < L; k0 += kBK) {
    __syncthreads();
    stage_f32(sK, kDH, (const float*)hd.k, hd.C3, k0, L);
    stage_f32(sV, kDH, (const float*)hd.v, hd.C3, k0, L);
    __syncthreads();
    const int n = min(kBK, L - k0);
    for (int j = 0; j < n; ++j) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < kDH; ++d) s += q[d] * sK[j * kDH + d];
      if (s > m) {                                    // rescale only when the running maximum moves
        const float c = exp2f(m - s);
        l *= c;
#pragma unroll
        for (int d = 0; d < kDH; ++d) o[d] *= c;
        m = s;
      }
      const float p = exp2f(s - m);
      l += p;
#pragma unroll
      for (int d = 0; d < kDH; ++d) o[d] += p * sV[j * kDH + d];
    }
  }
  if (i >= L) return;
  const float il = 1.f / l;
  float* op = out + ((int64_t)blockIdx.z * L + i) * hd.C + blockIdx.y * kDH;
#pragma unroll
  for (int d = 0; d < kDH; d += 4) *reinterpret_cast<float4*>(op + d) = make_float4(o[d] * il, o[d + 1] * il, o[d + 2] * il, o[d + 3] * il);
  lse[((int64_t)blockIdx.z * heads + blockIdx.y) * L + i] = (m + log2f(l)) * kLn2;
}

// dynamic shared memory of the two fp32 backward kernels: own rows [kBK][kOS] x 2, streamed rows [kBK][kDH] x 2, 2 x kBK
constexpr size_t kSmemBwdF32 = sizeof(float) * (2 * kBK * kOS + 2 * kBK * kDH + 2 * kBK);

// one thread per key: dV_j = sum_i P_ij dO_i, dK_j = scale * sum_i dS_ij q_i
__global__ void __launch_bounds__(kThreads)
attn_bwd_dkdv_f32_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                         const float* __restrict__ delta, float* __restrict__ dqkv, int L, int heads, float scale, float sl2) {
  extern __shared__ __align__(16) float smf[];
  float* sKo = smf;                        // this CTA's keys, one row per thread
  float* sVo = sKo + kBK * kOS;
  float* sQ = sVo + kBK * kOS;
  float* sdO = sQ + kBK * kDH;
  float* sL = sdO + kBK * kDH;
  float* sD = sL + kBK;
  const Head hd = head_of(qkv, L, heads);
  const float* dO = dout + (int64_t)blockIdx.z * L * hd.C + blockIdx.y * kDH;
  const int64_t s0 = ((int64_t)blockIdx.z * heads + blockIdx.y) * L;
  const int j0 = blockIdx.x * kBK, j = j0 + threadIdx.x;
  stage_f32(sKo, kOS, (const float*)hd.k, hd.C3, j0, L);
  stage_f32(sVo, kOS, (const float*)hd.v, hd.C3, j0, L);
  const float* kj = sKo + threadIdx.x * kOS;
  const float* vj = sVo + threadIdx.x * kOS;
  float dk[kDH], dv[kDH];
#pragma unroll
  for (int d = 0; d < kDH; ++d) dk[d] = dv[d] = 0.f;
  for (int i0 = 0; i0 < L; i0 += kBK) {
    __syncthreads();
    stage_f32(sQ, kDH, (const float*)hd.q, hd.C3, i0, L);
    stage_f32(sdO, kDH, dO, hd.C, i0, L);
    for (int r = threadIdx.x; r < kBK; r += kThreads) {
      const bool ok = i0 + r < L;
      sL[r] = ok ? lse[s0 + i0 + r] * kLog2e : 0.f;
      sD[r] = ok ? delta[s0 + i0 + r] : 0.f;
    }
    __syncthreads();
    const int n = min(kBK, L - i0);
    for (int r = 0; r < n; ++r) {
      const float* qi = sQ + r * kDH;
      const float* gi = sdO + r * kDH;
      float s = 0.f, dp = 0.f;
#pragma unroll 8
      for (int d = 0; d < kDH; ++d) { s += kj[d] * qi[d]; dp += vj[d] * gi[d]; }
      const float p = exp2f(s * sl2 - sL[r]);
      const float ds = p * (dp - sD[r]);
#pragma unroll
      for (int d = 0; d < kDH; ++d) { dv[d] += p * gi[d]; dk[d] += ds * qi[d]; }
    }
  }
  if (j >= L) return;
  float* p = dqkv + ((int64_t)blockIdx.z * L + j) * hd.C3 + blockIdx.y * kDH;
#pragma unroll
  for (int d = 0; d < kDH; d += 4) {
    *reinterpret_cast<float4*>(p + hd.C + d) = make_float4(dk[d] * scale, dk[d + 1] * scale, dk[d + 2] * scale, dk[d + 3] * scale);
    *reinterpret_cast<float4*>(p + 2 * hd.C + d) = make_float4(dv[d], dv[d + 1], dv[d + 2], dv[d + 3]);
  }
}

// one thread per query: dQ_i = scale * sum_j dS_ij k_j
__global__ void __launch_bounds__(kThreads)
attn_bwd_dq_f32_kernel(const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ lse,
                       const float* __restrict__ delta, float* __restrict__ dqkv, int L, int heads, float scale, float sl2) {
  extern __shared__ __align__(16) float smf[];
  float* sQo = smf;                        // this CTA's queries and their output gradients, one row per thread
  float* sGo = sQo + kBK * kOS;
  float* sK = sGo + kBK * kOS;
  float* sV = sK + kBK * kDH;
  const Head hd = head_of(qkv, L, heads);
  const float* dO = dout + (int64_t)blockIdx.z * L * hd.C + blockIdx.y * kDH;
  const int64_t s0 = ((int64_t)blockIdx.z * heads + blockIdx.y) * L;
  const int i0 = blockIdx.x * kBK, i = i0 + threadIdx.x;
  stage_f32(sQo, kOS, (const float*)hd.q, hd.C3, i0, L);
  stage_f32(sGo, kOS, dO, hd.C, i0, L);
  const float* qi = sQo + threadIdx.x * kOS;
  const float* gi = sGo + threadIdx.x * kOS;
  const float ls = i < L ? lse[s0 + i] * kLog2e : 0.f, dl = i < L ? delta[s0 + i] : 0.f;
  float dq[kDH];
#pragma unroll
  for (int d = 0; d < kDH; ++d) dq[d] = 0.f;
  for (int j0 = 0; j0 < L; j0 += kBK) {
    __syncthreads();
    stage_f32(sK, kDH, (const float*)hd.k, hd.C3, j0, L);
    stage_f32(sV, kDH, (const float*)hd.v, hd.C3, j0, L);
    __syncthreads();
    const int n = min(kBK, L - j0);
    for (int r = 0; r < n; ++r) {
      const float* kj = sK + r * kDH;
      const float* vj = sV + r * kDH;
      float s = 0.f, dp = 0.f;
#pragma unroll 8
      for (int d = 0; d < kDH; ++d) { s += qi[d] * kj[d]; dp += gi[d] * vj[d]; }
      const float ds = exp2f(s * sl2 - ls) * (dp - dl);
#pragma unroll
      for (int d = 0; d < kDH; ++d) dq[d] += ds * kj[d];
    }
  }
  if (i >= L) return;
  float* p = dqkv + ((int64_t)blockIdx.z * L + i) * hd.C3 + blockIdx.y * kDH;
#pragma unroll
  for (int d = 0; d < kDH; d += 4) *reinterpret_cast<float4*>(p + d) = make_float4(dq[d] * scale, dq[d + 1] * scale, dq[d + 2] * scale, dq[d + 3] * scale);
}

int check_args(const void* a, const void* b, const void* c, int B, int L, int heads, int dim_head, int dtype) {
  if (!a || !b || !c || B <= 0 || L <= 0 || heads <= 0) return B200SEG_EINVAL;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  if (dim_head != kDH) return B200SEG_EUNSUPPORTED;
  if (B > 65535 || heads > 65535) return B200SEG_EUNSUPPORTED;          // grid.z / grid.y
  return B200SEG_OK;
}
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" int b200seg_attention_fwd(const void* qkv, void* out, float* lse, int B, int L, int heads, int dim_head, int dtype,
                                     void* stream) {
  const int rc = check_args(qkv, out, lse, B, L, heads, dim_head, dtype);
  if (rc) return rc;
  if (!aligned16(qkv) || !aligned16(out)) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  const float scale = 1.f / sqrtf((float)kDH), sl2 = scale * kLog2e;
  if (dtype == B200SEG_F16) {
    attn_fwd_mma_kernel<<<dim3(ceil_div(L, kBQ), heads, B), kThreads, 0, st>>>((const __half*)qkv, (__half*)out, lse, L, heads, sl2);
    B200_CHECK_LAUNCH("attn_fwd_mma_kernel");
  } else {
    attn_fwd_f32_kernel<<<dim3(ceil_div(L, kBK), heads, B), kThreads, 0, st>>>((const float*)qkv, (float*)out, lse, L, heads, sl2);
    B200_CHECK_LAUNCH("attn_fwd_f32_kernel");
  }
  return B200SEG_OK;
}

extern "C" int b200seg_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                                     void* dqkv, int B, int L, int heads, int dim_head, int dtype, void* stream) {
  int rc = check_args(qkv, out, dout, B, L, heads, dim_head, dtype);
  if (rc) return rc;
  if (!lse || !delta || !dqkv) return B200SEG_EINVAL;
  if (!aligned16(qkv) || !aligned16(out) || !aligned16(dout) || !aligned16(dqkv)) return B200SEG_EINVAL;
  cudaStream_t st = as_stream(stream);
  const float scale = 1.f / sqrtf((float)kDH), sl2 = scale * kLog2e;
  const int64_t rows = (int64_t)B * L * heads;
  const int nb = (int)((rows + 255) / 256);
  if (dtype == B200SEG_F16) {
    attn_delta_kernel<__half><<<nb, 256, 0, st>>>((const __half*)out, (const __half*)dout, delta, B, L, heads);
    B200_CHECK_LAUNCH("attn_delta_kernel");
    const dim3 grid(ceil_div(L, kBQ), heads, B);
    attn_bwd_dkdv_mma_kernel<<<grid, kThreads, 0, st>>>((const __half*)qkv, (const __half*)dout, lse, delta, (__half*)dqkv, L, heads, scale, sl2);
    B200_CHECK_LAUNCH("attn_bwd_dkdv_mma_kernel");
    attn_bwd_dq_mma_kernel<<<grid, kThreads, 0, st>>>((const __half*)qkv, (const __half*)dout, lse, delta, (__half*)dqkv, L, heads, scale, sl2);
    B200_CHECK_LAUNCH("attn_bwd_dq_mma_kernel");
  } else {
    attn_delta_kernel<float><<<nb, 256, 0, st>>>((const float*)out, (const float*)dout, delta, B, L, heads);
    B200_CHECK_LAUNCH("attn_delta_kernel");
    B200_CUDA(cudaFuncSetAttribute(attn_bwd_dkdv_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBwdF32));
    B200_CUDA(cudaFuncSetAttribute(attn_bwd_dq_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBwdF32));
    const dim3 grid(ceil_div(L, kBK), heads, B);
    attn_bwd_dkdv_f32_kernel<<<grid, kThreads, kSmemBwdF32, st>>>((const float*)qkv, (const float*)dout, lse, delta, (float*)dqkv, L, heads, scale, sl2);
    B200_CHECK_LAUNCH("attn_bwd_dkdv_f32_kernel");
    attn_bwd_dq_f32_kernel<<<grid, kThreads, kSmemBwdF32, st>>>((const float*)qkv, (const float*)dout, lse, delta, (float*)dqkv, L, heads, scale, sl2);
    B200_CHECK_LAUNCH("attn_bwd_dq_f32_kernel");
  }
  return B200SEG_OK;
}
