// biattn.cu — MedFormer's bidirectional multi-head attention core (B-MHA), fused, forward and backward.
// Reference: BidirectionAttention.forward, model/dim3/medformer_utils.py:63-97 — the part between the q/v
// projections and the output projections:
//     S  = scale * einsum('bhid,bhjd->bhij', feat_q, map_q)            (:77-78)    i in N voxels, j in M map tokens
//     A1 = softmax(S, dim=-1) ; A2 = softmax(S, dim=-2)                (:80,82)
//     feat_out = A1 @ map_v ; map_out = A2^T @ feat_v                  (:84,89)
// The reference materialises S, A1, A2 as [B,h,N,M] fp32 tensors plus six relayout copies; here every voxel is
// visited ONCE per direction: the M<=32 map tokens live in shared memory, the row softmax is thread-local, the
// column softmax (over up to 55k voxels) is an online max/sum with per-block partials merged by a tiny kernel,
// and in the backward the column term  c_j = sum_i A2_ij dA2_ij  collapses to  <dmap_out_j, map_out_j>, so the
// backward is a single pass over N as well.  HBM-bound: fwd reads q_f, v_f and writes out_f (3*B*N*inner*s bytes).
// Channel convention (rearrange1, :43-51): channel c of the `inner` block = d * heads + h.
#include "common.cuh"

namespace {

constexpr int kT = 128;           // voxels per block (one per thread)
constexpr int MAXM_CAP = 64;      // map tokens: 27 (BCV 3x3x3) run the 32-row build, 64 (4x4x4 maps) the 64-row one
constexpr int DH = 32;            // head dimension (all BASELINE MedFormer levels use 32)

struct BiArgs {
  const void* fq; int fq_ld, fq_coff;
  const void* fv; int fv_ld, fv_coff;
  const void* mq; const void* mv; int m_ld;        // [B][M][m_ld], q at +0.., channel = d*heads + h
  int mq_coff, mv_coff;
  void* fo; int fo_ld, fo_coff;
  void* mo; int mo_ld, mo_coff;
  float* colstat;                                  // [B][heads][M][2] = {max, sum} of the column softmax
  float* partial;                                  // fwd: [B][heads][nblk][M][2+DH]; bwd: [B][heads][nblk][M][2*DH]
  // backward only
  const void* dfo; int dfo_ld, dfo_coff;
  const void* dmo; int dmo_ld, dmo_coff;
  void* dfq; int dfq_ld, dfq_coff;
  void* dfv; int dfv_ld, dfv_coff;
  void* dmq; void* dmv; int dm_ld, dmq_coff, dmv_coff;
  int B, M, heads; int64_t N; float scale;
};

constexpr int VFS = DH + 4;        // row stride of the staged value tile: 16-byte aligned rows

__device__ __forceinline__ float dot4(float q0, float q1, float q2, float q3, const float4& w, float acc) {
  return fmaf(q0, w.x, fmaf(q1, w.y, fmaf(q2, w.z, fmaf(q3, w.w, acc))));
}

// The map-side operands live in shared memory zero-padded to MAXM rows (MAXM = 32 or 64: BCV's 27 tokens / the
// 64 of the 4x4x4 maps), so the token loops run unpredicated with one broadcast LDS.128 per four FMAs; padded
// tokens get S = -inf after the contraction.
template <typename T, int MAXM>
__global__ void __launch_bounds__(kT)
biattn_fwd_kernel(BiArgs a) {
  extern __shared__ float sm[];
  float* s_qm = sm;                       // [MAXM][DH] (pre-scaled, rows >= M zero)
  float* s_vm = s_qm + MAXM * DH;         // [MAXM][DH]
  float* s_e = s_vm + MAXM * DH;          // [kT][MAXM+1]
  float* s_vf = s_e + kT * (MAXM + 1);    // [kT][VFS]
  float* s_cmax = s_vf + kT * VFS;        // [4 warps][MAXM] then [MAXM]
  const int h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int o = tid; o < MAXM * DH; o += kT) {
    const int j = o / DH, d = o % DH;
    float q = 0.f, v = 0.f;
    if (j < M) {
      const int64_t off = ((int64_t)b * M + j) * a.m_ld + d * heads + h;
      q = Elem<T>::ld((const T*)a.mq + off + a.mq_coff) * a.scale;
      v = Elem<T>::ld((const T*)a.mv + off + a.mv_coff);
    }
    s_qm[o] = q; s_vm[o] = v;
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * kT + tid;
  const bool valid = i < a.N;
  float S[MAXM];
#pragma unroll
  for (int j = 0; j < MAXM; ++j) S[j] = 0.f;
  float* my_v = s_vf + tid * VFS;
  if (valid) {
    const T* qp = (const T*)a.fq + ((int64_t)b * a.N + i) * a.fq_ld + a.fq_coff + h;
    const T* vp = (const T*)a.fv + ((int64_t)b * a.N + i) * a.fv_ld + a.fv_coff + h;
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      const float q0 = Elem<T>::ld(qp + d0 * heads), q1 = Elem<T>::ld(qp + (d0 + 1) * heads);
      const float q2 = Elem<T>::ld(qp + (d0 + 2) * heads), q3 = Elem<T>::ld(qp + (d0 + 3) * heads);
      *reinterpret_cast<float4*>(my_v + d0) = make_float4(Elem<T>::ld(vp + d0 * heads), Elem<T>::ld(vp + (d0 + 1) * heads),
                                                          Elem<T>::ld(vp + (d0 + 2) * heads), Elem<T>::ld(vp + (d0 + 3) * heads));
#pragma unroll
      for (int j = 0; j < MAXM; ++j) S[j] = dot4(q0, q1, q2, q3, *reinterpret_cast<const float4*>(s_qm + j * DH + d0), S[j]);
    }
#pragma unroll
    for (int j = 0; j < MAXM; ++j) if (j >= M) S[j] = -INFINITY;
  } else {
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) *reinterpret_cast<float4*>(my_v + d0) = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < MAXM; ++j) S[j] = -INFINITY;
  }
  // ---- column direction first (it needs the raw scores): block max per token, exp into shared memory
#pragma unroll
  for (int j = 0; j < MAXM; ++j) {
    float mj = S[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mj = fmaxf(mj, __shfl_xor_sync(0xffffffffu, mj, o));
    if (lane == 0) s_cmax[wid * MAXM + j] = mj;
  }
  __syncthreads();
  if (tid < MAXM) {
    float mj = s_cmax[tid];
    for (int w = 1; w < kT / 32; ++w) mj = fmaxf(mj, s_cmax[w * MAXM + tid]);
    s_cmax[4 * MAXM + tid] = mj;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < MAXM; ++j) {
    const float cm = s_cmax[4 * MAXM + j];
    s_e[tid * (MAXM + 1) + j] = (cm == -INFINITY) ? 0.f : __expf(S[j] - cm);      // padded tokens / empty blocks
  }
  // ---- row softmax over the map tokens (probabilities overwrite the scores) + feat_out
  if (valid) {
    float m = -INFINITY;
#pragma unroll
    for (int j = 0; j < MAXM; ++j) m = fmaxf(m, S[j]);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAXM; ++j) { S[j] = __expf(S[j] - m); sum += S[j]; }
    const float inv = 1.f / sum;
    T* op = (T*)a.fo + ((int64_t)b * a.N + i) * a.fo_ld + a.fo_coff + h;
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < MAXM; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(s_vm + j * DH + d0);
        o.x = fmaf(S[j], w.x, o.x); o.y = fmaf(S[j], w.y, o.y); o.z = fmaf(S[j], w.z, o.z); o.w = fmaf(S[j], w.w, o.w);
      }
      Elem<T>::st(op + d0 * heads, o.x * inv); Elem<T>::st(op + (d0 + 1) * heads, o.y * inv);
      Elem<T>::st(op + (d0 + 2) * heads, o.z * inv); Elem<T>::st(op + (d0 + 3) * heads, o.w * inv);
    }
  }
  __syncthreads();
  // 128 threads = 32 tokens x 4 channel octets; each accumulates its 1x8 patch of E^T V over the block's voxels
  const int nblk = gridDim.x;
  float* pb = a.partial + ((((int64_t)b * heads + h) * nblk + blockIdx.x) * M) * (2 + DH);
  const int dg = (tid & 3) * 8;
#pragma unroll
  for (int jh = 0; jh < MAXM; jh += 32) {
    const int j = jh + (tid >> 2);
    float acc[8], esum = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
#pragma unroll 4
    for (int r = 0; r < kT; ++r) {
      const float e = s_e[r * (MAXM + 1) + j];
      const float4 v0 = *reinterpret_cast<const float4*>(s_vf + r * VFS + dg), v1 = *reinterpret_cast<const float4*>(s_vf + r * VFS + dg + 4);
      esum += e;
      acc[0] = fmaf(e, v0.x, acc[0]); acc[1] = fmaf(e, v0.y, acc[1]); acc[2] = fmaf(e, v0.z, acc[2]); acc[3] = fmaf(e, v0.w, acc[3]);
      acc[4] = fmaf(e, v1.x, acc[4]); acc[5] = fmaf(e, v1.y, acc[5]); acc[6] = fmaf(e, v1.z, acc[6]); acc[7] = fmaf(e, v1.w, acc[7]);
    }
    if (j < M) {
#pragma unroll
      for (int c = 0; c < 8; ++c) pb[j * (2 + DH) + 2 + dg + c] = acc[c];
      if (dg == 0) { pb[j * (2 + DH)] = s_cmax[4 * MAXM + j]; pb[j * (2 + DH) + 1] = esum; }
    }
  }
}

// merge the per-block column partials: map_out[j][:] and the {max, sum} the backward needs.
// grid (M, heads, B), 128 threads = 4 partitions of the block axis x 32 head channels, online-softmax combine.
template <typename T>
__global__ void biattn_fwd_merge_kernel(BiArgs a, int nblk) {
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int d = threadIdx.x & 31, part = threadIdx.x >> 5;
  const float* pb = a.partial + ((((int64_t)b * heads + h) * nblk) * M + j) * (2 + DH);
  float m = -INFINITY, sum = 0.f, acc = 0.f;
  for (int k = part; k < nblk; k += 4) {
    const float* q = pb + (int64_t)k * M * (2 + DH);
    const float mk = q[0];
    if (mk > m) { const float sc = __expf(m - mk); sum *= sc; acc *= sc; m = mk; }
    const float e = __expf(mk - m);
    sum = fmaf(q[1], e, sum); acc = fmaf(q[2 + d], e, acc);
  }
  __shared__ float s_m[4], s_s[4], s_a[4][DH];
  if (d == 0) { s_m[part] = m; s_s[part] = sum; }
  s_a[part][d] = acc;
  __syncthreads();
  if (part == 0) {
    const float gm = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float gs = 0.f, ga = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) { const float e = __expf(s_m[p] - gm); gs = fmaf(s_s[p], e, gs); ga = fmaf(s_a[p][d], e, ga); }
    Elem<T>::st((T*)a.mo + ((int64_t)b * M + j) * a.mo_ld + a.mo_coff + d * heads + h, ga / gs);
    if (d == 0) { float* cs = a.colstat + (((int64_t)b * heads + h) * M + j) * 2; cs[0] = gm; cs[1] = gs; }
  }
}

template <typename T, int MAXM>
__global__ void __launch_bounds__(kT)
biattn_bwd_kernel(BiArgs a) {
  extern __shared__ float sm[];
  float* s_qm = sm;                        // [MAXM][DH]  (unscaled; rows >= M zero)
  float* s_vm = s_qm + MAXM * DH;
  float* s_dmo = s_vm + MAXM * DH;         // [MAXM][DH]
  float* s_col = s_dmo + MAXM * DH;        // [MAXM][4] = {gmax, 1/gsum, c_j, -}
  float* s_p1 = s_col + MAXM * 4;          // [kT][MAXM+1]
  float* s_ds = s_p1 + kT * (MAXM + 1);    // [kT][MAXM+1]
  float* s_do = s_ds + kT * (MAXM + 1);    // [kT][VFS]
  float* s_q = s_do + kT * VFS;            // [kT][VFS]
  const int h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int tid = threadIdx.x;
  for (int o = tid; o < MAXM * DH; o += kT) {
    const int j = o / DH, d = o % DH;
    float q = 0.f, v = 0.f, g = 0.f;
    if (j < M) {
      const int64_t off = ((int64_t)b * M + j) * a.m_ld + d * heads + h;
      q = Elem<T>::ld((const T*)a.mq + off + a.mq_coff);
      v = Elem<T>::ld((const T*)a.mv + off + a.mv_coff);
      g = Elem<T>::ld((const T*)a.dmo + ((int64_t)b * M + j) * a.dmo_ld + a.dmo_coff + d * heads + h);
    }
    s_qm[o] = q; s_vm[o] = v; s_dmo[o] = g;
  }
  __syncthreads();
  if (tid < MAXM) {
    float g0 = 0.f, g1 = 0.f, c = 0.f;
    if (tid < M) {
      const float* cs = a.colstat + (((int64_t)b * heads + h) * M + tid) * 2;
      for (int d = 0; d < DH; ++d)
        c = fmaf(s_dmo[tid * DH + d], Elem<T>::ld((const T*)a.mo + ((int64_t)b * M + tid) * a.mo_ld + a.mo_coff + d * heads + h), c);
      g0 = cs[0]; g1 = 1.f / cs[1];
    }
    s_col[tid * 4] = g0; s_col[tid * 4 + 1] = g1; s_col[tid * 4 + 2] = c;
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * kT + tid;
  const bool valid = i < a.N;
  float S[MAXM], v[DH];
  float* my_q = s_q + tid * VFS;           // own rows double as register relief; re-read below without a barrier
  float* my_do = s_do + tid * VFS;
#pragma unroll
  for (int j = 0; j < MAXM; ++j) S[j] = 0.f;
  if (valid) {
    const int64_t row = (int64_t)b * a.N + i;
    const T* qp = (const T*)a.fq + row * a.fq_ld + a.fq_coff + h;
    const T* vp = (const T*)a.fv + row * a.fv_ld + a.fv_coff + h;
    const T* gp = (const T*)a.dfo + row * a.dfo_ld + a.dfo_coff + h;
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      const float q0 = Elem<T>::ld(qp + d0 * heads), q1 = Elem<T>::ld(qp + (d0 + 1) * heads);
      const float q2 = Elem<T>::ld(qp + (d0 + 2) * heads), q3 = Elem<T>::ld(qp + (d0 + 3) * heads);
#pragma unroll
      for (int u = 0; u < 4; ++u) v[d0 + u] = Elem<T>::ld(vp + (d0 + u) * heads);
      *reinterpret_cast<float4*>(my_q + d0) = make_float4(q0, q1, q2, q3);
      *reinterpret_cast<float4*>(my_do + d0) = make_float4(Elem<T>::ld(gp + d0 * heads), Elem<T>::ld(gp + (d0 + 1) * heads),
                                                           Elem<T>::ld(gp + (d0 + 2) * heads), Elem<T>::ld(gp + (d0 + 3) * heads));
#pragma unroll
      for (int j = 0; j < MAXM; ++j) S[j] = dot4(q0, q1, q2, q3, *reinterpret_cast<const float4*>(s_qm + j * DH + d0), S[j]);
    }
  } else {
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      *reinterpret_cast<float4*>(my_q + d0) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(my_do + d0) = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 4; ++u) v[d0 + u] = 0.f;
    }
  }
  // row softmax: p1_j = exp(S_j - m) * inv is recomputed where needed (keeps MAXM registers free for 64 tokens)
  float dS[MAXM];
  float m = -INFINITY, inv = 0.f;
  {
#pragma unroll
    for (int j = 0; j < MAXM; ++j) { S[j] = (j < M && valid) ? S[j] * a.scale : -INFINITY; m = fmaxf(m, S[j]); dS[j] = 0.f; }
    if (!valid) m = 0.f;                   // keeps exp(S - m) = exp(-inf) = 0 instead of NaN for padding threads
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < MAXM; ++j) sum += __expf(S[j] - m);
    inv = valid ? 1.f / sum : 0.f;
    // dA1_j = <dO, Vm_j>
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      const float4 g = *reinterpret_cast<const float4*>(my_do + d0);
#pragma unroll
      for (int j = 0; j < MAXM; ++j) dS[j] = dot4(g.x, g.y, g.z, g.w, *reinterpret_cast<const float4*>(s_vm + j * DH + d0), dS[j]);
    }
    float t1 = 0.f;
#pragma unroll
    for (int j = 0; j < MAXM; ++j) t1 = fmaf(__expf(S[j] - m) * inv, dS[j], t1);
#pragma unroll
    for (int j = 0; j < MAXM; ++j) dS[j] = __expf(S[j] - m) * inv * (dS[j] - t1);
  }
  // column direction: p2_ij = exp(S_ij - gmax_j) / gsum_j ; dS += p2 (dA2 - c_j) ; dVf = sum_j p2 dmo_j
  float dv[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) dv[d] = 0.f;
#pragma unroll
  for (int j = 0; j < MAXM; ++j) {
    const float p2 = __expf(S[j] - s_col[j * 4]) * s_col[j * 4 + 1];       // 0 for padded tokens / invalid voxels
    float dA2 = 0.f;
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      const float4 w = *reinterpret_cast<const float4*>(s_dmo + j * DH + d0);
      dA2 = dot4(v[d0], v[d0 + 1], v[d0 + 2], v[d0 + 3], w, dA2);
      dv[d0] = fmaf(p2, w.x, dv[d0]); dv[d0 + 1] = fmaf(p2, w.y, dv[d0 + 1]);
      dv[d0 + 2] = fmaf(p2, w.z, dv[d0 + 2]); dv[d0 + 3] = fmaf(p2, w.w, dv[d0 + 3]);
    }
    dS[j] += p2 * (dA2 - s_col[j * 4 + 2]);
  }
  if (valid) {
    const int64_t row = (int64_t)b * a.N + i;
    T* dqp = (T*)a.dfq + row * a.dfq_ld + a.dfq_coff + h;
    T* dvp = (T*)a.dfv + row * a.dfv_ld + a.dfv_coff + h;
#pragma unroll
    for (int d0 = 0; d0 < DH; d0 += 4) {
      float4 dq = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < MAXM; ++j) {
        const float4 w = *reinterpret_cast<const float4*>(s_qm + j * DH + d0);
        dq.x = fmaf(dS[j], w.x, dq.x); dq.y = fmaf(dS[j], w.y, dq.y); dq.z = fmaf(dS[j], w.z, dq.z); dq.w = fmaf(dS[j], w.w, dq.w);
      }
      Elem<T>::st(dqp + d0 * heads, dq.x * a.scale); Elem<T>::st(dqp + (d0 + 1) * heads, dq.y * a.scale);
      Elem<T>::st(dqp + (d0 + 2) * heads, dq.z * a.scale); Elem<T>::st(dqp + (d0 + 3) * heads, dq.w * a.scale);
#pragma unroll
      for (int u = 0; u < 4; ++u) Elem<T>::st(dvp + (d0 + u) * heads, dv[d0 + u]);
    }
  }
  // block partials of the map-side gradients: dVm[j][d] = sum_i p1_ij dO_i[d] ; dQm[j][d] = scale sum_i dS_ij q_i[d]
#pragma unroll
  for (int j = 0; j < MAXM; ++j) { s_p1[tid * (MAXM + 1) + j] = __expf(S[j] - m) * inv; s_ds[tid * (MAXM + 1) + j] = dS[j]; }
  __syncthreads();
  const int nblk = gridDim.x;
  float* pb = a.partial + ((((int64_t)b * heads + h) * nblk + blockIdx.x) * M) * (2 * DH);
  const int dg = (tid & 3) * 8;                        // 32 tokens x 4 channel octets per pass, 1x8 register patch each
#pragma unroll
  for (int jh = 0; jh < MAXM; jh += 32) {
    const int j = jh + (tid >> 2);
    float av[8], aq[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) { av[c] = 0.f; aq[c] = 0.f; }
#pragma unroll 2
    for (int r = 0; r < kT; ++r) {
      const float pp = s_p1[r * (MAXM + 1) + j], dd = s_ds[r * (MAXM + 1) + j];
      const float4 g0 = *reinterpret_cast<const float4*>(s_do + r * VFS + dg), g1 = *reinterpret_cast<const float4*>(s_do + r * VFS + dg + 4);
      const float4 q0 = *reinterpret_cast<const float4*>(s_q + r * VFS + dg), q1 = *reinterpret_cast<const float4*>(s_q + r * VFS + dg + 4);
      av[0] = fmaf(pp, g0.x, av[0]); av[1] = fmaf(pp, g0.y, av[1]); av[2] = fmaf(pp, g0.z, av[2]); av[3] = fmaf(pp, g0.w, av[3]);
      av[4] = fmaf(pp, g1.x, av[4]); av[5] = fmaf(pp, g1.y, av[5]); av[6] = fmaf(pp, g1.z, av[6]); av[7] = fmaf(pp, g1.w, av[7]);
      aq[0] = fmaf(dd, q0.x, aq[0]); aq[1] = fmaf(dd, q0.y, aq[1]); aq[2] = fmaf(dd, q0.z, aq[2]); aq[3] = fmaf(dd, q0.w, aq[3]);
      aq[4] = fmaf(dd, q1.x, aq[4]); aq[5] = fmaf(dd, q1.y, aq[5]); aq[6] = fmaf(dd, q1.z, aq[6]); aq[7] = fmaf(dd, q1.w, aq[7]);
    }
    if (j < M) {
#pragma unroll
      for (int c = 0; c < 8; ++c) { pb[j * 2 * DH + dg + c] = aq[c] * a.scale; pb[j * 2 * DH + DH + dg + c] = av[c]; }
    }
  }
}

template <typename T>
__global__ void biattn_bwd_merge_kernel(BiArgs a, int nblk) {
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int c = threadIdx.x & 63, part = threadIdx.x >> 6;            // 64 values (dq | dv) x 4 partitions
  const float* pb = a.partial + ((((int64_t)b * heads + h) * nblk) * M + j) * (2 * DH);
  float acc = 0.f;
  for (int k = part; k < nblk; k += 4) acc += pb[(int64_t)k * M * (2 * DH) + c];
  __shared__ float s_a[4][2 * DH];
  s_a[part][c] = acc;
  __syncthreads();
  if (part == 0) {
    const float v = s_a[0][c] + s_a[1][c] + s_a[2][c] + s_a[3][c];
    const int d = c & 31;
    const int64_t off = ((int64_t)b * M + j) * a.dm_ld + d * heads + h;
    if (c < DH) Elem<T>::st((T*)a.dmq + off + a.dmq_coff, v);
    else Elem<T>::st((T*)a.dmv + off + a.dmv_coff, v);
  }
}

}  // namespace

extern "C" size_t b200seg_biattn_workspace(int B, int64_t N, int M, int heads) {
  const int64_t nblk = (N + kT - 1) / kT;
  return (size_t)B * heads * nblk * M * (2 * DH) * sizeof(float);
}

static int check_args(int B, int64_t N, int M, int heads, int dim_head, int dtype) {
  if (B <= 0 || N <= 0 || M <= 0 || heads <= 0) return B200SEG_EINVAL;
  if (dim_head != DH || M > MAXM_CAP) return B200SEG_EUNSUPPORTED;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  if ((N + kT - 1) / kT > 65535 * 1024) return B200SEG_EUNSUPPORTED;
  return B200SEG_OK;
}

extern "C" int b200seg_biattn_fwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                                  const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                                  void* fo, int fo_ld, int fo_coff, void* mo, int mo_ld, int mo_coff,
                                  float* colstat, float* workspace, int B, int64_t N, int M, int heads, int dim_head,
                                  float scale, int dtype, void* stream) {
  int rc = check_args(B, N, M, heads, dim_head, dtype);
  if (rc) return rc;
  if (!fq || !fv || !mq || !mv || !fo || !mo || !colstat || !workspace) return B200SEG_EINVAL;
  BiArgs a; memset(&a, 0, sizeof(a));
  a.fq = fq; a.fq_ld = fq_ld; a.fq_coff = fq_coff; a.fv = fv; a.fv_ld = fv_ld; a.fv_coff = fv_coff;
  a.mq = mq; a.mv = mv; a.m_ld = m_ld; a.mq_coff = mq_coff; a.mv_coff = mv_coff;
  a.fo = fo; a.fo_ld = fo_ld; a.fo_coff = fo_coff; a.mo = mo; a.mo_ld = mo_ld; a.mo_coff = mo_coff;
  a.colstat = colstat; a.partial = workspace; a.B = B; a.N = N; a.M = M; a.heads = heads; a.scale = scale;
  cudaStream_t st = as_stream(stream);
  const int nblk = (int)((N + kT - 1) / kT);
  dim3 grid(nblk, heads, B);
  const int MM = M <= 32 ? 32 : 64;
  const size_t sm = sizeof(float) * (2 * MM * DH + kT * (MM + 1) + kT * VFS + 5 * MM);
#define B200_BIATTN_FWD(TT, MMM)                                                                              \
  do {                                                                                                        \
    B200_CUDA(cudaFuncSetAttribute(biattn_fwd_kernel<TT, MMM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); \
    biattn_fwd_kernel<TT, MMM><<<grid, kT, sm, st>>>(a);                                                      \
    biattn_fwd_merge_kernel<TT><<<dim3(M, heads, B), 128, 0, st>>>(a, nblk);                                  \
  } while (0)
  if (dtype == B200SEG_F16) { if (MM == 32) B200_BIATTN_FWD(__half, 32); else B200_BIATTN_FWD(__half, 64); }
  else { if (MM == 32) B200_BIATTN_FWD(float, 32); else B200_BIATTN_FWD(float, 64); }
#undef B200_BIATTN_FWD
  B200_CHECK_LAUNCH("biattn_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_biattn_bwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                                  const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                                  const void* mo, int mo_ld, int mo_coff, const float* colstat,
                                  const void* dfo, int dfo_ld, int dfo_coff, const void* dmo, int dmo_ld, int dmo_coff,
                                  void* dfq, int dfq_ld, int dfq_coff, void* dfv, int dfv_ld, int dfv_coff,
                                  void* dmq, int dmq_coff, void* dmv, int dmv_coff, int dm_ld,
                                  float* workspace, int B, int64_t N, int M, int heads, int dim_head, float scale,
                                  int dtype, void* stream) {
  int rc = check_args(B, N, M, heads, dim_head, dtype);
  if (rc) return rc;
  if (!fq || !fv || !mq || !mv || !mo || !colstat || !dfo || !dmo || !dfq || !dfv || !dmq || !dmv || !workspace) return B200SEG_EINVAL;
  BiArgs a; memset(&a, 0, sizeof(a));
  a.fq = fq; a.fq_ld = fq_ld; a.fq_coff = fq_coff; a.fv = fv; a.fv_ld = fv_ld; a.fv_coff = fv_coff;
  a.mq = mq; a.mv = mv; a.m_ld = m_ld; a.mq_coff = mq_coff; a.mv_coff = mv_coff;
  a.mo = const_cast<void*>(mo); a.mo_ld = mo_ld; a.mo_coff = mo_coff; a.colstat = const_cast<float*>(colstat);
  a.dfo = dfo; a.dfo_ld = dfo_ld; a.dfo_coff = dfo_coff; a.dmo = dmo; a.dmo_ld = dmo_ld; a.dmo_coff = dmo_coff;
  a.dfq = dfq; a.dfq_ld = dfq_ld; a.dfq_coff = dfq_coff; a.dfv = dfv; a.dfv_ld = dfv_ld; a.dfv_coff = dfv_coff;
  a.dmq = dmq; a.dmv = dmv; a.dm_ld = dm_ld; a.dmq_coff = dmq_coff; a.dmv_coff = dmv_coff;
  a.partial = workspace; a.B = B; a.N = N; a.M = M; a.heads = heads; a.scale = scale;
  cudaStream_t st = as_stream(stream);
  const int nblk = (int)((N + kT - 1) / kT);
  dim3 grid(nblk, heads, B);
  const int MM = M <= 32 ? 32 : 64;
  const size_t sm = sizeof(float) * (3 * MM * DH + 4 * MM + 2 * kT * (MM + 1) + 2 * kT * VFS);
#define B200_BIATTN_BWD(TT, MMM)                                                                              \
  do {                                                                                                        \
    B200_CUDA(cudaFuncSetAttribute(biattn_bwd_kernel<TT, MMM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); \
    biattn_bwd_kernel<TT, MMM><<<grid, kT, sm, st>>>(a);                                                      \
    biattn_bwd_merge_kernel<TT><<<dim3(M, heads, B), 256, 0, st>>>(a, nblk);                                  \
  } while (0)
  if (dtype == B200SEG_F16) { if (MM == 32) B200_BIATTN_BWD(__half, 32); else B200_BIATTN_BWD(__half, 64); }
  else { if (MM == 32) B200_BIATTN_BWD(float, 32); else B200_BIATTN_BWD(float, 64); }
#undef B200_BIATTN_BWD
  B200_CHECK_LAUNCH("biattn_bwd");
  return B200SEG_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Wide B-MHA: dim_head 32 / 64 / 80 over up to 80 map tokens (ACDC's 2x6x6 = 72 maps at dim_head 32, 64 and 80),
// for every shape the entry points above refuse.  The one-voxel-per-thread layout above keeps S[M], v[DH] and dv[DH]
// in registers, which spills at 80 x 80.  Here a block owns WT = 64 voxels and every operand lives in shared memory:
// the voxel tiles [WT][DH], the map operands [MP][DH] (zero-padded to MP = 80 tokens) and the score-shaped tiles
// [WT][MP].  Each contraction is a small register-tiled product between two of them (20 or 25 accumulators per thread),
// so no thread holds a dim_head- or token-long array.  The column softmax and its merge are those of the kernels above.
namespace {

constexpr int WT = 64;             // voxels per block
constexpr int WTHREADS = 256;
constexpr int MP = 80;             // map-token rows of the shared operands
constexpr int SLD = MP + 1;        // row stride of the score-shaped tiles (odd: conflict-free per-voxel rows)

template <int DH> struct WideCfg {
  static constexpr int LD = DH + 4;                  // row stride of the [*][DH] tiles: 16-byte rows
  static constexpr int NW = DH / 4;                  // channels per thread in the voxel-major products
  static constexpr int CW = DH / 16;                 // channels per thread in the token-major products
};

// out[i][j] = alpha * <A_i, B_j> for the WT voxels x MP tokens; thread = (voxel i, a warp-uniform group of 20 tokens)
template <int DH>
__device__ __forceinline__ void wide_nt(const float* A, const float* Bm, float* out, float alpha) {
  constexpr int LD = WideCfg<DH>::LD;
  const int i = threadIdx.x & (WT - 1), j0 = (threadIdx.x >> 6) * 20;
  float acc[20];
#pragma unroll
  for (int t = 0; t < 20; ++t) acc[t] = 0.f;
#pragma unroll 2
  for (int d0 = 0; d0 < DH; d0 += 4) {
    const float4 a = *reinterpret_cast<const float4*>(A + i * LD + d0);
#pragma unroll
    for (int t = 0; t < 20; ++t) acc[t] = dot4(a.x, a.y, a.z, a.w, *reinterpret_cast<const float4*>(Bm + (j0 + t) * LD + d0), acc[t]);
  }
#pragma unroll
  for (int t = 0; t < 20; ++t) out[i * SLD + j0 + t] = acc[t] * alpha;
}

// acc[c] = sum_{j<M} P[i][j] * Bm[j][d0 + c] for the thread's voxel i = tid % WT and channels d0 = (tid / WT) * NW ..
template <int DH>
__device__ __forceinline__ void wide_nn(const float* P, const float* Bm, int M, float (&acc)[WideCfg<DH>::NW]) {
  constexpr int LD = WideCfg<DH>::LD, NW = WideCfg<DH>::NW;
  const int i = threadIdx.x & (WT - 1), d0 = (threadIdx.x >> 6) * NW;
#pragma unroll
  for (int c = 0; c < NW; ++c) acc[c] = 0.f;
  for (int j = 0; j < M; ++j) {
    const float p = P[i * SLD + j];
#pragma unroll
    for (int c = 0; c < NW; c += 4) {
      const float4 w = *reinterpret_cast<const float4*>(Bm + j * LD + d0 + c);
      acc[c] = fmaf(p, w.x, acc[c]); acc[c + 1] = fmaf(p, w.y, acc[c + 1]);
      acc[c + 2] = fmaf(p, w.z, acc[c + 2]); acc[c + 3] = fmaf(p, w.w, acc[c + 3]);
    }
  }
}

// acc[t][c] = sum_{i<WT} P[i][j0 + t] * X[i][d0 + c]; thread = (5 tokens j0 = (tid / 16) * 5, CW channels d0 = (tid % 16) * CW)
template <int DH>
__device__ __forceinline__ void wide_tn(const float* P, const float* X, float (&acc)[5][WideCfg<DH>::CW]) {
  constexpr int LD = WideCfg<DH>::LD, CW = WideCfg<DH>::CW;
  const int j0 = (threadIdx.x >> 4) * 5, d0 = (threadIdx.x & 15) * CW;
#pragma unroll
  for (int t = 0; t < 5; ++t)
#pragma unroll
    for (int c = 0; c < CW; ++c) acc[t][c] = 0.f;
#pragma unroll 2
  for (int i = 0; i < WT; ++i) {
    float p[5], x[CW];
#pragma unroll
    for (int t = 0; t < 5; ++t) p[t] = P[i * SLD + j0 + t];
#pragma unroll
    for (int c = 0; c < CW; ++c) x[c] = X[i * LD + d0 + c];
#pragma unroll
    for (int t = 0; t < 5; ++t)
#pragma unroll
      for (int c = 0; c < CW; ++c) acc[t][c] = fmaf(p[t], x[c], acc[t][c]);
  }
}

// [rows][DH] operand rows r < nrows of channel d*heads + h, scaled; rows >= nrows (and the stride padding) zero
template <typename T, int DH>
__device__ __forceinline__ void wide_stage(float* dst, int rows, const T* src, int64_t row0, int64_t ld, int nrows,
                                           int heads, int h, float alpha) {
  constexpr int LD = WideCfg<DH>::LD;
  for (int o = threadIdx.x; o < rows * LD; o += WTHREADS) {
    const int r = o / LD, d = o % LD;
    dst[o] = (r < nrows && d < DH) ? Elem<T>::ld(src + (row0 + r) * ld + d * heads + h) * alpha : 0.f;
  }
}

template <typename T, int DH>
__global__ void __launch_bounds__(WTHREADS)
biattn_wide_fwd_kernel(BiArgs a) {
  using C = WideCfg<DH>;
  extern __shared__ float sm[];
  float* s_qm = sm;                        // [MP][LD] pre-scaled map queries
  float* s_vm = s_qm + MP * C::LD;         // [MP][LD]
  float* s_qf = s_vm + MP * C::LD;         // [WT][LD]
  float* s_vf = s_qf + WT * C::LD;         // [WT][LD]
  float* s_s = s_vf + WT * C::LD;          // [WT][SLD] scores, then the row softmax
  float* s_e = s_s + WT * SLD;             // [WT][SLD] exp(S - block column max)
  float* s_cmax = s_e + WT * SLD;          // [MP]
  float* s_row = s_cmax + MP;              // [WT][2] row max, 1 / row sum
  const int h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads, tid = threadIdx.x;
  const int64_t i0 = (int64_t)blockIdx.x * WT;
  const int nv = (int)min((int64_t)WT, a.N - i0);
  wide_stage<T, DH>(s_qm, MP, (const T*)a.mq + a.mq_coff, (int64_t)b * M, a.m_ld, M, heads, h, a.scale);
  wide_stage<T, DH>(s_vm, MP, (const T*)a.mv + a.mv_coff, (int64_t)b * M, a.m_ld, M, heads, h, 1.f);
  wide_stage<T, DH>(s_qf, WT, (const T*)a.fq + a.fq_coff, (int64_t)b * a.N + i0, a.fq_ld, nv, heads, h, 1.f);
  wide_stage<T, DH>(s_vf, WT, (const T*)a.fv + a.fv_coff, (int64_t)b * a.N + i0, a.fv_ld, nv, heads, h, 1.f);
  __syncthreads();
  wide_nt<DH>(s_qf, s_qm, s_s, 1.f);
  __syncthreads();
  if (tid < M) {                                            // column max over the block's voxels
    float m = -INFINITY;
    for (int i = 0; i < nv; ++i) m = fmaxf(m, s_s[i * SLD + tid]);
    s_cmax[tid] = m;
  } else if (tid >= 128 && tid < 128 + nv) {                // row softmax statistics
    const int i = tid - 128;
    float m = -INFINITY, sum = 0.f;
    for (int j = 0; j < M; ++j) m = fmaxf(m, s_s[i * SLD + j]);
    for (int j = 0; j < M; ++j) sum += __expf(s_s[i * SLD + j] - m);
    s_row[2 * i] = m; s_row[2 * i + 1] = 1.f / sum;
  }
  __syncthreads();
  for (int o = tid; o < WT * MP; o += WTHREADS) {
    const int i = o / MP, j = o % MP;
    const bool ok = i < nv && j < M;
    const float s = s_s[i * SLD + j];
    s_e[i * SLD + j] = ok ? __expf(s - s_cmax[j]) : 0.f;
    s_s[i * SLD + j] = ok ? __expf(s - s_row[2 * i]) * s_row[2 * i + 1] : 0.f;
  }
  __syncthreads();
  {
    float acc[C::NW];
    wide_nn<DH>(s_s, s_vm, M, acc);
    const int i = tid & (WT - 1), d0 = (tid >> 6) * C::NW;
    if (i < nv) {
      T* op = (T*)a.fo + ((int64_t)b * a.N + i0 + i) * a.fo_ld + a.fo_coff + h;
#pragma unroll
      for (int c = 0; c < C::NW; ++c) Elem<T>::st(op + (d0 + c) * heads, acc[c]);
    }
  }
  {
    float acc[5][C::CW];
    wide_tn<DH>(s_e, s_vf, acc);
    const int nblk = gridDim.x, j0 = (tid >> 4) * 5, d0 = (tid & 15) * C::CW;
    float* pb = a.partial + ((((int64_t)b * heads + h) * nblk + blockIdx.x) * M) * (2 + DH);
#pragma unroll
    for (int t = 0; t < 5; ++t)
      if (j0 + t < M)
#pragma unroll
        for (int c = 0; c < C::CW; ++c) pb[(j0 + t) * (2 + DH) + 2 + d0 + c] = acc[t][c];
    if (tid < M) {
      float esum = 0.f;
      for (int i = 0; i < nv; ++i) esum += s_e[i * SLD + tid];
      pb[tid * (2 + DH)] = s_cmax[tid]; pb[tid * (2 + DH) + 1] = esum;
    }
  }
}

// the forward merge of biattn_fwd_merge_kernel for DH channels: 4 partitions of the block axis x 32 lanes, each lane
// owning channels lane, lane + 32, lane + 64 (< DH)
template <typename T, int DH>
__global__ void biattn_wide_fwd_merge_kernel(BiArgs a, int nblk) {
  constexpr int NC = (DH + 31) / 32;
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int lane = threadIdx.x & 31, part = threadIdx.x >> 5;
  const float* pb = a.partial + ((((int64_t)b * heads + h) * nblk) * M + j) * (2 + DH);
  float m = -INFINITY, sum = 0.f, acc[NC];
#pragma unroll
  for (int u = 0; u < NC; ++u) acc[u] = 0.f;
  for (int k = part; k < nblk; k += 4) {
    const float* q = pb + (int64_t)k * M * (2 + DH);
    const float mk = q[0];
    if (mk > m) {
      const float sc = __expf(m - mk);
      sum *= sc;
#pragma unroll
      for (int u = 0; u < NC; ++u) acc[u] *= sc;
      m = mk;
    }
    const float e = __expf(mk - m);
    sum = fmaf(q[1], e, sum);
#pragma unroll
    for (int u = 0; u < NC; ++u) if (lane + 32 * u < DH) acc[u] = fmaf(q[2 + lane + 32 * u], e, acc[u]);
  }
  __shared__ float s_m[4], s_s[4], s_a[4][NC * 32];
  if (lane == 0) { s_m[part] = m; s_s[part] = sum; }
#pragma unroll
  for (int u = 0; u < NC; ++u) s_a[part][lane + 32 * u] = acc[u];
  __syncthreads();
  if (part == 0) {
    const float gm = fmaxf(fmaxf(s_m[0], s_m[1]), fmaxf(s_m[2], s_m[3]));
    float gs = 0.f, ga[NC];
#pragma unroll
    for (int u = 0; u < NC; ++u) ga[u] = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const float e = __expf(s_m[p] - gm);
      gs = fmaf(s_s[p], e, gs);
#pragma unroll
      for (int u = 0; u < NC; ++u) ga[u] = fmaf(s_a[p][lane + 32 * u], e, ga[u]);
    }
#pragma unroll
    for (int u = 0; u < NC; ++u) {
      const int d = lane + 32 * u;
      if (d < DH) Elem<T>::st((T*)a.mo + ((int64_t)b * M + j) * a.mo_ld + a.mo_coff + d * heads + h, ga[u] / gs);
    }
    if (lane == 0) { float* cs = a.colstat + (((int64_t)b * heads + h) * M + j) * 2; cs[0] = gm; cs[1] = gs; }
  }
}

template <typename T, int DH>
__global__ void __launch_bounds__(WTHREADS)
biattn_wide_bwd_kernel(BiArgs a) {
  using C = WideCfg<DH>;
  extern __shared__ float sm[];
  float* s_qm = sm;                        // [MP][LD] (unscaled)
  float* s_vm = s_qm + MP * C::LD;
  float* s_dmo = s_vm + MP * C::LD;
  float* s_qf = s_dmo + MP * C::LD;        // [WT][LD]
  float* s_vf = s_qf + WT * C::LD;
  float* s_do = s_vf + WT * C::LD;
  float* s_p1 = s_do + WT * C::LD;         // [WT][SLD] scores, then the row softmax p1
  float* s_ds = s_p1 + WT * SLD;           // [WT][SLD] dA1, then dS
  float* s_p2 = s_ds + WT * SLD;           // [WT][SLD] dA2, then the column softmax p2
  float* s_col = s_p2 + WT * SLD;          // [MP][3] gmax, 1 / gsum, c_j
  float* s_row = s_col + 3 * MP;           // [WT][3] row max, 1 / row sum, t1
  const int h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads, tid = threadIdx.x;
  const int64_t i0 = (int64_t)blockIdx.x * WT, row0 = (int64_t)b * a.N + i0;
  const int nv = (int)min((int64_t)WT, a.N - i0);
  wide_stage<T, DH>(s_qm, MP, (const T*)a.mq + a.mq_coff, (int64_t)b * M, a.m_ld, M, heads, h, 1.f);
  wide_stage<T, DH>(s_vm, MP, (const T*)a.mv + a.mv_coff, (int64_t)b * M, a.m_ld, M, heads, h, 1.f);
  wide_stage<T, DH>(s_dmo, MP, (const T*)a.dmo + a.dmo_coff, (int64_t)b * M, a.dmo_ld, M, heads, h, 1.f);
  wide_stage<T, DH>(s_qf, WT, (const T*)a.fq + a.fq_coff, row0, a.fq_ld, nv, heads, h, 1.f);
  wide_stage<T, DH>(s_vf, WT, (const T*)a.fv + a.fv_coff, row0, a.fv_ld, nv, heads, h, 1.f);
  wide_stage<T, DH>(s_do, WT, (const T*)a.dfo + a.dfo_coff, row0, a.dfo_ld, nv, heads, h, 1.f);
  __syncthreads();
  if (tid < M) {                           // c_j = <dmap_out_j, map_out_j>
    const float* cs = a.colstat + (((int64_t)b * heads + h) * M + tid) * 2;
    const T* mo = (const T*)a.mo + ((int64_t)b * M + tid) * a.mo_ld + a.mo_coff + h;
    float c = 0.f;
    for (int d = 0; d < DH; ++d) c = fmaf(s_dmo[tid * C::LD + d], Elem<T>::ld(mo + d * heads), c);
    s_col[3 * tid] = cs[0]; s_col[3 * tid + 1] = 1.f / cs[1]; s_col[3 * tid + 2] = c;
  }
  wide_nt<DH>(s_qf, s_qm, s_p1, a.scale);  // S
  wide_nt<DH>(s_do, s_vm, s_ds, 1.f);      // dA1_ij = <dO_i, Vm_j>
  wide_nt<DH>(s_vf, s_dmo, s_p2, 1.f);     // dA2_ij = <Vf_i, dmo_j>
  __syncthreads();
  if (tid < nv) {
    float m = -INFINITY, sum = 0.f, t1 = 0.f;
    for (int j = 0; j < M; ++j) m = fmaxf(m, s_p1[tid * SLD + j]);
    for (int j = 0; j < M; ++j) {
      const float e = __expf(s_p1[tid * SLD + j] - m);
      sum += e; t1 = fmaf(e, s_ds[tid * SLD + j], t1);
    }
    s_row[3 * tid] = m; s_row[3 * tid + 1] = 1.f / sum; s_row[3 * tid + 2] = t1 / sum;
  }
  __syncthreads();
  for (int o = tid; o < WT * MP; o += WTHREADS) {
    const int i = o / MP, j = o % MP;
    float p1 = 0.f, p2 = 0.f, ds = 0.f;
    if (i < nv && j < M) {
      const float s = s_p1[i * SLD + j];
      p1 = __expf(s - s_row[3 * i]) * s_row[3 * i + 1];
      p2 = __expf(s - s_col[3 * j]) * s_col[3 * j + 1];
      ds = p1 * (s_ds[i * SLD + j] - s_row[3 * i + 2]) + p2 * (s_p2[i * SLD + j] - s_col[3 * j + 2]);
    }
    s_p1[i * SLD + j] = p1; s_p2[i * SLD + j] = p2; s_ds[i * SLD + j] = ds;
  }
  __syncthreads();
  {
    const int i = tid & (WT - 1), d0 = (tid >> 6) * C::NW;
    float acc[C::NW];
    wide_nn<DH>(s_ds, s_qm, M, acc);       // dQf = scale * dS Qm
    if (i < nv) {
      T* p = (T*)a.dfq + (row0 + i) * a.dfq_ld + a.dfq_coff + h;
#pragma unroll
      for (int c = 0; c < C::NW; ++c) Elem<T>::st(p + (d0 + c) * heads, acc[c] * a.scale);
    }
    wide_nn<DH>(s_p2, s_dmo, M, acc);      // dVf = p2 dmo
    if (i < nv) {
      T* p = (T*)a.dfv + (row0 + i) * a.dfv_ld + a.dfv_coff + h;
#pragma unroll
      for (int c = 0; c < C::NW; ++c) Elem<T>::st(p + (d0 + c) * heads, acc[c]);
    }
  }
  {
    const int nblk = gridDim.x, j0 = (tid >> 4) * 5, d0 = (tid & 15) * C::CW;
    float* pb = a.partial + ((((int64_t)b * heads + h) * nblk + blockIdx.x) * M) * (2 * DH);
    float acc[5][C::CW];
    wide_tn<DH>(s_ds, s_qf, acc);          // dQm partial = scale * dS^T Qf
#pragma unroll
    for (int t = 0; t < 5; ++t)
      if (j0 + t < M)
#pragma unroll
        for (int c = 0; c < C::CW; ++c) pb[(j0 + t) * 2 * DH + d0 + c] = acc[t][c] * a.scale;
    wide_tn<DH>(s_p1, s_do, acc);          // dVm partial = p1^T dO
#pragma unroll
    for (int t = 0; t < 5; ++t)
      if (j0 + t < M)
#pragma unroll
        for (int c = 0; c < C::CW; ++c) pb[(j0 + t) * 2 * DH + DH + d0 + c] = acc[t][c];
  }
}

// sum of the per-block map-gradient partials in block order: 4 partitions x 64 lanes, lane owning values
// lane, lane + 64, lane + 128 (< 2 * DH) of [dq | dv]
template <typename T, int DH>
__global__ void biattn_wide_bwd_merge_kernel(BiArgs a, int nblk) {
  constexpr int NC = (2 * DH + 63) / 64;
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z, M = a.M, heads = a.heads;
  const int lane = threadIdx.x & 63, part = threadIdx.x >> 6;
  const float* pb = a.partial + ((((int64_t)b * heads + h) * nblk) * M + j) * (2 * DH);
  float acc[NC];
#pragma unroll
  for (int u = 0; u < NC; ++u) acc[u] = 0.f;
  for (int k = part; k < nblk; k += 4)
#pragma unroll
    for (int u = 0; u < NC; ++u) if (lane + 64 * u < 2 * DH) acc[u] += pb[(int64_t)k * M * (2 * DH) + lane + 64 * u];
  __shared__ float s_a[4][NC * 64];
#pragma unroll
  for (int u = 0; u < NC; ++u) s_a[part][lane + 64 * u] = acc[u];
  __syncthreads();
  if (part == 0) {
#pragma unroll
    for (int u = 0; u < NC; ++u) {
      const int c = lane + 64 * u;
      if (c >= 2 * DH) continue;
      const float v = s_a[0][c] + s_a[1][c] + s_a[2][c] + s_a[3][c];
      const int d = c < DH ? c : c - DH;
      const int64_t off = ((int64_t)b * M + j) * a.dm_ld + d * heads + h;
      if (c < DH) Elem<T>::st((T*)a.dmq + off + a.dmq_coff, v);
      else Elem<T>::st((T*)a.dmv + off + a.dmv_coff, v);
    }
  }
}

template <int DH> constexpr size_t wide_fwd_smem() { return sizeof(float) * (2 * MP * WideCfg<DH>::LD + 2 * WT * WideCfg<DH>::LD + 2 * WT * SLD + MP + 2 * WT); }
template <int DH> constexpr size_t wide_bwd_smem() { return sizeof(float) * (3 * MP * WideCfg<DH>::LD + 3 * WT * WideCfg<DH>::LD + 3 * WT * SLD + 3 * MP + 3 * WT); }

}  // namespace

// the shapes b200seg_biattn_fwd / _bwd do not take: dim_head 32 with 65..80 tokens, dim_head 64 / 80 with 1..80
static int check_wide_args(int B, int64_t N, int M, int heads, int dim_head, int dtype) {
  if (B <= 0 || N <= 0 || M <= 0 || heads <= 0) return B200SEG_EINVAL;
  if (dtype != B200SEG_F16 && dtype != B200SEG_F32) return B200SEG_EINVAL;
  if (dim_head != 32 && dim_head != 64 && dim_head != 80) return B200SEG_EUNSUPPORTED;
  if (M > MP || (dim_head == DH && M <= MAXM_CAP)) return B200SEG_EUNSUPPORTED;
  if ((N + WT - 1) / WT > 2147483647LL || heads > 65535 || B > 65535) return B200SEG_EUNSUPPORTED;
  return B200SEG_OK;
}

extern "C" size_t b200seg_biattn_wide_workspace(int B, int64_t N, int M, int heads, int dim_head) {
  const int64_t nblk = (N + WT - 1) / WT;
  return (size_t)B * heads * nblk * M * (2 * dim_head) * sizeof(float);
}

extern "C" int b200seg_biattn_wide_fwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                                       const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                                       void* fo, int fo_ld, int fo_coff, void* mo, int mo_ld, int mo_coff,
                                       float* colstat, float* workspace, int B, int64_t N, int M, int heads,
                                       int dim_head, float scale, int dtype, void* stream) {
  int rc = check_wide_args(B, N, M, heads, dim_head, dtype);
  if (rc) return rc;
  if (!fq || !fv || !mq || !mv || !fo || !mo || !colstat || !workspace) return B200SEG_EINVAL;
  BiArgs a; memset(&a, 0, sizeof(a));
  a.fq = fq; a.fq_ld = fq_ld; a.fq_coff = fq_coff; a.fv = fv; a.fv_ld = fv_ld; a.fv_coff = fv_coff;
  a.mq = mq; a.mv = mv; a.m_ld = m_ld; a.mq_coff = mq_coff; a.mv_coff = mv_coff;
  a.fo = fo; a.fo_ld = fo_ld; a.fo_coff = fo_coff; a.mo = mo; a.mo_ld = mo_ld; a.mo_coff = mo_coff;
  a.colstat = colstat; a.partial = workspace; a.B = B; a.N = N; a.M = M; a.heads = heads; a.scale = scale;
  cudaStream_t st = as_stream(stream);
  const int nblk = (int)((N + WT - 1) / WT);
  dim3 grid(nblk, heads, B);
#define B200_WIDE_FWD(TT, D)                                                                                   \
  do {                                                                                                         \
    constexpr size_t sm = wide_fwd_smem<D>();                                                                  \
    B200_CUDA(cudaFuncSetAttribute(biattn_wide_fwd_kernel<TT, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); \
    biattn_wide_fwd_kernel<TT, D><<<grid, WTHREADS, sm, st>>>(a);                                              \
    biattn_wide_fwd_merge_kernel<TT, D><<<dim3(M, heads, B), 128, 0, st>>>(a, nblk);                           \
  } while (0)
#define B200_WIDE_FWD_T(TT) \
  do { if (dim_head == 32) B200_WIDE_FWD(TT, 32); else if (dim_head == 64) B200_WIDE_FWD(TT, 64); else B200_WIDE_FWD(TT, 80); } while (0)
  if (dtype == B200SEG_F16) B200_WIDE_FWD_T(__half); else B200_WIDE_FWD_T(float);
#undef B200_WIDE_FWD_T
#undef B200_WIDE_FWD
  B200_CHECK_LAUNCH("biattn_wide_fwd");
  return B200SEG_OK;
}

extern "C" int b200seg_biattn_wide_bwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                                       const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                                       const void* mo, int mo_ld, int mo_coff, const float* colstat,
                                       const void* dfo, int dfo_ld, int dfo_coff, const void* dmo, int dmo_ld, int dmo_coff,
                                       void* dfq, int dfq_ld, int dfq_coff, void* dfv, int dfv_ld, int dfv_coff,
                                       void* dmq, int dmq_coff, void* dmv, int dmv_coff, int dm_ld,
                                       float* workspace, int B, int64_t N, int M, int heads, int dim_head, float scale,
                                       int dtype, void* stream) {
  int rc = check_wide_args(B, N, M, heads, dim_head, dtype);
  if (rc) return rc;
  if (!fq || !fv || !mq || !mv || !mo || !colstat || !dfo || !dmo || !dfq || !dfv || !dmq || !dmv || !workspace) return B200SEG_EINVAL;
  BiArgs a; memset(&a, 0, sizeof(a));
  a.fq = fq; a.fq_ld = fq_ld; a.fq_coff = fq_coff; a.fv = fv; a.fv_ld = fv_ld; a.fv_coff = fv_coff;
  a.mq = mq; a.mv = mv; a.m_ld = m_ld; a.mq_coff = mq_coff; a.mv_coff = mv_coff;
  a.mo = const_cast<void*>(mo); a.mo_ld = mo_ld; a.mo_coff = mo_coff; a.colstat = const_cast<float*>(colstat);
  a.dfo = dfo; a.dfo_ld = dfo_ld; a.dfo_coff = dfo_coff; a.dmo = dmo; a.dmo_ld = dmo_ld; a.dmo_coff = dmo_coff;
  a.dfq = dfq; a.dfq_ld = dfq_ld; a.dfq_coff = dfq_coff; a.dfv = dfv; a.dfv_ld = dfv_ld; a.dfv_coff = dfv_coff;
  a.dmq = dmq; a.dmv = dmv; a.dm_ld = dm_ld; a.dmq_coff = dmq_coff; a.dmv_coff = dmv_coff;
  a.partial = workspace; a.B = B; a.N = N; a.M = M; a.heads = heads; a.scale = scale;
  cudaStream_t st = as_stream(stream);
  const int nblk = (int)((N + WT - 1) / WT);
  dim3 grid(nblk, heads, B);
#define B200_WIDE_BWD(TT, D)                                                                                   \
  do {                                                                                                         \
    constexpr size_t sm = wide_bwd_smem<D>();                                                                  \
    B200_CUDA(cudaFuncSetAttribute(biattn_wide_bwd_kernel<TT, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); \
    biattn_wide_bwd_kernel<TT, D><<<grid, WTHREADS, sm, st>>>(a);                                              \
    biattn_wide_bwd_merge_kernel<TT, D><<<dim3(M, heads, B), 256, 0, st>>>(a, nblk);                           \
  } while (0)
#define B200_WIDE_BWD_T(TT) \
  do { if (dim_head == 32) B200_WIDE_BWD(TT, 32); else if (dim_head == 64) B200_WIDE_BWD(TT, 64); else B200_WIDE_BWD(TT, 80); } while (0)
  if (dtype == B200SEG_F16) B200_WIDE_BWD_T(__half); else B200_WIDE_BWD_T(float);
#undef B200_WIDE_BWD_T
#undef B200_WIDE_BWD
  B200_CHECK_LAUNCH("biattn_wide_bwd");
  return B200SEG_OK;
}
