// tc_common.cuh — pieces shared by the tensor-core kernels (conv_tc.cu, wgrad_tc.cu): PTX wrappers for mbarrier,
// bulk-TMA, cp.async, SWIZZLE_NONE wgmma matrix descriptors and warpgroup register re-distribution; the loaders'
// normalise + activate of one staged chunk; the run-time N -> consumer template dispatch.
// sm_90a; every wrapper is a thin inline-asm statement so the SASS shows HGMMA / UBLKCP / UTMALDG / SYNCS.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>
#include "common.cuh"

namespace tc {

constexpr long long kWaitTimeoutCycles = 4000000000ll;   // ~2 s at 1.9 GHz: a protocol bug traps, it never hangs the GPU
constexpr uint32_t kSuspendNs = 20000;         // suspend-time hint of a blocked try_wait (the thread is woken on completion)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity), "n"(kSuspendNs) : "memory");
  return ok != 0;
}
// bounded wait: a protocol bug must surface as a trap (launch failure), never as a hung GPU.  No out-of-line
// diagnostics: a CALL anywhere in a kernel that uses setmaxnreg makes ptxas keep every role inside the SMALLEST
// register allotment (measured: the epilogue stayed below R88 and spilled its accumulators), and a call inside the
// MMA issue loop pushes the loop off the uniform datapath.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > kWaitTimeoutCycles) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 1-D bulk TMA global -> shared, completion counted on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// 5-D tensor TMA load (SASS: UTMALDG): one box of the tensor map into shared memory, zero-filling out-of-bound
// coordinates (negative ones included), completion counted in bytes on an mbarrier
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
               ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
// 16-byte cp.async (SASS: LDGSTS); src_bytes == 0 zero-fills the destination (out-of-volume voxels)
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory matrix descriptor, SWIZZLE_NONE (layout type 0): 8 x 16-byte core matrices.
//   K-major operand : lbo = stride between core matrices along K, sbo = stride between 8-row groups along M/N
//   MN-major operand: lbo = stride between core matrices along K (voxel groups), sbo = stride along M/N (channel planes)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;                    // base_offset = 0, layout_type = SWIZZLE_NONE (0)
}

// Register re-distribution between warpgroups (4 consecutive warps execute it together).  The kernel is launched with
// 65536 / blockDim registers per thread; role code then grows / shrinks its warpgroup's allotment.
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

struct Ring {
  int idx; uint32_t phase; int n;
  __device__ __forceinline__ void init(int n_) { idx = 0; phase = 0; n = n_; }
  __device__ __forceinline__ void advance() { if (++idx == n) { idx = 0; phase ^= 1; } }
};

// InstanceNorm-normalise + activate one staged 16-byte chunk (8 fp16 channels) in registers: x*sc + sf (== (x - mean)
// * rstd), the activation, fp16 rounding.  RELU is a template parameter so the activation choice stays out of the
// per-element code (common.cuh, act_apply_s).  ReLU is fmaxf(h, 0) (NaN -> 0, never -0); LeakyReLU and "none" are
// h > 0 ? h : slope * h.
template <bool RELU>
__device__ __forceinline__ uint4 norm_act8(uint4 raw, const float (&sc)[8], const float (&sf)[8], float slope) {
  __half2* hv = reinterpret_cast<__half2*>(&raw);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 f = __half22float2(hv[j]);
    f.x = fmaf(f.x, sc[2 * j], sf[2 * j]); f.y = fmaf(f.y, sc[2 * j + 1], sf[2 * j + 1]);
    if (RELU) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); }
    else { f.x = act_apply_s(f.x, slope); f.y = act_apply_s(f.y, slope); }
    hv[j] = __floats2half2_rn(f.x, f.y);
  }
  return raw;
}

// fp32 -> the nearest TF32 value (round to nearest, ties away from zero), kept in fp32 storage with the low 13 mantissa
// bits zero: what the library writes as a TF32 operand, so the tensor core's own treatment of those bits never matters
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// The fp32 form of norm_act8: one 16-byte chunk holds 4 fp32 channels; the result is rounded to TF32.
template <bool RELU>
__device__ __forceinline__ uint4 norm_act4(uint4 raw, const float (&sc)[4], const float (&sf)[4], float slope) {
  float* fv = reinterpret_cast<float*>(&raw);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float f = fmaf(fv[j], sc[j], sf[j]);
    f = RELU ? fmaxf(f, 0.f) : act_apply_s(f, slope);
    fv[j] = round_tf32(f);
  }
  return raw;
}

// Calls f(std::integral_constant<int, N>{}) for the run-time GEMM N of a consumer warpgroup (a multiple of 16 up to
// 128): the one place where an operand width becomes a template argument (of a kernel on the host, of a role on the
// device).  The caller's lambda is host-only or device-only; the check is disabled so neither side warns about the other.
#pragma nv_exec_check_disable
template <class F>
__host__ __device__ __forceinline__ void dispatch_n(int n, F&& f) {
  switch (n) {
    case 16: f(std::integral_constant<int, 16>{}); break;
    case 32: f(std::integral_constant<int, 32>{}); break;
    case 48: f(std::integral_constant<int, 48>{}); break;
    case 64: f(std::integral_constant<int, 64>{}); break;
    case 80: f(std::integral_constant<int, 80>{}); break;
    case 96: f(std::integral_constant<int, 96>{}); break;
    case 112: f(std::integral_constant<int, 112>{}); break;
    default: f(std::integral_constant<int, 128>{}); break;
  }
}

}  // namespace tc
