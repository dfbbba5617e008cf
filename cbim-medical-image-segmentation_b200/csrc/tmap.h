// tmap.h — host-side construction of TMA tensor maps (CUtensorMap) for channels-last activations, without linking
// libcuda: cuTensorMapEncodeTiled is fetched through the runtime's driver-entry-point query.
//
// An activation slice x[b][d][h][w][coff : coff + C] (fp16, row pitch ld; fp32 strides are twice these) is described
// as the 5-D tensor
//   dim0 = g channels (2g B, contiguous)      dim1 = w (stride ld*2 B)      dim2 = h (stride W*ld*2)
//   dim3 = channel group c/g (stride 2g B)    dim4 = b*D + d (stride H*W*ld*2)
// so that ONE cp.async.bulk.tensor box {g, bw, bh, groups, 1} lands in shared memory as [group][bh x bw voxels][g ch],
// with out-of-volume voxels (conv padding, ragged tiles) zero-filled by the TMA unit.  The group width g picks the image:
//   g = 8:  16-byte channel planes, no swizzle — the wgmma operand image of conv_tc.cu (K-major) and of wgrad_tc.cu's
//           plane path (MN-major); g = 4 fp32 channels make the same 16-byte planes for conv_tc.cu's TF32 kernels;
//   g = 32 / 64: one 64- / 128-byte row of channels per voxel, stored SWIZZLE_64B / SWIZZLE_128B (the 16-byte chunk j of
//           the row at shared address A lands at chunk j ^ ((A >> 7) & 3 / 7)) — the MN-major swizzled wgmma image of
//           wgrad_tc.cu's row path.  The destination must be 512- / 1024-byte aligned.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

typedef CUresult (*b200seg_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                            const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                            CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline b200seg_encode_tiled_fn b200seg_encode_tiled() {
  static b200seg_encode_tiled_fn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<b200seg_encode_tiled_fn>(p);
  }
  return fn;
}

// returns false when the map cannot be built (driver entry point missing / shape rejected): callers use their
// cp.async staging path then.  box_groups counts groups of ch_box channels (C must be a multiple of it).  The element
// type is fp16 (f32 = false; ch_box 8, 32 or 64) or fp32 (f32 = true; ch_box 4, the 16-byte planes of conv_tc.cu's TF32
// instantiations); all strides above scale with the element size.
static inline bool b200seg_make_act_tmap(CUtensorMap* m, const void* base_ptr, int ld, int coff, int C, int BD, int H, int W,
                                         int box_w, int box_h, int box_groups, int ch_box = 8, bool f32 = false) {
  b200seg_encode_tiled_fn enc = b200seg_encode_tiled();
  const int es = f32 ? 4 : 2;
  if (!enc || (C % ch_box) || ((ld * es) % 16) || ((coff * es) % 16)) return false;
  const int group_bytes = ch_box * es;
  if (group_bytes != 16 && group_bytes != 64 && group_bytes != 128) return false;
  const char* base = reinterpret_cast<const char*>(base_ptr) + (size_t)coff * es;
  if (reinterpret_cast<uintptr_t>(base) & 15) return false;
  if (box_w > 256 || box_h > 256 || box_groups > 256) return false;
  const CUtensorMapSwizzle swz = group_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : group_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                                                     : CU_TENSOR_MAP_SWIZZLE_NONE;
  cuuint64_t dims[5] = {(cuuint64_t)ch_box, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)(C / ch_box), (cuuint64_t)BD};
  cuuint64_t strides[4] = {(cuuint64_t)ld * es, (cuuint64_t)W * ld * es, (cuuint64_t)ch_box * es, (cuuint64_t)H * W * ld * es};
  cuuint32_t box[5] = {(cuuint32_t)ch_box, (cuuint32_t)box_w, (cuuint32_t)box_h, (cuuint32_t)box_groups, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return enc(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<char*>(base), dims, strides,
             box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
