// Host-side helper shared by the kernels that stage tiles with TMA: the driver's
// cuTensorMapEncodeTiled is fetched through the runtime (cudaGetDriverEntryPoint), so that
// libmm_b200.so carries no link-time dependency on libcuda.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <mutex>

namespace mm {

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                  const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

// Row-major 2-D array of `rows` x `cols` elements of `elem_bytes` (1, 2, 4 or 8) bytes, tiles of
// box_rows x box_cols elements, no swizzle, out-of-bounds elements read as zero.
// Returns 0 on success, the CUresult otherwise, -1 if the entry point is unavailable.
inline int encode_plain_2d(CUtensorMap *map, const void *base, size_t elem_bytes, uint64_t rows, uint64_t cols,
                           uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  const CUtensorMapDataType dt = elem_bytes == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                 : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                 : elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_UINT32
                                                   : CU_TENSOR_MAP_DATA_TYPE_UINT64;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return static_cast<int>(enc(map, dt, 2, const_cast<void *>(base), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}

// Same array, 8-byte elements, 128-byte-swizzled tiles of box_rows x 16 elements (one 128-byte
// swizzle row per tile row); out-of-bounds elements read as zero.
inline int encode_sw128_2d_f64(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {cols * 8};
  cuuint32_t box[2] = {16, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return static_cast<int>(enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 2, const_cast<void *>(base), gdim, gstride, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}

// `count` packed arrays of rows x cols as one 3-D tensor {cols, rows, count}: the same tiles, but
// out-of-bounds reads past `rows` are zeros per array instead of the next array's first rows.
inline int encode_sw128_3d_f64(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint64_t count,
                               uint32_t box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  cuuint64_t gdim[3] = {cols, rows, count};
  cuuint64_t gstride[2] = {cols * 8, rows * cols * 8};
  cuuint32_t box[3] = {16, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  return static_cast<int>(enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, const_cast<void *>(base), gdim, gstride, box,
                              estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}

}  // namespace mm
