// Host-side TMA descriptor construction without linking libcuda: the driver entry point is
// resolved at run time through the CUDA runtime (the build box has no GPU / driver).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
      fprintf(stderr, "[b200] cuTensorMapEncodeTiled unavailable (%d)\n", (int)e);
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// Generic rank-N bf16/fp32 tiled map. dims/box innermost first; strides (bytes) for dims 1..rank-1.
inline int make_tmap(CUtensorMap* m, CUtensorMapDataType dt, int rank, const void* ptr, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return -1;
  // The encode call is a DRIVER API call and needs a context current in the calling thread.  PyTorch's autograd worker
  // threads only get one lazily, on their first runtime-API call -- a backward node whose first CUDA action is a GEMM
  // (tensor-map encode, output served from the caching allocator) got CUDA_ERROR_INVALID_CONTEXT.  cudaFree(0) binds the
  // primary context of the current device to this thread; once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(0);
    ctx_bound = true;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(ptr), (const cuuint64_t*)dims,
                  (const cuuint64_t*)strides_bytes, (const cuuint32_t*)box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {   // e.g. the thread switched devices: bind again and retry once
    cudaFree(0);
    r = fn(m, dt, (cuuint32_t)rank, const_cast<void*>(ptr), (const cuuint64_t*)dims, (const cuuint64_t*)strides_bytes,
           (const cuuint32_t*)box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[b200] cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu box %u %u stride %llu)\n", (int)r,
            rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
            rank > 1 ? box[1] : 0, (unsigned long long)(rank > 1 ? strides_bytes[0] : 0));
    return -2;
  }
  return 0;
}

inline int make_tmap_2d_bf16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                             uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {ld_elems * 2};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// e4m3 / uint8 operand tiles: one element = one byte, 128-byte swizzle atoms hold 128 elements along K
inline int make_tmap_2d_u8(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_bytes,
                           uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {ld_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

inline int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace b200
