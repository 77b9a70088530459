// Host side of the GEMM kernels (gemm_wgmma.cu, wgrad_wgmma.cu, gemm_fp8.cu): TMA descriptors (CUtensorMap) for
// row-major bf16 and fp8 matrices, the operand alignment test, the persistent grid and the checked launch.
// cuTensorMapEncodeTiled is resolved through the runtime (cudaGetDriverEntryPoint), so the
// extension does not link libcuda.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "../runtime/common.h"
#include "kernels.h"

namespace m4t {

// TMA bases and the epilogues' 16-byte vector accesses need 16-byte-aligned addresses.
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// One persistent CTA per SM, never more CTAs than tiles, and at least one.
inline int persistent_grid(int64_t tiles, int sm_count) {
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(tiles, sm_count)));
}

// Launches Kernel<<<grid, threads, smem, stream>>>(args...), checks the launch and counts it under `what`.  A kernel
// with dynamic shared memory (smem > 0; always the same amount for one kernel) gets its limit raised on first use.
template <auto Kernel, typename... Args>
void launch_kernel(dim3 grid, int threads, int smem, cudaStream_t stream, const char* what, const Args&... args) {
  if (smem > 0) {
    static std::once_flag once;
    std::call_once(once, [smem] {
      const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      M4T_CHECK(e == cudaSuccess, "cudaFuncSetAttribute(smem) failed: " << cudaGetErrorString(e));
    });
  }
  Kernel<<<grid, threads, smem, stream>>>(args...);
  const cudaError_t err = cudaGetLastError();
  M4T_CHECK(err == cudaSuccess, what << " launch failed: " << cudaGetErrorString(err));
  note_kernel_launch(what);
}

inline CUresult encode_tiled_2d(CUtensorMap* map, CUtensorMapDataType dt, void* base, const cuuint64_t* dims,
                                const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  using Fn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                          const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                          CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static Fn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    M4T_CHECK(e == cudaSuccess && q == cudaDriverEntryPointSuccess && p, "cuTensorMapEncodeTiled unavailable");
    return reinterpret_cast<Fn>(p);
  }();
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, dt, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // A thread that has made no runtime call yet, such as autograd's CUDA worker thread running a node's backward,
    // has no current context; cudaFree(nullptr) binds the device's primary context to it.
    const cudaError_t e = cudaFree(nullptr);
    M4T_CHECK(e == cudaSuccess, "cudaFree(nullptr) failed: " << cudaGetErrorString(e));
    r = fn(map, dt, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  return r;
}

// Row-major [rows, cols] bf16 matrix with leading dimension `ld` (elements); boxes of
// box_cols contiguous elements (<= 64 = one 128-byte swizzle span) x box_rows rows.
inline CUtensorMap make_tmap_bf16_sw128(const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols,
                                        int box_rows) {
  CUtensorMap m;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  CUresult r = encode_tiled_2d(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, const_cast<void*>(base), dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
  M4T_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " << static_cast<int>(r));
  return m;
}

// Row-major [rows, cols] one-byte (fp8) matrix with leading dimension `ld` (bytes, a multiple of 16); boxes of
// 128 contiguous bytes (one 128-byte swizzle span) x box_rows rows.
inline CUtensorMap make_tmap_u8_sw128(const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  CUtensorMap m;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld)};
  const cuuint32_t box[2] = {128u, static_cast<cuuint32_t>(box_rows)};
  CUresult r = encode_tiled_2d(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, const_cast<void*>(base), dims, strides, box,
                               CU_TENSOR_MAP_SWIZZLE_128B);
  M4T_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code " << static_cast<int>(r));
  return m;
}

}  // namespace m4t
