// Library plumbing: version, architecture gate, TMA descriptor encoding.
#include "rtti_internal.h"

#include <cudaTypedefs.h>

extern "C" int rtti_version(void) { return 100; /* 0.1.0 */ }

extern "C" int rtti_arch_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return RTTI_ERR_CUDA;
  int major = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return RTTI_ERR_CUDA;
  return major == 9 ? RTTI_OK : RTTI_ERR_ARCH;
}

namespace rtti {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}

int encode_tiled_f16(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return RTTI_ERR_CUDA;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims,
                  strides_bytes, box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? RTTI_OK : RTTI_ERR_SHAPE;
}

int make_head_map(CUtensorMap* m, const void* ptr, int head_dim, int heads, int rows, int batch, long long bs,
                  long long rs, int box_rows) {
  cuuint64_t dims[4] = {(cuuint64_t)head_dim, (cuuint64_t)heads, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t strides[3] = {(cuuint64_t)head_dim * 2, (cuuint64_t)rs * 2, (cuuint64_t)bs * 2};
  cuuint32_t box[4] = {64, 1, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return encode_tiled_f16(m, ptr, 4, dims, strides, box, estr);
}

}  // namespace rtti
