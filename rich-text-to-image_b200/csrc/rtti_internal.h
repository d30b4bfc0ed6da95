// Internal helpers shared by the rtti_b200 translation units (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rtti_b200.h"

namespace rtti {

// cuTensorMapEncodeTiled resolved through the runtime (no link-time dependency on libcuda).
int encode_tiled_f16(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims,
                     const cuuint64_t* strides_bytes, const cuuint32_t* box, const cuuint32_t* elem_strides);

// 4-D map {head_dim, heads, rows, batch} over a [batch, rows, heads*head_dim] fp16 tensor with element
// strides bs (batch) and rs (row); box = {64, 1, box_rows, 1}, SWIZZLE_128B, zero OOB fill.
int make_head_map(CUtensorMap* m, const void* ptr, int head_dim, int heads, int rows, int batch, long long bs,
                  long long rs, int box_rows);

inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace rtti
