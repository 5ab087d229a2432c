// Host-side CUtensorMap construction (driver entry point fetched through the runtime: no -lcuda link dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace msam {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled();  // engine.cu

// bf16 row-major 2D tensor [rows, cols] with row pitch `ld` elements; box = [box_rows, 64 cols] (128 B, SWIZZLE_128B).
// Out-of-bounds box elements are zero-filled.  Returns 0 on success.
int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);
// row-major 2D tensor of bf16 (elem_bytes 2) or fp32 (4); box = [box_rows, 128 / elem_bytes cols] (128-B rows, SWIZZLE_128B)
int make_tmap_2d(CUtensorMap* out, const void* gptr, int elem_bytes, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows);
// fp16 variant of make_tmap_bf16_2d
int make_tmap_f16_2d(CUtensorMap* out, const void* gptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows);

// bf16 NHWC tensor [B, H, W, C] as a 4-D map (C, W, H, B), box {64 ch, 64 x, 2 y, 1 image}, SWIZZLE_128B, out-of-bounds
// elements zero (ais.cu)
int make_tmap_nhwc(CUtensorMap* m, const void* x, int B, int H, int W, int C);

}  // namespace msam
