// og_host.cuh — host-side helpers shared by the launchers: error reporting, TMA tensor-map encoding
// (driver entry point fetched at run time, so the library does not link libcuda), tile selection.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>

#include "../../include/opengenie_b200.h"

namespace og {

void set_error(const char* fmt, ...);

#define OG_CHECK_CUDA(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      og::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return OG_ERR_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

#define OG_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      og::set_error(__VA_ARGS__);      \
      return OG_ERR_INVALID_ARGUMENT;  \
    }                                  \
  } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled();

// Encode a bf16 tensor map with zero OOB fill and the given swizzle (128-byte by default).
// dims[0] is the contiguous dimension; strides_bytes[i] is the stride of dims[i+1].
// elem_strides (optional): TMA traversal stride per dimension — box[i] then counts the SOURCE span, and
// ceil(box[i] / elem_strides[i]) elements land in shared memory (strided convolution input boxes).
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides = nullptr,
                   CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B);

int num_sms();

// Reproducible sums of per-block partial results: out[(g*width + i) / row_len * out_ld + (g*width + i) % row_len] +=
// sum over b < nparts of partials[(g * nparts + b) * width + i], added in b order (grid: groups g; see og_host.cu).
int sum_partials(const float* partials, int groups, int nparts, long long width, long long row_len, long long out_ld,
                 float* out, cudaStream_t stream);


// Decompose a block of `vox` (power of two) voxels into a (bw, bh, bt, bn) box over (W, H, T, N):
// widest-first powers of two. Dimensions need not divide: partial boxes are zero-filled by TMA on
// load and masked on store.
void choose_voxel_box(int vox, int N, int T, int H, int W, int* bw, int* bh, int* bt, int* bn);

static inline int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

}  // namespace og
