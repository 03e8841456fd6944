// Host-side helpers shared by all translation units: error reporting and TMA tensor-map construction.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace qfx {

void set_error(const char* fmt, ...);

#define QFX_CHECK_ARG(cond, ...)       \
  do {                                 \
    if (!(cond)) {                     \
      ::qfx::set_error(__VA_ARGS__);   \
      return -1;                       \
    }                                  \
  } while (0)

#define QFX_CUDA(expr)                                                                      \
  do {                                                                                      \
    cudaError_t e__ = (expr);                                                               \
    if (e__ != cudaSuccess) {                                                               \
      ::qfx::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return (int)e__;                                                                      \
    }                                                                                       \
  } while (0)

// 2-D / 3-D bf16 tensor map with 128-byte swizzle.  dims/box innermost first; strides (bytes) for dims 1.. .
// Returns 0 on success.
int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box);
// same, fp32 elements (used for TMA reduce-add of fp32 tiles)
int make_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box);

int num_sms();

// Fixed-order reduction of per-CTA partials (the deterministic entry points): element e = (row, col) of a rows x cols grid is
//   acc = part[0*split_stride + e] + part[1*split_stride + e] + ... (split order)
// and goes to dst[row / rows_per_dst + col / cols_per_dst][(row % rows_per_dst) * ld_row + (col % cols_per_dst) * ld_col]
// (+= when accumulate, else =); a NULL dst skips its elements.  One thread per element: no atomics.
struct SplitSum {
  const float* part;
  int64_t split_stride;
  int splits, rows, cols;
  float* dst[3];
  int rows_per_dst, cols_per_dst;
  int64_t ld_row, ld_col;
  int accumulate;
};
int launch_split_sum(const SplitSum& S, cudaStream_t stream);  // elementwise.cu

}  // namespace qfx
