// FP8 frozen weights -> bf16 (qfx_fp8_expand): out[i] = bf16(e4m3fn code[i]).  Every finite e4m3fn value (normals, the subnormals
// down to 2^-9, +-0) is exactly representable in f16 and in bf16, so the expansion is exact: no rounding rule to restate.
// Bandwidth-bound: each thread turns 16 code bytes into 16 bf16 (one 16-byte load, two 16-byte stores).
#include <cuda_bf16.h>

#include "../../include/qfx.h"
#include "host_common.h"

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 16;  // elements per thread step: 16 code bytes

struct Segments {
  qfx_fp8_segment s[QFX_FP8_MAX_SEGMENTS];
  int64_t chunk_end[QFX_FP8_MAX_SEGMENTS];  // inclusive prefix sum of n / 16
  int nseg;
};

// Two e4m3fn codes (byte 0 in the low half) -> two bf16 (element 0 in the low half).  Spelled out in PTX so that the library's
// --use_fast_math cannot flush anything: e4m3 -> f16 is exact (cvt.rn.f16x2.e4m3x2, sm_89+), f16 -> f32 is exact, and every value
// in this range is a bf16 normal (or zero), so the final round-to-nearest never rounds.
__device__ __forceinline__ uint32_t e4m3x2_to_bf16x2(uint16_t codes) {
  uint32_t h2, r;
  float lo, hi;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(codes));
  asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %2;\n\tcvt.f32.f16 %0, l;\n\tcvt.f32.f16 %1, h;\n\t}"
      : "=f"(lo), "=f"(hi) : "r"(h2));
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

__global__ void __launch_bounds__(kThreads) fp8_expand_kernel(const __grid_constant__ Segments segs, int64_t total) {
  for (int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x; c < total; c += (int64_t)gridDim.x * kThreads) {
    int i = 0;
    while (c >= segs.chunk_end[i]) ++i;
    const qfx_fp8_segment& sg = segs.s[i];
    const int64_t local = c - (i ? segs.chunk_end[i - 1] : 0);
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(sg.codes) + local);
    const uint32_t words[4] = {q.x, q.y, q.z, q.w};
    uint4 out[2];
    uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll
    for (int w = 0; w < 4; ++w) {  // little-endian: bytes 4w .. 4w+3 of the chunk
      o[2 * w] = e4m3x2_to_bf16x2((uint16_t)(words[w] & 0xffffu));
      o[2 * w + 1] = e4m3x2_to_bf16x2((uint16_t)(words[w] >> 16));
    }
    uint4* dst = reinterpret_cast<uint4*>(sg.out) + local * 2;
    dst[0] = out[0];
    dst[1] = out[1];
  }
}

}  // namespace

extern "C" int qfx_fp8_expand(const qfx_fp8_segment* segs, int nseg, void* stream) {
  QFX_CHECK_ARG(segs && nseg > 0 && nseg <= QFX_FP8_MAX_SEGMENTS, "qfx_fp8_expand: nseg=%d (1..%d)", nseg, QFX_FP8_MAX_SEGMENTS);
  Segments p;
  int64_t total = 0;
  for (int i = 0; i < nseg; ++i) {
    const qfx_fp8_segment& s = segs[i];
    QFX_CHECK_ARG(s.codes && s.out, "qfx_fp8_expand: segment %d has a NULL pointer", i);
    QFX_CHECK_ARG(s.n > 0 && s.n % kChunk == 0, "qfx_fp8_expand: segment %d: n=%lld is not a positive multiple of 16", i,
                  (long long)s.n);
    QFX_CHECK_ARG(((uintptr_t)s.codes | (uintptr_t)s.out) % 16 == 0,
                  "qfx_fp8_expand: segment %d: codes and out must be 16-byte aligned", i);
    p.s[i] = s;
    total += s.n / kChunk;
    p.chunk_end[i] = total;
  }
  p.nseg = nseg;
  const int64_t blocks_needed = (total + kThreads - 1) / kThreads;
  const int grid = (int)(blocks_needed < (int64_t)qfx::num_sms() * 8 ? blocks_needed : (int64_t)qfx::num_sms() * 8);
  fp8_expand_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(p, total);
  QFX_CUDA(cudaGetLastError());
  return 0;
}
