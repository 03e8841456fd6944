// NF4 frozen weights -> bf16 (qfx_nf4_dequant): bitsandbytes `dequantize_4bit(..., quant_type="nf4")` for the blockwise
// kernel (kDequantizeBlockwise): w[i] = bf16_rn(NF4[nibble_i] * absmax[i / blocksize]), product in fp32, element 2k in the high
// nibble of byte k.  Bandwidth-bound: each thread turns 16 code bytes into 32 bf16 (one 16-byte load, four 16-byte stores).
#include <cuda_bf16.h>

#include "../../include/qfx.h"
#include "host_common.h"

namespace {

// bitsandbytes' built-in NF4 code book (the kernel uses these constants, not the quant_map stored with a checkpoint)
__constant__ float kNF4[16] = {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f,
                               -0.28444138169288635f, -0.18477343022823334f, -0.09105003625154495f, 0.0f,
                               0.07958029955625534f, 0.16093020141124725f, 0.24611230194568634f, 0.33791524171829224f,
                               0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f};

constexpr int kThreads = 256;
constexpr int kChunk = 32;  // elements per thread step: 16 code bytes

struct Segments {
  qfx_nf4_segment s[QFX_NF4_MAX_SEGMENTS];
  int64_t chunk_end[QFX_NF4_MAX_SEGMENTS];  // inclusive prefix sum of n / 32
  int nseg;
};

// IEEE fp32 product and round-to-nearest-even bf16 pair, spelled out in PTX so that the library's --use_fast_math (flush to zero)
// cannot change a subnormal product: the result must equal bitsandbytes' bit for bit.
__device__ __forceinline__ float mul_rn(float a, float b) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

__global__ void __launch_bounds__(kThreads) nf4_dequant_kernel(const __grid_constant__ Segments segs, int64_t total) {
  __shared__ float nf4[16];
  if (threadIdx.x < 16) nf4[threadIdx.x] = kNF4[threadIdx.x];
  __syncthreads();
  for (int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x; c < total; c += (int64_t)gridDim.x * kThreads) {
    int i = 0;
    while (c >= segs.chunk_end[i]) ++i;
    const qfx_nf4_segment& sg = segs.s[i];
    const int64_t local = c - (i ? segs.chunk_end[i - 1] : 0);
    const uint4 q = __ldg(reinterpret_cast<const uint4*>(sg.codes) + local);
    const float a = __ldg(sg.absmax + (local * kChunk) / sg.blocksize);  // blocksize % 32 == 0: one absmax per chunk
    const uint32_t words[4] = {q.x, q.y, q.z, q.w};
    uint4 out[4];
    uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint32_t byte = (words[w] >> (8 * b)) & 0xffu;  // little-endian: byte 4w + b of the chunk
        o[w * 4 + b] = pack_bf16(mul_rn(nf4[byte >> 4], a), mul_rn(nf4[byte & 0xfu], a));
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(sg.out) + local * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[k] = out[k];
  }
}

}  // namespace

extern "C" int qfx_nf4_dequant(const qfx_nf4_segment* segs, int nseg, void* stream) {
  QFX_CHECK_ARG(segs && nseg > 0 && nseg <= QFX_NF4_MAX_SEGMENTS, "qfx_nf4_dequant: nseg=%d (1..%d)", nseg, QFX_NF4_MAX_SEGMENTS);
  Segments p;
  int64_t total = 0;
  for (int i = 0; i < nseg; ++i) {
    const qfx_nf4_segment& s = segs[i];
    QFX_CHECK_ARG(s.codes && s.absmax && s.out, "qfx_nf4_dequant: segment %d has a NULL pointer", i);
    QFX_CHECK_ARG(s.n > 0 && s.n % kChunk == 0, "qfx_nf4_dequant: segment %d: n=%lld is not a positive multiple of 32", i,
                  (long long)s.n);
    QFX_CHECK_ARG(s.blocksize > 0 && s.blocksize % kChunk == 0 && s.n % s.blocksize == 0,
                  "qfx_nf4_dequant: segment %d: blocksize %d must be a multiple of 32 dividing n=%lld", i, s.blocksize,
                  (long long)s.n);
    QFX_CHECK_ARG(((uintptr_t)s.codes | (uintptr_t)s.out) % 16 == 0 && (uintptr_t)s.absmax % 4 == 0,
                  "qfx_nf4_dequant: segment %d: codes and out must be 16-byte aligned", i);
    p.s[i] = s;
    total += s.n / kChunk;
    p.chunk_end[i] = total;
  }
  p.nseg = nseg;
  const int64_t blocks_needed = (total + kThreads - 1) / kThreads;
  const int grid = (int)(blocks_needed < (int64_t)qfx::num_sms() * 8 ? blocks_needed : (int64_t)qfx::num_sms() * 8);
  nf4_dequant_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(p, total);
  QFX_CUDA(cudaGetLastError());
  return 0;
}
