// Fixed-order sum of the ranks' flat fp32 LoRA gradients (qfx_dp_reduce_det): dst[i] = ((+0 + src[0][i]) + src[1][i]) + ... in
// source order, every add an IEEE round-to-nearest add with denormals kept and no contraction.  The library builds with
// --use_fast_math (-ftz=true), so the adds are spelled out in PTX: `add.rn.f32` has no .ftz and its explicit rounding mode keeps
// ptxas from fusing anything into an FFMA.  Each element depends on its own inputs only, so the grid size never changes a bit.
// Bandwidth-bound: each thread step loads one 16-byte vector from every source and stores one.
#include "../../include/qfx.h"
#include "host_common.h"

namespace {

constexpr int kThreads = 256;

struct Sources {
  const float* p[QFX_MAX_RANKS];
};

__device__ __forceinline__ float add_rn(float a, float b) {
  float c;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(c) : "f"(a), "f"(b));
  return c;
}

// Elements [head, head + 4 * nvec) are read and written as 16-byte vectors (every pointer is 16-byte aligned there); the
// n - 4 * nvec others ([0, head) and the tail) one by one.
template <int NS>
__global__ void __launch_bounds__(kThreads) dp_reduce_kernel(const __grid_constant__ Sources s, float* dst, int64_t n, int64_t head,
                                                             int64_t nvec) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int64_t t0 = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  for (int64_t v = t0; v < nvec; v += stride) {
    float4 x[NS];
#pragma unroll
    for (int r = 0; r < NS; ++r) x[r] = __ldcs(reinterpret_cast<const float4*>(s.p[r] + head) + v);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < NS; ++r) {
      acc.x = add_rn(acc.x, x[r].x);
      acc.y = add_rn(acc.y, x[r].y);
      acc.z = add_rn(acc.z, x[r].z);
      acc.w = add_rn(acc.w, x[r].w);
    }
    reinterpret_cast<float4*>(dst + head)[v] = acc;
  }
  const int64_t nscalar = n - 4 * nvec;
  for (int64_t k = t0; k < nscalar; k += stride) {
    const int64_t i = k < head ? k : k + 4 * nvec;
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < NS; ++r) acc = add_rn(acc, s.p[r][i]);
    dst[i] = acc;
  }
}

template <int NS>
void launch(const Sources& s, float* dst, int64_t n, int64_t head, int64_t nvec, cudaStream_t stream) {
  const int64_t work = nvec > n - 4 * nvec ? nvec : n - 4 * nvec;
  const int64_t cap = (int64_t)qfx::num_sms() * (2048 / kThreads);
  const int64_t blocks = (work + kThreads - 1) / kThreads;
  dp_reduce_kernel<NS><<<(int)(blocks < cap ? blocks : cap), kThreads, 0, stream>>>(s, dst, n, head, nvec);
}

}  // namespace

extern "C" int qfx_dp_reduce_det(const float* const* src, int nsrc, float* dst, int64_t n, void* stream) {
  QFX_CHECK_ARG(src && dst && nsrc >= 1 && nsrc <= QFX_MAX_RANKS && n >= 0,
                "qfx_dp_reduce_det: bad arguments (nsrc=%d of 1..%d, n=%lld)", nsrc, QFX_MAX_RANKS, (long long)n);
  QFX_CHECK_ARG((uintptr_t)dst % 4 == 0, "qfx_dp_reduce_det: dst must be 4-byte aligned");
  Sources s;
  const uintptr_t d0 = (uintptr_t)dst, d1 = d0 + (uintptr_t)n * 4;
  bool vec = true;
  for (int r = 0; r < nsrc; ++r) {
    const uintptr_t a = (uintptr_t)src[r];
    QFX_CHECK_ARG(a && a % 4 == 0, "qfx_dp_reduce_det: src[%d] is NULL or not 4-byte aligned", r);
    QFX_CHECK_ARG(a == d0 || a + (uintptr_t)n * 4 <= d0 || a >= d1,
                  "qfx_dp_reduce_det: src[%d] overlaps dst without being dst", r);
    vec = vec && a % 16 == d0 % 16;
    s.p[r] = src[r];
  }
  if (n == 0) return 0;
  // vectors start at the first 16-byte boundary of dst, which is a 16-byte boundary of every source when they share dst's offset
  int64_t head = vec ? (int64_t)(((16 - d0 % 16) % 16) / 4) : n;
  if (head > n) head = n;
  const int64_t nvec = (n - head) / 4;
  const cudaStream_t st = (cudaStream_t)stream;
  switch (nsrc) {
    case 1: launch<1>(s, dst, n, head, nvec, st); break;
    case 2: launch<2>(s, dst, n, head, nvec, st); break;
    case 3: launch<3>(s, dst, n, head, nvec, st); break;
    case 4: launch<4>(s, dst, n, head, nvec, st); break;
    case 5: launch<5>(s, dst, n, head, nvec, st); break;
    case 6: launch<6>(s, dst, n, head, nvec, st); break;
    case 7: launch<7>(s, dst, n, head, nvec, st); break;
    default: launch<8>(s, dst, n, head, nvec, st); break;
  }
  QFX_CUDA(cudaGetLastError());
  return 0;
}
