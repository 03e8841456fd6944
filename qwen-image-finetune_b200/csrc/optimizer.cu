// Fused gradient-clip + AdamW over the flat LoRA gradient buffer (SURVEY.md §8 f1).
// Replaces clip_gradients + optimizer.step() of the reference's step body
// (/root/reference/src/qflux/trainer/base_trainer.py:449-455, 528-533; optimizer built at :884-916, default torch AdamW):
// torch runs a global-norm reduction, a foreach scale and ~10 foreach kernels over 480+ small bf16 tensors.  Here the (already
// all-reduced) fp32 accumulator is read ONCE: sum of squares -> one kernel that applies 1/world, the clip coefficient, decoupled
// weight decay and the Adam update, and writes the bf16 parameters in place (they live inside the padded LoRA factor buffers
// the GEMMs read, so B factors are row-strided).  Moments are fp32 (torch keeps them in the parameter dtype, bf16).
#include <string.h>

#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"

namespace qfx {

// kPartial (deterministic variant): out[blockIdx.x] receives the CTA's share instead of an atomic add.
template <bool kPartial = false>
__global__ void __launch_bounds__(256) adamw_sumsq_kernel(const float* __restrict__ g, int64_t n, float pre_scale, float* __restrict__ out) {
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = g[i] * pre_scale;
    acc += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    if constexpr (kPartial) out[blockIdx.x] = s;
    else atomicAdd(out, s);
  }
}

// One CTA per chunk (<= QFX_ADAMW_CHUNK consecutive elements of ONE tensor, so the row/column split is per tensor).
__global__ void __launch_bounds__(256) fused_adamw_kernel(const qfx_adamw_tensor* __restrict__ tensors, const int2* __restrict__ chunks,
                                                          const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                          const float* __restrict__ sumsq, float pre_scale, float max_norm, float lr,
                                                          float beta1, float beta2, float eps, float weight_decay, float bc1,
                                                          float bc2_sqrt) {
  const int2 ck = chunks[blockIdx.x];
  const qfx_adamw_tensor t = tensors[ck.x];
  float coef = pre_scale;
  if (max_norm > 0.f) {
    const float c = max_norm / (sqrtf(*sumsq) + 1e-6f);  // torch.nn.utils.clip_grad_norm_
    coef *= c < 1.f ? c : 1.f;
  }
  bf16* p = reinterpret_cast<bf16*>(t.param);
  const int end = min(t.numel, ck.y + QFX_ADAMW_CHUNK);
  const float step_size = lr / bc1;
  for (int e = ck.y + threadIdx.x; e < end; e += blockDim.x) {
    const int64_t fi = t.grad_offset + e;
    const int row = e / t.cols, col = e - row * t.cols;
    bf16* pp = p + (int64_t)row * t.ld + col;
    const float gi = g[fi] * coef;
    float w = __bfloat162float(*pp);
    w *= 1.f - lr * weight_decay;
    const float mi = beta1 * m[fi] + (1.f - beta1) * gi;
    const float vi = beta2 * v[fi] + (1.f - beta2) * gi * gi;
    m[fi] = mi;
    v[fi] = vi;
    w -= step_size * mi / (sqrtf(vi) / bc2_sqrt + eps);
    *pp = __float2bfloat16_rn(w);
  }
}

}  // namespace qfx

using namespace qfx;

extern "C" int qfx_fused_adamw(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const float* grad,
                               int64_t n_grad, float* exp_avg, float* exp_avg_sq, float* sumsq, float pre_scale, float max_norm,
                               float lr, float beta1, float beta2, float eps, float weight_decay, int step, void* stream) {
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && grad && exp_avg && exp_avg_sq && sumsq && step >= 1,
                "qfx_fused_adamw: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  QFX_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float), st));
  adamw_sumsq_kernel<<<4 * num_sms(), 256, 0, st>>>(grad, n_grad, pre_scale, sumsq);
  QFX_CUDA(cudaGetLastError());
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  fused_adamw_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), grad, exp_avg, exp_avg_sq, sumsq,
                                              pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, bc1, sqrtf(bc2));
  QFX_CUDA(cudaGetLastError());
  return 0;
}

/* Deterministic variant: QFX_DET_NORM_PARTIALS per-CTA shares of ||grad * pre_scale||^2 go to `scratch` and are summed in a fixed
 * order into sumsq before the update kernel reads it. */
extern "C" int qfx_fused_adamw_det(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const float* grad,
                                   int64_t n_grad, float* exp_avg, float* exp_avg_sq, float* sumsq, float pre_scale, float max_norm,
                                   float lr, float beta1, float beta2, float eps, float weight_decay, int step, float* scratch,
                                   int64_t scratch_floats, void* stream) {
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && grad && exp_avg && exp_avg_sq && sumsq && step >= 1,
                "qfx_fused_adamw_det: bad arguments");
  QFX_CHECK_ARG(scratch && scratch_floats >= QFX_DET_NORM_PARTIALS, "qfx_fused_adamw_det: scratch holds %lld floats, needs %d",
                (long long)scratch_floats, QFX_DET_NORM_PARTIALS);
  cudaStream_t st = (cudaStream_t)stream;
  adamw_sumsq_kernel<true><<<QFX_DET_NORM_PARTIALS, 256, 0, st>>>(grad, n_grad, pre_scale, scratch);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_NORM_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = sumsq; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  int rc = launch_split_sum(S, st);
  if (rc) return rc;
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  fused_adamw_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), grad, exp_avg, exp_avg_sq, sumsq,
                                              pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, bc1, sqrtf(bc2));
  QFX_CUDA(cudaGetLastError());
  return 0;
}
