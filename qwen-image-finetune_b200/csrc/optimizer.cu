// Fused gradient-clip + AdamW over the flat LoRA gradient buffer (SURVEY.md §8 f1).
// Replaces clip_gradients + optimizer.step() of the reference's step body
// (/root/reference/src/qflux/trainer/base_trainer.py:449-455, 528-533; optimizer built at :884-916, default torch AdamW):
// torch runs a global-norm reduction, a foreach scale and ~10 foreach kernels over 480+ small bf16 tensors.  Here the (already
// all-reduced) fp32 accumulator is read ONCE: sum of squares -> one kernel that applies 1/world, the clip coefficient, decoupled
// weight decay and the Adam update, and writes the bf16 parameters in place (they live inside the padded LoRA factor buffers
// the GEMMs read, so B factors are row-strided).  Moments are fp32 (torch keeps them in the parameter dtype, bf16).
// The same tables drive the configs' other optimizer, prodigyopt.Prodigy (qfx_fused_prodigy): its two global sums (sum g*(p0-p) and
// sum |s|) are per-CTA partials added in a fixed order on the device, where prodigyopt calls .item() twice per parameter tensor.
// And bitsandbytes' block-wise Adam8bit (qfx_fused_adam8bit): one pass over the chunks with uint8 states and per-block absmax.
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

// ---- Prodigy (qfx.h qfx_fused_prodigy).  dlr = d * lr * bias_correction(k), from the device scalars, identical in every kernel.
__device__ __forceinline__ double prodigy_dlr(const double* sc, double lr, double beta1, double beta2, int use_bias_correction) {
  const double k = sc[QFX_PRODIGY_K];
  const double bc = use_bias_correction ? sqrt(1.0 - pow(beta2, k + 1.0)) / (1.0 - pow(beta1, k + 1.0)) : 1.0;
  return sc[QFX_PRODIGY_D] * lr * bc;
}

// Pass A: one CTA per chunk.  Updates m, v, s with the OLD d and dlr and stores the CTA's (sum g*(p0 - p), sum |s|) in part[2*cta].
__global__ void __launch_bounds__(256) prodigy_pass_a_kernel(const qfx_adamw_tensor* __restrict__ tensors, const int2* __restrict__ chunks,
                                                             const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                             float* __restrict__ s, const bf16* __restrict__ p0, const double* __restrict__ sc,
                                                             const float* __restrict__ sumsq, float pre_scale, float max_norm, double lr,
                                                             double beta1, double beta2, double beta3, float weight_decay, int decouple,
                                                             int use_bias_correction, int safeguard_warmup, double d0, double* __restrict__ part) {
  const int2 ck = chunks[blockIdx.x];
  const qfx_adamw_tensor t = tensors[ck.x];
  float coef = pre_scale;
  if (max_norm > 0.f) {
    const float c = max_norm / (sqrtf(*sumsq) + 1e-6f);  // torch.nn.utils.clip_grad_norm_
    coef *= c < 1.f ? c : 1.f;
  }
  const double d = sc[QFX_PRODIGY_D], dlr = prodigy_dlr(sc, lr, beta1, beta2, use_bias_correction);
  const float b1 = (float)beta1, b2 = (float)beta2, b3 = (float)beta3;
  const float cm = beta1 > 0.0 ? (float)(d * (1.0 - beta1)) : 1.f, cv = (float)(d * d * (1.0 - beta2)), cs = (float)(d / d0 * (safeguard_warmup ? d : dlr));
  const float wd = decouple ? 0.f : weight_decay;  // coupled weight decay joins the (clipped) gradient
  const bf16* p = reinterpret_cast<const bf16*>(t.param);
  const int end = min(t.numel, ck.y + QFX_ADAMW_CHUNK);
  float dot = 0.f, sabs = 0.f;
  for (int e = ck.y + threadIdx.x; e < end; e += blockDim.x) {
    const int64_t fi = t.grad_offset + e;
    const int row = e / t.cols, col = e - row * t.cols;
    const float w = __bfloat162float(p[(int64_t)row * t.ld + col]);
    const float gi = g[fi] * coef + wd * w;
    dot += gi * (__bfloat162float(p0[fi]) - w);
    m[fi] = b1 * m[fi] + cm * gi;
    v[fi] = b2 * v[fi] + cv * gi * gi;
    const float si = b3 * s[fi] + cs * gi;
    s[fi] = si;
    sabs += fabsf(si);
  }
  double a = dot, b = sabs;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  __shared__ double red[2][8];
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = a;
    red[1][threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb = 0.0;
    for (int i = 0; i < 8; ++i) {
      sa += red[0][i];
      sb += red[1][i];
    }
    part[2 * blockIdx.x] = sa;
    part[2 * blockIdx.x + 1] = sb;
  }
}

// One CTA: the partials of pass A summed in a fixed order (thread i takes chunks i, i+256, ... in turn, then thread 0 adds the 256
// sums in thread order), then thread 0 updates d, d_max, d_numerator, k and the skip flag.
__global__ void __launch_bounds__(256) prodigy_scalar_kernel(double* __restrict__ sc, const double* __restrict__ part, int n_parts,
                                                             double lr, double beta1, double beta2, double beta3, int use_bias_correction,
                                                             double d0, double d_coef, double growth_rate) {
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n_parts; i += blockDim.x) {
    a += part[2 * i];
    b += part[2 * i + 1];
  }
  __shared__ double red[2][256];
  red[0][threadIdx.x] = a;
  red[1][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.x != 0) return;
  double dot = 0.0, den = 0.0;
  for (int i = 0; i < blockDim.x; ++i) {
    dot += red[0][i];
    den += red[1][i];
  }
  double d = sc[QFX_PRODIGY_D], d_max = sc[QFX_PRODIGY_D_MAX];
  const double dlr = prodigy_dlr(sc, lr, beta1, beta2, use_bias_correction);
  const double d_num = beta3 * sc[QFX_PRODIGY_D_NUM] + d / d0 * dlr * dot;
  sc[QFX_PRODIGY_DLR] = dlr;
  if (den == 0.0) {  // no progress yet (every gradient so far was zero): prodigyopt returns before touching d or the parameters
    sc[QFX_PRODIGY_SKIPPED] = 1.0;
    return;
  }
  const double d_hat = d_coef * d_num / den;
  if (d == d0) d = fmax(d, d_hat);
  d_max = fmax(d_max, d_hat);
  d = fmin(d_max, d * growth_rate);
  sc[QFX_PRODIGY_D] = d;
  sc[QFX_PRODIGY_D_MAX] = d_max;
  sc[QFX_PRODIGY_D_NUM] = d_num;
  sc[QFX_PRODIGY_K] += 1.0;
  sc[QFX_PRODIGY_SKIPPED] = 0.0;
  sc[QFX_PRODIGY_D_DEN] = den;
  sc[QFX_PRODIGY_D_HAT] = d_hat;
}

// Pass B: one CTA per chunk, unless the scalar kernel skipped the step.  Decoupled weight decay and the update with the OLD dlr, the
// denominator with the NEW d; the parameter is rounded to bf16 once.  beta1 == 0: m holds the gradient and the step is dlr * d_new * g,
// as prodigyopt takes it.
__global__ void __launch_bounds__(256) prodigy_pass_b_kernel(const qfx_adamw_tensor* __restrict__ tensors, const int2* __restrict__ chunks,
                                                             const float* __restrict__ m, const float* __restrict__ v,
                                                             const double* __restrict__ sc, float eps, float weight_decay, int decouple,
                                                             int has_ema) {
  if (sc[QFX_PRODIGY_SKIPPED] != 0.0) return;
  const int2 ck = chunks[blockIdx.x];
  const qfx_adamw_tensor t = tensors[ck.x];
  const float dlr = (float)sc[QFX_PRODIGY_DLR], deps = (float)(sc[QFX_PRODIGY_D] * (double)eps);
  const float ms = has_ema ? 1.f : (float)sc[QFX_PRODIGY_D];
  const float wd = decouple ? weight_decay : 0.f;
  bf16* p = reinterpret_cast<bf16*>(t.param);
  const int end = min(t.numel, ck.y + QFX_ADAMW_CHUNK);
  for (int e = ck.y + threadIdx.x; e < end; e += blockDim.x) {
    const int64_t fi = t.grad_offset + e;
    const int row = e / t.cols, col = e - row * t.cols;
    bf16* pp = p + (int64_t)row * t.ld + col;
    const float w = __bfloat162float(*pp);
    *pp = __float2bfloat16_rn(w - dlr * (wd * w + ms * m[fi] / (sqrtf(v[fi]) + deps)));
  }
}

// ---- 8-bit Adam (qfx.h qfx_fused_adam8bit).  The nearest entry of the sorted 256-entry map q (shared memory) to x; a tie takes the
// lower code.  lo ends as the last index with q[lo] <= x (0 when x < q[0]).
__device__ __forceinline__ int adam8bit_quantize(const float* q, float x) {
  int lo = 0;
#pragma unroll
  for (int s = 128; s > 0; s >>= 1)
    if (q[lo + s] <= x) lo += s;
  return lo < 255 && x > 0.5f * (q[lo] + q[lo + 1]) ? lo + 1 : lo;
}

// One CTA per chunk.  Warp w takes the chunk's blocks w, w + 8 (QFX_ADAMW_CHUNK / QFX_ADAM8BIT_BLOCK = 16 of them), lane l the block's
// elements l, l + 32, ..., so a block's absmax is one warp reduction and no block is split between warps.
constexpr int kAdam8bitPerLane = QFX_ADAM8BIT_BLOCK / 32;
static_assert(QFX_ADAMW_CHUNK % QFX_ADAM8BIT_BLOCK == 0, "a block must not cross a chunk");

__global__ void __launch_bounds__(256) fused_adam8bit_kernel(const qfx_adamw_tensor* __restrict__ tensors, const int2* __restrict__ chunks,
                                                             const int64_t* __restrict__ state_offsets, const float* __restrict__ g,
                                                             uint8_t* __restrict__ code1, uint8_t* __restrict__ code2,
                                                             float* __restrict__ absmax1, float* __restrict__ absmax2,
                                                             float* __restrict__ s1_32, float* __restrict__ s2_32,
                                                             const float* __restrict__ qmap1, const float* __restrict__ qmap2,
                                                             const float* __restrict__ sumsq, float pre_scale, float max_norm, float beta1,
                                                             float beta2, float c2eps, float step_size, float decay, int min_8bit_size) {
  __shared__ float q1[256], q2[256];
  q1[threadIdx.x] = qmap1[threadIdx.x];
  q2[threadIdx.x] = qmap2[threadIdx.x];
  __syncthreads();
  const int2 ck = chunks[blockIdx.x];
  const qfx_adamw_tensor t = tensors[ck.x];
  const int64_t so = state_offsets[ck.x];
  const bool blockwise = t.numel >= min_8bit_size;
  float coef = pre_scale;
  if (max_norm > 0.f) {
    const float c = max_norm / (sqrtf(*sumsq) + 1e-6f);  // torch.nn.utils.clip_grad_norm_
    coef *= c < 1.f ? c : 1.f;
  }
  bf16* p = reinterpret_cast<bf16*>(t.param);
  const int end = min(t.numel, ck.y + QFX_ADAMW_CHUNK), lane = threadIdx.x & 31;
  for (int b0 = ck.y + (threadIdx.x >> 5) * QFX_ADAM8BIT_BLOCK; b0 < end; b0 += 8 * QFX_ADAM8BIT_BLOCK) {
    const int64_t blk = so + b0 / QFX_ADAM8BIT_BLOCK;
    const float a1 = blockwise ? absmax1[blk] : 0.f, a2 = blockwise ? absmax2[blk] : 0.f;
    float s1[kAdam8bitPerLane], s2[kAdam8bitPerLane], m1 = 0.f, m2 = 0.f;
    unsigned finite = 0;  // bit j: element j of this lane has a finite gradient
#pragma unroll
    for (int j = 0; j < kAdam8bitPerLane; ++j) {
      const int e = b0 + lane + 32 * j;
      s1[j] = s2[j] = 0.f;
      if (e >= end) continue;
      const int64_t fi = t.grad_offset + e;
      const float gi = g[fi] * coef;
      if (!isfinite(gi)) continue;  // bitsandbytes: both states 0, the parameter untouched
      finite |= 1u << j;
      const float o1 = blockwise ? q1[code1[fi]] * a1 : s1_32[so + e];
      const float o2 = blockwise ? q2[code2[fi]] * a2 : s2_32[so + e];
      s1[j] = o1 * beta1 + (1.f - beta1) * gi;
      // the 8-bit kernel forms (1 - beta2) g g left to right, the 32-bit kernel (1 - beta2) (g g)
      s2[j] = blockwise ? o2 * beta2 + (1.f - beta2) * gi * gi : o2 * beta2 + (1.f - beta2) * (gi * gi);
      m1 = fmaxf(m1, fabsf(s1[j]));
      m2 = fmaxf(m2, fabsf(s2[j]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
      m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
    }
    if (blockwise && lane == 0) {
      absmax1[blk] = m1;
      absmax2[blk] = m2;
    }
#pragma unroll
    for (int j = 0; j < kAdam8bitPerLane; ++j) {
      const int e = b0 + lane + 32 * j;
      if (e >= end) continue;
      const int64_t fi = t.grad_offset + e;
      const int row = e / t.cols, col = e - row * t.cols;
      bf16* pp = p + (int64_t)row * t.ld + col;
      if (finite >> j & 1) {
        // decay is 1 without weight decay: the second rounding then returns the bf16 value unchanged
        const bf16 w = __float2bfloat16_rn(__bfloat162float(*pp) + step_size * (s1[j] / (sqrtf(s2[j]) + c2eps)));
        *pp = __float2bfloat16_rn(__bfloat162float(w) * decay);
      }
      if (!blockwise) {
        s1_32[so + e] = s1[j];
        s2_32[so + e] = s2[j];
        continue;
      }
      int c1 = QFX_ADAM8BIT_CODE1_ZERO, c2 = QFX_ADAM8BIT_CODE2_ZERO;
      if (m1 > 0.f) {
        c1 = adam8bit_quantize(q1, s1[j] / m1);
        if (signbit(q1[c1]) != signbit(s1[j])) c1 += s1[j] > 0.f ? 1 : -1;
      }
      if (m2 > 0.f) c2 = adam8bit_quantize(q2, s2[j] / m2);
      code1[fi] = (uint8_t)c1;
      code2[fi] = (uint8_t)c2;
    }
  }
}

}  // namespace qfx

using namespace qfx;

extern "C" int qfx_fused_adam8bit(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const int64_t* state_offsets,
                                  const float* grad, int64_t n_grad, unsigned char* state1, unsigned char* state2, float* absmax1,
                                  float* absmax2, float* s1_32, float* s2_32, const float* qmap1, const float* qmap2, float* sumsq,
                                  float* scratch, int64_t scratch_floats, float pre_scale, float max_norm, float lr, float beta1,
                                  float beta2, float eps, float weight_decay, int step, int min_8bit_size, void* stream) {
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && state_offsets && grad && n_grad > 0 && state1 && state2 && absmax1 &&
                    absmax2 && s1_32 && s2_32 && qmap1 && qmap2 && sumsq && step >= 1 && min_8bit_size >= 0,
                "qfx_fused_adam8bit: bad arguments");
  QFX_CHECK_ARG(scratch && scratch_floats >= QFX_DET_NORM_PARTIALS, "qfx_fused_adam8bit: scratch holds %lld floats, needs %d",
                (long long)scratch_floats, QFX_DET_NORM_PARTIALS);
  QFX_CHECK_ARG(lr >= 0.f, "qfx_fused_adam8bit: needs lr >= 0, got %g", (double)lr);
  cudaStream_t st = (cudaStream_t)stream;
  adamw_sumsq_kernel<true><<<QFX_DET_NORM_PARTIALS, 256, 0, st>>>(grad, n_grad, pre_scale, scratch);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_NORM_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = sumsq; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  int rc = launch_split_sum(S, st);
  if (rc) return rc;
  // bitsandbytes forms these in fp32 (kernels.cu: correction1, correction2, step_size; the decay factor 1 - lr * weight_decay)
  const float c1 = 1.f - powf(beta1, (float)step), c2 = sqrtf(1.f - powf(beta2, (float)step));
  const float step_size = -lr * c2 / c1, decay = weight_decay > 0.f ? 1.f - lr * weight_decay : 1.f;
  fused_adam8bit_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), state_offsets, grad, state1,
                                                  state2, absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq, pre_scale, max_norm, beta1,
                                                  beta2, c2 * eps, step_size, decay, min_8bit_size);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_fused_prodigy(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const float* grad,
                                 int64_t n_grad, float* exp_avg, float* exp_avg_sq, float* s, const void* p0, double* scalars,
                                 float* sumsq, float* scratch, int64_t scratch_floats, float pre_scale, float max_norm, double lr,
                                 double beta1, double beta2, double beta3, double eps, double weight_decay, int decouple,
                                 int use_bias_correction, int safeguard_warmup, double d0, double d_coef, double growth_rate,
                                 void* stream) {
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && grad && n_grad > 0 && exp_avg && exp_avg_sq && s && p0 && scalars && sumsq,
                "qfx_fused_prodigy: bad arguments");
  QFX_CHECK_ARG(scratch && ((uintptr_t)scratch & 7) == 0 && scratch_floats >= QFX_PRODIGY_SCRATCH(n_chunks),
                "qfx_fused_prodigy: scratch holds %lld floats (8-byte aligned needed), needs %lld", (long long)scratch_floats,
                (long long)QFX_PRODIGY_SCRATCH(n_chunks));
  QFX_CHECK_ARG(lr > 0.0 && d0 > 0.0, "qfx_fused_prodigy: needs lr > 0 (a step with lr == 0 is a no-op the caller skips) and d0 > 0");
  cudaStream_t st = (cudaStream_t)stream;
  adamw_sumsq_kernel<true><<<QFX_DET_NORM_PARTIALS, 256, 0, st>>>(grad, n_grad, pre_scale, scratch);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_NORM_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = sumsq; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  int rc = launch_split_sum(S, st);
  if (rc) return rc;
  double* part = reinterpret_cast<double*>(scratch + QFX_DET_NORM_PARTIALS);
  const int2* ck = reinterpret_cast<const int2*>(chunks_dev);
  prodigy_pass_a_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, ck, grad, exp_avg, exp_avg_sq, s, reinterpret_cast<const bf16*>(p0), scalars,
                                                  sumsq, pre_scale, max_norm, lr, beta1, beta2, beta3, (float)weight_decay, decouple,
                                                  use_bias_correction, safeguard_warmup, d0, part);
  QFX_CUDA(cudaGetLastError());
  prodigy_scalar_kernel<<<1, 256, 0, st>>>(scalars, part, n_chunks, lr, beta1, beta2, beta3, use_bias_correction, d0, d_coef, growth_rate);
  QFX_CUDA(cudaGetLastError());
  prodigy_pass_b_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, ck, exp_avg, exp_avg_sq, scalars, (float)eps, (float)weight_decay, decouple,
                                                  beta1 > 0.0);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_fused_adamw(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const float* grad,
                               int64_t n_grad, float* exp_avg, float* exp_avg_sq, float* sumsq, float pre_scale, float max_norm,
                               float lr, float beta1, float beta2, float eps, float weight_decay, int step, void* stream) {
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && grad && n_grad > 0 && exp_avg && exp_avg_sq && sumsq && step >= 1,
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
  QFX_CHECK_ARG(tensors_dev && chunks_dev && n_chunks > 0 && grad && n_grad > 0 && exp_avg && exp_avg_sq && sumsq && step >= 1,
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

/* ---- Sharded optimizer state (qfx.h "slice forms"; qflux_b200/optim.py shard_state=True).  Each data-parallel rank steps only the
 * chunks of its slice [state_base, state_base + n_state) of the flat gradient and keeps state for that range alone.  The kernels above
 * index the state by the gradient offset fi; the slice entry points hand them state pointers moved back by state_base, so element fi
 * lands at state[fi - state_base] and the replicated launches keep their code.  The norm behind the clip is the caller's: sumsq holds
 * ||grad * pre_scale||^2 summed over the ranks' slices.  Each replaces, for its slice, the reference's optimizer.step()
 * (/root/reference/src/qflux/trainer/base_trainer.py:528-533). */
template <typename T>
static T* state_at(T* p, int64_t state_base) {  // p - state_base, formed on the integer so no pointer leaves the allocation in C++ terms
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) - (uintptr_t)state_base * sizeof(T));
}

static bool slice_args_ok(int n_chunks, int64_t n_grad, int64_t state_base, int64_t n_state) {
  return n_chunks >= 0 && n_grad > 0 && state_base >= 0 && n_state >= 0 && state_base + n_state <= n_grad;
}

extern "C" int qfx_sumsq_det(const float* x, int64_t n, float pre_scale, float* out, float* scratch, int64_t scratch_floats,
                             void* stream) {
  QFX_CHECK_ARG(out && n >= 0 && (x || n == 0), "qfx_sumsq_det: bad arguments");
  QFX_CHECK_ARG(scratch && scratch_floats >= QFX_DET_NORM_PARTIALS, "qfx_sumsq_det: scratch holds %lld floats, needs %d",
                (long long)scratch_floats, QFX_DET_NORM_PARTIALS);
  cudaStream_t st = (cudaStream_t)stream;
  adamw_sumsq_kernel<true><<<QFX_DET_NORM_PARTIALS, 256, 0, st>>>(x, n, pre_scale, scratch);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_NORM_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = out; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  return launch_split_sum(S, st);
}

extern "C" int qfx_fused_adamw_slice(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, const float* grad,
                                     int64_t n_grad, int64_t state_base, int64_t n_state, float* exp_avg, float* exp_avg_sq,
                                     const float* sumsq, float pre_scale, float max_norm, float lr, float beta1, float beta2, float eps,
                                     float weight_decay, int step, void* stream) {
  QFX_CHECK_ARG(slice_args_ok(n_chunks, n_grad, state_base, n_state) && grad && sumsq && step >= 1 &&
                    (n_chunks == 0 || (tensors_dev && chunks_dev && exp_avg && exp_avg_sq)),
                "qfx_fused_adamw_slice: bad arguments");
  if (n_chunks == 0) return 0;
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  fused_adamw_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), grad,
                                                                 state_at(exp_avg, state_base), state_at(exp_avg_sq, state_base), sumsq,
                                                                 pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, bc1, sqrtf(bc2));
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_fused_adam8bit_slice(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks,
                                        const int64_t* state_offsets, const float* grad, int64_t n_grad, int64_t state_base,
                                        int64_t n_state, unsigned char* state1, unsigned char* state2, float* absmax1, float* absmax2,
                                        float* s1_32, float* s2_32, const float* qmap1, const float* qmap2, const float* sumsq,
                                        float pre_scale, float max_norm, float lr, float beta1, float beta2, float eps, float weight_decay,
                                        int step, int min_8bit_size, void* stream) {
  QFX_CHECK_ARG(slice_args_ok(n_chunks, n_grad, state_base, n_state) && grad && sumsq && step >= 1 && min_8bit_size >= 0 &&
                    (n_chunks == 0 || (tensors_dev && chunks_dev && state_offsets && state1 && state2 && absmax1 && absmax2 && s1_32 &&
                                       s2_32 && qmap1 && qmap2)),
                "qfx_fused_adam8bit_slice: bad arguments");
  QFX_CHECK_ARG(lr >= 0.f, "qfx_fused_adam8bit_slice: needs lr >= 0, got %g", (double)lr);
  if (n_chunks == 0) return 0;
  const float c1 = 1.f - powf(beta1, (float)step), c2 = sqrtf(1.f - powf(beta2, (float)step));
  const float step_size = -lr * c2 / c1, decay = weight_decay > 0.f ? 1.f - lr * weight_decay : 1.f;
  fused_adam8bit_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>(
      tensors_dev, reinterpret_cast<const int2*>(chunks_dev), state_offsets, grad, state_at(state1, state_base),
      state_at(state2, state_base), absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq, pre_scale, max_norm, beta1, beta2, c2 * eps,
      step_size, decay, min_8bit_size);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_prodigy_slice_partials(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, int chunk0,
                                          const float* grad, int64_t n_grad, int64_t state_base, int64_t n_state, float* exp_avg,
                                          float* exp_avg_sq, float* s, const void* p0, const double* scalars, const float* sumsq,
                                          double* part, int n_parts, float pre_scale, float max_norm, double lr, double beta1,
                                          double beta2, double beta3, double weight_decay, int decouple, int use_bias_correction,
                                          int safeguard_warmup, double d0, void* stream) {
  QFX_CHECK_ARG(slice_args_ok(n_chunks, n_grad, state_base, n_state) && grad && scalars && sumsq && part && chunk0 >= 0 &&
                    (int64_t)chunk0 + n_chunks <= n_parts &&
                    (n_chunks == 0 || (tensors_dev && chunks_dev && exp_avg && exp_avg_sq && s && p0)),
                "qfx_prodigy_slice_partials: bad arguments");
  QFX_CHECK_ARG(lr > 0.0 && d0 > 0.0, "qfx_prodigy_slice_partials: needs lr > 0 and d0 > 0");
  if (n_chunks == 0) return 0;
  prodigy_pass_a_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>(
      tensors_dev, reinterpret_cast<const int2*>(chunks_dev), grad, state_at(exp_avg, state_base), state_at(exp_avg_sq, state_base),
      state_at(s, state_base), state_at(reinterpret_cast<const bf16*>(p0), state_base), scalars, sumsq, pre_scale, max_norm, lr, beta1,
      beta2, beta3, (float)weight_decay, decouple, use_bias_correction, safeguard_warmup, d0, part + 2 * (int64_t)chunk0);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_prodigy_slice_update(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, int64_t n_grad,
                                        int64_t state_base, int64_t n_state, const float* exp_avg, const float* exp_avg_sq,
                                        double* scalars, const double* part, int n_parts, double lr, double beta1, double beta2,
                                        double beta3, double eps, double weight_decay, int decouple, int use_bias_correction, double d0,
                                        double d_coef, double growth_rate, void* stream) {
  QFX_CHECK_ARG(slice_args_ok(n_chunks, n_grad, state_base, n_state) && scalars && part && n_parts > 0 && n_chunks <= n_parts &&
                    (n_chunks == 0 || (tensors_dev && chunks_dev && exp_avg && exp_avg_sq)),
                "qfx_prodigy_slice_update: bad arguments");
  QFX_CHECK_ARG(lr > 0.0 && d0 > 0.0, "qfx_prodigy_slice_update: needs lr > 0 and d0 > 0");
  cudaStream_t st = (cudaStream_t)stream;
  prodigy_scalar_kernel<<<1, 256, 0, st>>>(scalars, part, n_parts, lr, beta1, beta2, beta3, use_bias_correction, d0, d_coef, growth_rate);
  QFX_CUDA(cudaGetLastError());
  if (n_chunks == 0) return 0;
  prodigy_pass_b_kernel<<<n_chunks, 256, 0, st>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), state_at(exp_avg, state_base),
                                                  state_at(exp_avg_sq, state_base), scalars, (float)eps, (float)weight_decay, decouple,
                                                  beta1 > 0.0);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

namespace qfx {
// One CTA per chunk: the chunk's elements whose gradient offset lies in [g_lo, g_hi) move between the bf16 parameter (row-strided) and
// flat[fi - g_lo].  Runs of 8 elements move as one 16-byte vector when a run is one row and both sides are 16-byte aligned.
template <bool kUnpack>
__global__ void __launch_bounds__(256) lora_pack_kernel(const qfx_adamw_tensor* __restrict__ tensors, const int2* __restrict__ chunks,
                                                        int64_t g_lo, int64_t g_hi, bf16* __restrict__ flat) {
  const int2 ck = chunks[blockIdx.x];
  const qfx_adamw_tensor t = tensors[ck.x];
  const int e0 = (int)max((int64_t)ck.y, g_lo - t.grad_offset);
  const int e1 = (int)min((int64_t)min(t.numel, ck.y + QFX_ADAMW_CHUNK), g_hi - t.grad_offset);
  if (e0 >= e1) return;
  bf16* p = reinterpret_cast<bf16*>(t.param);
  const int64_t fo = t.grad_offset - g_lo;  // flat index of the tensor's element e is fo + e
  const bool vec = (t.cols & 7) == 0 && (t.ld & 7) == 0 && ((uintptr_t)p & 15) == 0 && (((uintptr_t)flat + 2 * fo) & 15) == 0;
  const int v0 = vec ? min(e1, (e0 + 7) & ~7) : e1, v1 = vec ? max(v0, e1 & ~7) : e1;  // [v0, v1): whole 8-runs
  for (int e = v0 + 8 * threadIdx.x; e < v1; e += 8 * blockDim.x) {
    const int row = e / t.cols, col = e - row * t.cols;
    uint4* pp = reinterpret_cast<uint4*>(p + (int64_t)row * t.ld + col);
    uint4* fp = reinterpret_cast<uint4*>(flat + fo + e);
    if constexpr (kUnpack) *pp = *fp;
    else *fp = *pp;
  }
  const int head = v0 - e0;  // [e0, v0) and [v1, e1): fewer than 8 elements each when vec, everything otherwise
  for (int i = threadIdx.x; i < head + (e1 - v1); i += blockDim.x) {
    const int e = i < head ? e0 + i : v1 + (i - head);
    const int row = e / t.cols, col = e - row * t.cols;
    bf16* pp = p + (int64_t)row * t.ld + col;
    if constexpr (kUnpack) *pp = flat[fo + e];
    else flat[fo + e] = *pp;
  }
}
}  // namespace qfx

template <bool kUnpack>
static int lora_pack(const char* what, const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, int64_t g_lo,
                     int64_t g_hi, void* flat, void* stream) {
  QFX_CHECK_ARG(n_chunks >= 0 && g_lo >= 0 && g_hi >= g_lo && (n_chunks == 0 || (tensors_dev && chunks_dev && flat)),
                "%s: bad arguments", what);
  QFX_CHECK_ARG(((uintptr_t)flat & 1) == 0, "%s: flat must be 2-byte aligned", what);
  if (n_chunks == 0 || g_hi == g_lo) return 0;
  lora_pack_kernel<kUnpack><<<n_chunks, 256, 0, (cudaStream_t)stream>>>(tensors_dev, reinterpret_cast<const int2*>(chunks_dev), g_lo, g_hi,
                                                                         reinterpret_cast<bf16*>(flat));
  QFX_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int qfx_lora_pack(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, int64_t g_lo, int64_t g_hi,
                             void* flat, void* stream) {
  return lora_pack<false>("qfx_lora_pack", tensors_dev, chunks_dev, n_chunks, g_lo, g_hi, flat, stream);
}

extern "C" int qfx_lora_unpack(const qfx_adamw_tensor* tensors_dev, const int* chunks_dev, int n_chunks, int64_t g_lo, int64_t g_hi,
                               const void* flat, void* stream) {
  return lora_pack<true>("qfx_lora_unpack", tensors_dev, chunks_dev, n_chunks, g_lo, g_hi, const_cast<void*>(flat), stream);
}
