// HBM-bound glue kernels of the MMDiT training step (everything that is not a tensor-core contraction).
// One warp per row, 16-byte vector accesses, fp32 math, bf16 rounding at the reference's eager rounding points.
//
// Reference call sites (paths under /root/reference/src/qflux/models/):
//   ln_modulate_*      transformer_qwenimage.py:420-423,443-448,477-484  (LayerNorm(no affine, eps 1e-6) + AdaLN modulate)
//   qk_norm_rope_*     transformer_qwenimage.py:296-326,93-140           (per-head RMSNorm, complex RoPE, [txt;img] concat)
//   gemv_act           transformer_qwenimage.py:143-156,389-392,435-436   (SiLU -> Linear on the [B, D] conditioning vector)
//   rmsnorm_rows       transformer_qwenimage.py:549,625                   (txt_norm)
//   flow_* / loss      trainer/qwen_image_edit_trainer.py:796-812,839-847 ; losses/mse_loss.py:68-82
//   lora_wgrad         peft LoRA Linear autograd: dB = dY^T (s X A^T),  dA = (s dY B)^T X
#include <string.h>
#include <type_traits>

#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"

namespace qfx {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = bf16_lo(w[i]);
    f[2 * i + 1] = bf16_hi(w[i]);
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}

// ============================================================================================ LayerNorm + modulate
// Row kernels are HBM-bound, so they are organised for bytes in flight: a row of D = W*32*VPT*8 elements is owned by W warps
// (VPT 16-byte vectors per thread, 24-48 live floats instead of a whole row per warp), 256-thread CTAs hold 8/W rows and the
// row's warps meet on a named barrier.  (Round-1 first version: one warp per row kept 96-192 floats per lane -> 8-16 warps
// per SM -> 2.6 TB/s forward, 1.9 TB/s backward.)
template <int W>
__device__ __forceinline__ void row_sum2(float& a, float& b, float* red) {  // red: [2 * W] floats private to this row and use
  a = warp_sum(a);
  b = warp_sum(b);
  if (W > 1) {
    const int w = (threadIdx.x >> 5) % W;
    if ((threadIdx.x & 31) == 0) {
      red[w] = a;
      red[W + w] = b;
    }
    asm volatile("bar.sync %0, %1;" ::"r"(1 + (int)(threadIdx.x >> 5) / W), "r"(W * 32) : "memory");
    a = 0.f;
    b = 0.f;
#pragma unroll
    for (int i = 0; i < W; ++i) {
      a += red[i];
      b += red[W + i];
    }
  }
}

// y = bf16( bf16( bf16(LN(x)) * bf16(1 + scale[b]) ) + shift[b] ),   b = row / rows_per_batch.
template <int W, int VPT>
__global__ void __launch_bounds__(256) ln_modulate_fwd_kernel(const bf16* __restrict__ x, int64_t ldx, bf16* __restrict__ y,
                                                              int64_t ldy, const bf16* __restrict__ shift,
                                                              const bf16* __restrict__ scale, int64_t ldmod,
                                                              int rows_per_batch, float* __restrict__ mean_out,
                                                              float* __restrict__ rstd_out, int M, float eps, int split,
                                                              const bf16* __restrict__ shift1, const bf16* __restrict__ scale1,
                                                              int rows_per_batch1) {
  // rows >= split form a second row group with its own modulation vectors (the image stream behind the text stream of a
  // stream-major activation buffer): one launch serves both streams
  constexpr int T = W * 32, D = T * VPT * 8, RPC = 8 / W;
  __shared__ float red[RPC][4 * W];
  const int rl = (threadIdx.x >> 5) / W;
  const int row = min(blockIdx.x * RPC + rl, M - 1);  // surplus rows of the last CTA redo row M-1 (keeps the barrier uniform)
  const int t = threadIdx.x % T;
  float v[VPT][8];
  const uint4* xr = reinterpret_cast<const uint4*>(x + (int64_t)row * ldx);
  float s = 0.f, unused = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    unpack8(xr[i * T + t], v[i]);
#pragma unroll
    for (int e = 0; e < 8; ++e) s += v[i][e];
  }
  row_sum2<W>(s, unused, red[rl]);
  const float mean = s * (1.f / D);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float d = v[i][e] - mean;
      ss += d * d;
    }
  row_sum2<W>(ss, unused, red[rl] + 2 * W);
  const float rstd = rsqrtf(ss * (1.f / D) + eps);
  if (t == 0 && mean_out) {
    mean_out[row] = mean;
    rstd_out[row] = rstd;
  }
  const bool g1 = row >= split;
  const int b = g1 ? (row - split) / rows_per_batch1 : row / rows_per_batch;
  const uint4* sh = reinterpret_cast<const uint4*>((g1 ? shift1 : shift) + (int64_t)b * ldmod);
  const uint4* sc = reinterpret_cast<const uint4*>((g1 ? scale1 : scale) + (int64_t)b * ldmod);
  uint4* yr = reinterpret_cast<uint4*>(y + (int64_t)row * ldy);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    float fs[8], fc[8], o[8];
    unpack8(__ldg(sh + i * T + t), fs);
    unpack8(__ldg(sc + i * T + t), fc);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float n = round_bf16((v[i][e] - mean) * rstd);
      float m = round_bf16(n * round_bf16(1.f + fc[e]));
      o[e] = m + fs[e];
    }
    yr[i * T + t] = pack8(o);
  }
}

// dx = dres + LN_bwd( dy * (1 + scale[b]) );  optional second output dx_gated = dx * gate[b]  (feeds the next dgrad GEMM)
template <int W, int VPT>
__global__ void __launch_bounds__(256) ln_modulate_bwd_kernel(const bf16* __restrict__ dy, int64_t lddy,
                                                              const bf16* __restrict__ x, int64_t ldx,
                                                              const float* __restrict__ mean_in,
                                                              const float* __restrict__ rstd_in,
                                                              const bf16* __restrict__ scale, int64_t ldmod,
                                                              int rows_per_batch, const bf16* __restrict__ dres,
                                                              int64_t lddres, bf16* __restrict__ dx, int64_t lddx,
                                                              const bf16* __restrict__ gate, int64_t ldgate,
                                                              bf16* __restrict__ dx_gated, int64_t lddxg, int M, int split,
                                                              const bf16* __restrict__ scale1, const bf16* __restrict__ gate1,
                                                              int rows_per_batch1) {
  constexpr int T = W * 32, D = T * VPT * 8, RPC = 8 / W;
  __shared__ float red[RPC][2 * W];
  const int rl = (threadIdx.x >> 5) / W;
  const int row = min(blockIdx.x * RPC + rl, M - 1);
  const int t = threadIdx.x % T;
  const bool g1 = row >= split;  // second row group (see ln_modulate_fwd_kernel)
  const int b = g1 ? (row - split) / rows_per_batch1 : row / rows_per_batch;
  if (g1) {
    scale = scale1;
    gate = gate1;
  }
  const float mean = mean_in[row], rstd = rstd_in[row];
  const uint4* dyr = reinterpret_cast<const uint4*>(dy + (int64_t)row * lddy);
  const uint4* xr = reinterpret_cast<const uint4*>(x + (int64_t)row * ldx);
  const uint4* sc = reinterpret_cast<const uint4*>(scale + (int64_t)b * ldmod);
  const uint4* rr = dres ? reinterpret_cast<const uint4*>(dres + (int64_t)row * lddres) : nullptr;
  uint4 rv[VPT];
  if (rr) {  // issued up front: these loads do not depend on the row statistics
#pragma unroll
    for (int i = 0; i < VPT; ++i) rv[i] = rr[i * T + t];
  }
  float g[VPT][8], xh[VPT][8];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    float fd[8], fx[8], fc[8];
    unpack8(dyr[i * T + t], fd);
    unpack8(xr[i * T + t], fx);
    unpack8(__ldg(sc + i * T + t), fc);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      g[i][e] = round_bf16(fd[e] * round_bf16(1.f + fc[e]));  // autograd: grad wrt LN output, bf16
      xh[i][e] = (fx[e] - mean) * rstd;
      s1 += g[i][e];
      s2 += g[i][e] * xh[i][e];
    }
  }
  row_sum2<W>(s1, s2, red[rl]);
  s1 *= (1.f / D);
  s2 *= (1.f / D);
  uint4* dxr = reinterpret_cast<uint4*>(dx + (int64_t)row * lddx);
  const uint4* gt = dx_gated ? reinterpret_cast<const uint4*>(gate + (int64_t)b * ldgate) : nullptr;
  uint4* dxg = dx_gated ? reinterpret_cast<uint4*>(dx_gated + (int64_t)row * lddxg) : nullptr;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    float o[8], fr[8];
    if (rr) unpack8(rv[i], fr);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float d = round_bf16(rstd * (g[i][e] - s1 - xh[i][e] * s2));
      o[e] = rr ? round_bf16(fr[e] + d) : d;
    }
    dxr[i * T + t] = pack8(o);
    if (dxg) {
      float fg[8], og[8];
      unpack8(__ldg(gt + i * T + t), fg);
#pragma unroll
      for (int e = 0; e < 8; ++e) og[e] = o[e] * fg[e];
      dxg[i * T + t] = pack8(og);
    }
  }
}

// Column reductions over the tokens of each sample for the modulation gradients (see qfx_mod_grad in qfx.h).
// grid (D/256, B, row splits): a CTA owns 256 columns (one uint4 per lane) of one sample's row range, its 8 warps stride over
// the rows, partials meet in shared memory and leave as one fp32 atomic per column and CTA.
// kPartial (deterministic variant): sum_out is the split-major partial buffer [splits][2][B][D] (sum, then product) and every CTA
// stores its column totals there; launch_split_sum adds them up in split order.
template <bool kPartial = false>
__global__ void __launch_bounds__(256) mod_grad_kernel(const bf16* __restrict__ g, int64_t ldg, const bf16* __restrict__ m, int64_t ldm,
                                                       const float* __restrict__ mean, const float* __restrict__ rstd,
                                                       int rows_per_batch, float* __restrict__ sum_out, float* __restrict__ prod_out,
                                                       int64_t ldo, int D) {
  __shared__ float red[2][8][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = blockIdx.x * 256 + lane * 8;
  const int b = blockIdx.y;
  const int per = (rows_per_batch + gridDim.z - 1) / gridDim.z;
  const int r0 = blockIdx.z * per, r1 = min(rows_per_batch, r0 + per);
  float s[8], p[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) s[e] = p[e] = 0.f;
  if (col < D) {
    for (int r = r0 + warp; r < r1; r += 8) {
      const int64_t row = (int64_t)b * rows_per_batch + r;
      float fg[8], fm[8];
      unpack8(*reinterpret_cast<const uint4*>(g + row * ldg + col), fg);
      if (m != nullptr) {
        unpack8(*reinterpret_cast<const uint4*>(m + row * ldm + col), fm);
        if (mean != nullptr) {
          const float mu = mean[row], rs = rstd[row];
#pragma unroll
          for (int e = 0; e < 8; ++e) fm[e] = round_bf16((fm[e] - mu) * rs);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) p[e] += fg[e] * fm[e];
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) s[e] += fg[e];
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    red[0][warp][lane * 8 + e] = s[e];
    red[1][warp][lane * 8 + e] = p[e];
  }
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < D) {
    float ts = 0.f, tp = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      ts += red[0][w][threadIdx.x];
      tp += red[1][w][threadIdx.x];
    }
    if constexpr (kPartial) {
      float* part = sum_out + ((int64_t)blockIdx.z * 2 * gridDim.y + b) * D + c;
      part[0] = ts;
      part[(int64_t)gridDim.y * D] = tp;
    } else {
      if (sum_out != nullptr) atomicAdd(sum_out + (int64_t)b * ldo + c, ts);
      if (prod_out != nullptr && m != nullptr) atomicAdd(prod_out + (int64_t)b * ldo + c, tp);
    }
  }
}

// out = a * gate[b]   (backward of the gated residual branch when no LN-bwd kernel precedes it)
__global__ void __launch_bounds__(256) gate_mul_kernel(const bf16* __restrict__ a, int64_t lda, const bf16* __restrict__ gate,
                                                       int64_t ldg, int rows_per_batch, bf16* __restrict__ out, int64_t ldo,
                                                       int M, int D) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int b = row / rows_per_batch;
  const uint4* ar = reinterpret_cast<const uint4*>(a + (int64_t)row * lda);
  const uint4* gr = reinterpret_cast<const uint4*>(gate + (int64_t)b * ldg);
  uint4* orow = reinterpret_cast<uint4*>(out + (int64_t)row * ldo);
  for (int i = lane; i < D / 8; i += 32) {
    float fa[8], fg[8], o[8];
    unpack8(ar[i], fa);
    unpack8(__ldg(gr + i), fg);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = fa[e] * fg[e];
    orow[i] = pack8(o);
  }
}

__global__ void add_bf16_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(__bfloat162float(a[i]) + __bfloat162float(b[i]));
}

// ============================================================================================ RMSNorm over rows (txt_norm)
// diffusers RMSNorm: y = bf16( bf16(x * rsqrt(mean(x^2)+eps)) * w )
__global__ void __launch_bounds__(256) rmsnorm_rows_kernel(const bf16* __restrict__ x, int64_t ldx, const bf16* __restrict__ w,
                                                           bf16* __restrict__ y, int64_t ldy, int M, int D, float eps) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (int64_t)row * ldx);
  float ss = 0.f;
  for (int i = lane; i < D / 8; i += 32) {
    float f[8];
    unpack8(xr[i], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) ss += f[e] * f[e];
  }
  const float r = rsqrtf(warp_sum(ss) / D + eps);
  uint4* yr = reinterpret_cast<uint4*>(y + (int64_t)row * ldy);
  const uint4* wr = reinterpret_cast<const uint4*>(w);
  for (int i = lane; i < D / 8; i += 32) {
    float f[8], fw[8], o[8];
    unpack8(xr[i], f);
    unpack8(__ldg(wr + i), fw);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = round_bf16(f[e] * r) * fw[e];
    yr[i] = pack8(o);
  }
}

// ============================================================================================ q/k RMSNorm + RoPE + layout
// Token-major projections qkv[tok, q|k|v, H, 128]  ->  head-major joint tensors Q/K/V[B, H, S, 128] at joint position
// s = s_offset + (tok % tokens_per_sample).  rope[(b*rope_bstride) + s][64] = (cos, sin) fp32 pairs; pair i rotates
// elements (2i, 2i+1).  One warp per (token, head); lane owns 4 consecutive elements.
template <bool ROUND_MID>
__global__ void __launch_bounds__(256) qk_norm_rope_fwd_kernel(const bf16* __restrict__ qkv, int64_t ldqkv,
                                                               const bf16* __restrict__ wq, const bf16* __restrict__ wk,
                                                               const float2* __restrict__ rope, int64_t rope_bstride,
                                                               bf16* __restrict__ Q, bf16* __restrict__ K, bf16* __restrict__ V,
                                                               int tokens, int tokens_per_sample, int s_offset, int S, int H,
                                                               float eps, int split, const bf16* __restrict__ wq1,
                                                               const bf16* __restrict__ wk1, int tokens_per_sample1, int s_offset1) {
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= tokens * H) return;
  const int tok = gw / H, h = gw - tok * H;
  int b, s;
  if (tok >= split) {  // second token group: its own norm weights, sample length and joint-sequence offset (image stream behind text)
    b = (tok - split) / tokens_per_sample1;
    s = s_offset1 + (tok - split) - b * tokens_per_sample1;
    wq = wq1;
    wk = wk1;
  } else {
    b = tok / tokens_per_sample;
    s = s_offset + tok - b * tokens_per_sample;
  }
  const int D = H * 128;
  const bf16* base = qkv + (int64_t)tok * ldqkv + h * 128 + lane * 4;
  const int64_t dst = (((int64_t)b * H + h) * S + s) * 128 + lane * 4;
  const float4 cs = *reinterpret_cast<const float4*>(rope + ((int64_t)b * rope_bstride + s) * 64 + lane * 2);
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    const uint2 raw = *reinterpret_cast<const uint2*>(base + which * D);
    float f[4] = {bf16_lo(raw.x), bf16_hi(raw.x), bf16_lo(raw.y), bf16_hi(raw.y)};
    float ss = warp_sum(f[0] * f[0] + f[1] * f[1] + f[2] * f[2] + f[3] * f[3]);
    const float r = rsqrtf(ss * (1.f / 128) + eps);
    const uint2 wr = __ldg(reinterpret_cast<const uint2*>((which ? wk : wq) + lane * 4));
    const float w[4] = {bf16_lo(wr.x), bf16_hi(wr.x), bf16_lo(wr.y), bf16_hi(wr.y)};
    float n[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) n[e] = ROUND_MID ? round_bf16(round_bf16(f[e] * r) * w[e]) : round_bf16(f[e] * r * w[e]);
    float o[4];
    o[0] = n[0] * cs.x - n[1] * cs.y;
    o[1] = n[0] * cs.y + n[1] * cs.x;
    o[2] = n[2] * cs.z - n[3] * cs.w;
    o[3] = n[2] * cs.w + n[3] * cs.z;
    *reinterpret_cast<uint2*>((which ? K : Q) + dst) = make_uint2(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]));
  }
  *reinterpret_cast<uint2*>(V + dst) = *reinterpret_cast<const uint2*>(base + 2 * D);
}

// Backward: dQ/dK/dV[B,H,S,128] (bf16) + saved pre-norm qkv  ->  dqkv[tok, 3D].
template <bool ROUND_MID>
__global__ void __launch_bounds__(256) qk_norm_rope_bwd_kernel(float* __restrict__ dQ, const bf16* __restrict__ dK,
                                                               const bf16* __restrict__ dV, const bf16* __restrict__ qkv,
                                                               int64_t ldqkv, const bf16* __restrict__ wq,
                                                               const bf16* __restrict__ wk, const float2* __restrict__ rope,
                                                               int64_t rope_bstride, bf16* __restrict__ dqkv, int64_t lddqkv,
                                                               int tokens, int tokens_per_sample, int s_offset, int S, int H,
                                                               float eps, int split, const bf16* __restrict__ wq1,
                                                               const bf16* __restrict__ wk1, int tokens_per_sample1, int s_offset1,
                                                               int clear_dq) {
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= tokens * H) return;
  const int tok = gw / H, h = gw - tok * H;
  int b, s;
  if (tok >= split) {
    b = (tok - split) / tokens_per_sample1;
    s = s_offset1 + (tok - split) - b * tokens_per_sample1;
    wq = wq1;
    wk = wk1;
  } else {
    b = tok / tokens_per_sample;
    s = s_offset + tok - b * tokens_per_sample;
  }
  const int D = H * 128;
  const bf16* base = qkv + (int64_t)tok * ldqkv + h * 128 + lane * 4;
  bf16* obase = dqkv + (int64_t)tok * lddqkv + h * 128 + lane * 4;
  const int64_t src = (((int64_t)b * H + h) * S + s) * 128 + lane * 4;
  const float4 cs = *reinterpret_cast<const float4*>(rope + ((int64_t)b * rope_bstride + s) * 64 + lane * 2);
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    float go[4];
    if (which) {
      const uint2 graw = *reinterpret_cast<const uint2*>(dK + src);
      go[0] = bf16_lo(graw.x); go[1] = bf16_hi(graw.x); go[2] = bf16_lo(graw.y); go[3] = bf16_hi(graw.y);
    } else {  // dQ is the fp32 TMA-reduce accumulator of the attention backward; autograd would hold it in bf16
      const float4 gq = *reinterpret_cast<const float4*>(dQ + src);
      if (clear_dq) *reinterpret_cast<float4*>(dQ + src) = make_float4(0.f, 0.f, 0.f, 0.f);  // accumulator ready for the next backward
      go[0] = round_bf16(gq.x); go[1] = round_bf16(gq.y); go[2] = round_bf16(gq.z); go[3] = round_bf16(gq.w);
    }
    // rotate back by the conjugate angle (RoPE is orthogonal)
    float gn[4];
    gn[0] = round_bf16(go[0] * cs.x + go[1] * cs.y);
    gn[1] = round_bf16(-go[0] * cs.y + go[1] * cs.x);
    gn[2] = round_bf16(go[2] * cs.z + go[3] * cs.w);
    gn[3] = round_bf16(-go[2] * cs.w + go[3] * cs.z);
    const uint2 raw = *reinterpret_cast<const uint2*>(base + which * D);
    const float f[4] = {bf16_lo(raw.x), bf16_hi(raw.x), bf16_lo(raw.y), bf16_hi(raw.y)};
    const uint2 wr = __ldg(reinterpret_cast<const uint2*>((which ? wk : wq) + lane * 4));
    const float w[4] = {bf16_lo(wr.x), bf16_hi(wr.x), bf16_lo(wr.y), bf16_hi(wr.y)};
    const float ss = warp_sum(f[0] * f[0] + f[1] * f[1] + f[2] * f[2] + f[3] * f[3]);
    const float r = rsqrtf(ss * (1.f / 128) + eps);
    float gw4[4], dot = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      gw4[e] = gn[e] * w[e];
      dot += gw4[e] * f[e];
    }
    dot = warp_sum(dot) * (1.f / 128) * r * r * r;
    float o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = r * gw4[e] - f[e] * dot;
    *reinterpret_cast<uint2*>(obase + which * D) = make_uint2(pack_bf16(o[0], o[1]), pack_bf16(o[2], o[3]));
  }
  *reinterpret_cast<uint2*>(obase + 2 * D) = *reinterpret_cast<const uint2*>(dV + src);
}

// ============================================================================================ conditioning GEMV
// y[b, n] = bf16( sum_k act(x[b,k]) * W[n,k] + bias[n] ),  b < 8.  act: 0 none, 1 SiLU (rounded to bf16 like eager).
// HBM-bound: W is streamed exactly once (13.6 GB for the modulation linears of all 60 Qwen blocks in ONE launch), so the kernel is
// built around bytes in flight: persistent CTAs of 16 warps, each warp owns GEMV_ROWS output rows at a time and keeps GEMV_ROWS
// (x2 unrolled) independent 16-byte weight loads per lane in flight; act(x) is staged once per CTA in shared memory as fp32, laid
// out [batch][half][k/8][4] so that the lanes' 16-byte reads are contiguous (conflict-free) and every x read is shared by the
// GEMV_ROWS rows.  (The first version — one row per warp, 8 rows per CTA, scalar prologue per 8 rows — reached 0.76 TB/s.)
constexpr int GEMV_ROWS = 4;
template <int NB>
__global__ void __launch_bounds__(512) gemv_act_kernel(const bf16* __restrict__ x, int64_t ldx, const bf16* __restrict__ W,
                                                       int64_t ldw, const bf16* __restrict__ bias, bf16* __restrict__ y,
                                                       int64_t ldy, int N, int K, int act) {
  extern __shared__ __align__(16) float xs[];  // [NB][2][K/8][4]
  const int nvec = K / 8;
  for (int v = threadIdx.x; v < NB * nvec; v += blockDim.x) {
    const int b = v / nvec, i = v - b * nvec;
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + (int64_t)b * ldx) + i), f);
    if (act == 1) {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = round_bf16(f[e] / (1.f + __expf(-f[e])));
    }
    float4* dst = reinterpret_cast<float4*>(xs) + (int64_t)b * 2 * nvec + i;
    dst[0] = make_float4(f[0], f[1], f[2], f[3]);
    dst[nvec] = make_float4(f[4], f[5], f[6], f[7]);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  const int n_groups = (N + GEMV_ROWS - 1) / GEMV_ROWS;
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  for (int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); g < n_groups; g += warps_total) {
    const int n0 = g * GEMV_ROWS;
    const uint4* wr[GEMV_ROWS];
#pragma unroll
    for (int r = 0; r < GEMV_ROWS; ++r) wr[r] = reinterpret_cast<const uint4*>(W + (int64_t)min(n0 + r, N - 1) * ldw);
    float acc[GEMV_ROWS][NB];
#pragma unroll
    for (int r = 0; r < GEMV_ROWS; ++r)
#pragma unroll
      for (int b = 0; b < NB; ++b) acc[r][b] = 0.f;
#pragma unroll 2
    for (int i = lane; i < nvec; i += 32) {
      uint4 wv[GEMV_ROWS];
#pragma unroll
      for (int r = 0; r < GEMV_ROWS; ++r) wv[r] = __ldg(wr[r] + i);
      float fw[GEMV_ROWS][8];
#pragma unroll
      for (int r = 0; r < GEMV_ROWS; ++r) unpack8(wv[r], fw[r]);
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 x0 = xs4[(b * 2) * nvec + i], x1 = xs4[(b * 2 + 1) * nvec + i];
#pragma unroll
        for (int r = 0; r < GEMV_ROWS; ++r)
          acc[r][b] += fw[r][0] * x0.x + fw[r][1] * x0.y + fw[r][2] * x0.z + fw[r][3] * x0.w + fw[r][4] * x1.x + fw[r][5] * x1.y +
                       fw[r][6] * x1.z + fw[r][7] * x1.w;
      }
    }
    float mine = 0.f;  // lane r * NB + b keeps (row r, batch b)
#pragma unroll
    for (int r = 0; r < GEMV_ROWS; ++r)
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float v = warp_sum(acc[r][b]);
        if (lane == r * NB + b) mine = v;
      }
    if (lane < GEMV_ROWS * NB) {
      const int r = lane / NB, b = lane - r * NB, n = n0 + r;
      if (n < N) y[(int64_t)b * ldy + n] = __float2bfloat16_rn(mine + (bias ? __bfloat162float(bias[n]) : 0.f));
    }
  }
}

// sinusoidal timestep embedding, diffusers Timesteps(256, flip_sin_to_cos=True, shift=0, scale): out[b] = [cos | sin]
__global__ void timestep_sinusoid_kernel(const float* __restrict__ t, float scale, bf16* __restrict__ out, int B, int dim) {
  const int half = dim / 2;
  for (int i = threadIdx.x + blockIdx.x * blockDim.x; i < B * half; i += blockDim.x * gridDim.x) {
    int b = i / half, j = i - b * half;
    // timestep has been rounded to bf16 by the model (transformer_qwenimage.py:624) — the caller passes that value
    float freq = expf(-9.210340371976184f * (float)j / (float)half);
    float arg = scale * (t[b] * freq);
    out[(int64_t)b * dim + j] = __float2bfloat16_rn(cosf(arg));
    out[(int64_t)b * dim + half + j] = __float2bfloat16_rn(sinf(arg));
  }
}

// ============================================================================================ flow matching
// packed[b, 0:L] = bf16( bf16((1-sigma_b)*x0) + bf16(sigma_b*noise) ) ; packed[b, L:L+Lc] = control
__global__ void flow_noisy_input_kernel(const bf16* __restrict__ x0, const bf16* __restrict__ noise,
                                        const bf16* __restrict__ control, const float* __restrict__ sigma,
                                        bf16* __restrict__ packed, int B, int L, int Lc, int Cc) {
  const int64_t per = (int64_t)(L + Lc) * Cc;
  const int64_t total = (int64_t)B * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int b = (int)(i / per);
    int64_t r = i - (int64_t)b * per;
    if (r < (int64_t)L * Cc) {
      float sg = round_bf16(sigma[b]);
      float one_m = round_bf16(1.f - sg);
      float a = round_bf16(one_m * __bfloat162float(x0[(int64_t)b * L * Cc + r]));
      float c = round_bf16(sg * __bfloat162float(noise[(int64_t)b * L * Cc + r]));
      packed[i] = __float2bfloat16_rn(a + c);
    } else {
      packed[i] = control[(int64_t)b * Lc * Cc + (r - (int64_t)L * Cc)];
    }
  }
}

// multi-resolution variant: per-sample target / control lengths; sample b's sequence is [noisy target (Lt[b]) | control (Lc[b]) | 0-pad]
// (flux_kontext_trainer.py:660-700 builds the same per-sample concatenation before padding to the batch maximum)
__global__ void flow_noisy_input_var_kernel(const bf16* __restrict__ x0, const bf16* __restrict__ noise,
                                            const bf16* __restrict__ control, const float* __restrict__ sigma,
                                            const int* __restrict__ Lt, const int* __restrict__ Lc, bf16* __restrict__ packed, int B,
                                            int Ltmax, int Lcmax, int Ltot, int Cc) {
  const int64_t per = (int64_t)Ltot * Cc;
  const int64_t total = (int64_t)B * per;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / per);
    const int64_t r = i - (int64_t)b * per;
    const int t = (int)(r / Cc), c = (int)(r - (int64_t)t * Cc);
    const int lt = Lt[b], lc = Lc[b];
    float v = 0.f;
    if (t < lt) {
      const int64_t j = ((int64_t)b * Ltmax + t) * Cc + c;
      const float sg = round_bf16(sigma[b]);
      v = round_bf16(round_bf16(1.f - sg) * __bfloat162float(x0[j])) + round_bf16(sg * __bfloat162float(noise[j]));
    } else if (t < lt + lc) {
      v = __bfloat162float(control[((int64_t)b * Lcmax + (t - lt)) * Cc + c]);
    }
    packed[i] = __float2bfloat16_rn(v);
  }
}

// loss += norm * sum w[b,t] * (pred - (noise - x0))^2 ;  dpred = 2 * norm * w * (pred - target) * loss_scale  (bf16),
// zero for the control tokens.  pred is [B, Ltot, C]; only the first L tokens carry loss (trainer :839).
// kPartial (deterministic variant): loss[blockIdx.x] receives the CTA's share instead of an atomic add.
template <bool kPartial = false>
__global__ void __launch_bounds__(256) flow_loss_kernel(const bf16* __restrict__ pred, const bf16* __restrict__ x0,
                                                        const bf16* __restrict__ noise, const float* __restrict__ w,
                                                        float norm, float grad_scale, float* __restrict__ loss,
                                                        bf16* __restrict__ dpred, int B, int L, int Ltot, int Cc) {
  const int64_t total = (int64_t)B * Ltot * Cc;
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t bt = i / Cc;
    int c = (int)(i - bt * Cc);
    int b = (int)(bt / Ltot), t = (int)(bt - (int64_t)b * Ltot);
    float g = 0.f;
    if (t < L) {
      int64_t j = ((int64_t)b * L + t) * Cc + c;
      float target = round_bf16(__bfloat162float(noise[j]) - __bfloat162float(x0[j]));
      float d = __bfloat162float(pred[i]) - target;
      float wt = w ? w[(int64_t)b * L + t] : 1.f;
      acc += wt * d * d;
      g = 2.f * norm * wt * d * grad_scale;
    }
    if (dpred) dpred[i] = __float2bfloat16_rn(g);
  }
  acc = warp_sum(acc);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += red[i];
    if constexpr (kPartial) loss[blockIdx.x] = s * norm;
    else atomicAdd(loss, s * norm);
  }
}

// ============================================================================================ LoRA weight gradients
// G[i, j] += sum_m P[m, i] * Q[m, j]   (i < Dp, j < r <= 64), fp32 atomics into G with strides (gs_i, gs_j) so the same
// kernel writes dB[out, r] (P = dY, Q = s X A^T) and dA[r, in] (P = X, Q = s dY B; transposed store).
// Block: 128 columns of P x a chunk of rows; thread = one column i, r fp32 accumulators; Q rows broadcast from smem.
// kPartial (deterministic variant): G is the split-major partial buffer [splits][Dp][R], stored with plain stores.
template <int R, bool kPartial = false>
__global__ void __launch_bounds__(128) lora_wgrad_kernel(const bf16* __restrict__ P, int64_t ldp, const bf16* __restrict__ Q,
                                                         int64_t ldq, float* __restrict__ G, int64_t gs_i, int64_t gs_j, int M,
                                                         int Dp, int rows_per_block) {
  __shared__ float qs[64][R];
  const int i = blockIdx.x * 128 + threadIdx.x;
  const int m_begin = blockIdx.y * rows_per_block;
  const int m_end = min(M, m_begin + rows_per_block);
  float acc[R];
#pragma unroll
  for (int j = 0; j < R; ++j) acc[j] = 0.f;
  for (int m0 = m_begin; m0 < m_end; m0 += 64) {
    const int nrows = min(64, m_end - m0);
    __syncthreads();
    for (int e = threadIdx.x; e < 64 * R; e += 128) {
      int rr = e / R, j = e - rr * R;
      qs[rr][j] = rr < nrows ? __bfloat162float(Q[(int64_t)(m0 + rr) * ldq + j]) : 0.f;
    }
    __syncthreads();
    if (i < Dp) {
#pragma unroll 4
      for (int rr = 0; rr < nrows; ++rr) {
        const float p = __bfloat162float(P[(int64_t)(m0 + rr) * ldp + i]);
#pragma unroll
        for (int j = 0; j < R; ++j) acc[j] += p * qs[rr][j];
      }
    }
  }
  if (i < Dp) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if constexpr (kPartial) G[((int64_t)blockIdx.y * Dp + i) * R + j] = acc[j];
      else atomicAdd(G + (int64_t)i * gs_i + (int64_t)j * gs_j, acc[j]);
    }
  }
}

// delta[b,h,s] = sum_d dO * O over one head (token-major [tokens, H*128] operands) — softmax-backward row term.
__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ O, int64_t ldo, const bf16* __restrict__ dO,
                                                         int64_t lddo, float* __restrict__ delta, bf16* __restrict__ dOj,
                                                         int tokens, int tokens_per_sample, int s_offset, int S, int H, int split,
                                                         int tokens_per_sample1, int s_offset1) {
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= tokens * H) return;
  const int tok = gw / H, h = gw - tok * H;
  int b, s;
  if (tok >= split) {
    b = (tok - split) / tokens_per_sample1;
    s = s_offset1 + (tok - split) - b * tokens_per_sample1;
  } else {
    b = tok / tokens_per_sample;
    s = s_offset + tok - b * tokens_per_sample;
  }
  const uint2 a = *reinterpret_cast<const uint2*>(O + (int64_t)tok * ldo + h * 128 + lane * 4);
  const uint2 g = *reinterpret_cast<const uint2*>(dO + (int64_t)tok * lddo + h * 128 + lane * 4);
  float d = bf16_lo(a.x) * bf16_lo(g.x) + bf16_hi(a.x) * bf16_hi(g.x) + bf16_lo(a.y) * bf16_lo(g.y) + bf16_hi(a.y) * bf16_hi(g.y);
  d = warp_sum(d);
  if (lane == 0) delta[((int64_t)b * H + h) * S + s] = d;
  if (dOj) *reinterpret_cast<uint2*>(dOj + (((int64_t)b * H + h) * S + s) * 128 + lane * 4) = g;
}

// grads(fp32 accumulators) -> scale (1/world, clip) -> bf16 ; sumsq of the scaled-by-inv_world grads accumulated first
// kPartial (deterministic variant): out[blockIdx.x] receives the CTA's share instead of an atomic add.
template <bool kPartial = false>
__global__ void __launch_bounds__(256) sumsq_kernel(const float* __restrict__ g, int64_t n, float pre_scale, float* __restrict__ out) {
  float acc = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = g[i] * pre_scale;
    acc += v * v;
  }
  acc = warp_sum(acc);
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
// out_bf16 = g * pre_scale * min(1, max_norm / (sqrt(sumsq) + 1e-6))     (torch.nn.utils.clip_grad_norm_ semantics)
__global__ void __launch_bounds__(256) clip_cast_kernel(const float* __restrict__ g, int64_t n, float pre_scale,
                                                        const float* __restrict__ sumsq, float max_norm, bf16* __restrict__ out) {
  float coef = 1.f;
  if (max_norm > 0.f) {
    float c = max_norm / (sqrtf(*sumsq) + 1e-6f);
    coef = c < 1.f ? c : 1.f;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(g[i] * pre_scale * coef);
}

__global__ void __launch_bounds__(256) split_sum_kernel(const SplitSum S) {
  const int64_t n = (int64_t)S.rows * S.cols;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(e / S.cols), col = (int)(e - (int64_t)row * S.cols);
    const int di = row / S.rows_per_dst + col / S.cols_per_dst;
    float* d = di == 0 ? S.dst[0] : (di == 1 ? S.dst[1] : S.dst[2]);  // no dynamic index into the parameter: no local copy
    if (d == nullptr) continue;
    float acc = 0.f;
    for (int sp = 0; sp < S.splits; ++sp) acc += S.part[sp * S.split_stride + e];
    d += (int64_t)(row % S.rows_per_dst) * S.ld_row + (int64_t)(col % S.cols_per_dst) * S.ld_col;
    *d = S.accumulate ? *d + acc : acc;
  }
}

int launch_split_sum(const SplitSum& S, cudaStream_t stream) {
  const int64_t n = (int64_t)S.rows * S.cols;
  const int blocks = (int)(n < 256 * 1024 ? (n + 255) / 256 : 1024);
  split_sum_kernel<<<blocks, 256, 0, stream>>>(S);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace qfx

using namespace qfx;

#define LAUNCH_OK()              \
  QFX_CUDA(cudaGetLastError()); \
  return 0

// D = 256 * nv  ->  (warps per row, 16-byte vectors per thread)
template <typename F>
static int dispatch_nv(int D, F&& f) {
  switch (D / 256) {
    case 1: return f(std::integral_constant<int, 1>(), std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>(), std::integral_constant<int, 1>());
    case 4: return f(std::integral_constant<int, 4>(), std::integral_constant<int, 1>());
    case 8: return f(std::integral_constant<int, 4>(), std::integral_constant<int, 2>());
    case 12: return f(std::integral_constant<int, 4>(), std::integral_constant<int, 3>());
    case 16: return f(std::integral_constant<int, 4>(), std::integral_constant<int, 4>());
  }
  set_error("hidden size %d unsupported (need 256*{1,2,4,8,12,16})", D);
  return -1;
}

static bool aligned(const void* p, uintptr_t bytes) { return (uintptr_t)p % bytes == 0; }  // a null (unused) operand passes

extern "C" int qfx_ln_modulate_fwd_pair(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale,
                                        int64_t ldmod, int rows_per_batch, float* mean, float* rstd, int M, int D, float eps,
                                        int split, const void* shift1, const void* scale1, int rows_per_batch1, void* stream) {
  QFX_CHECK_ARG(D % 256 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldmod % 8 == 0, "qfx_ln_modulate_fwd: bad dims");
  QFX_CHECK_ARG(split >= M || (shift1 && scale1 && rows_per_batch1 > 0), "qfx_ln_modulate_fwd_pair: second group needs shift/scale/rows_per_batch");
  return dispatch_nv(D, [&](auto w, auto vpt) {
    constexpr int W = decltype(w)::value, RPC = 8 / W;
    ln_modulate_fwd_kernel<W, decltype(vpt)::value><<<(M + RPC - 1) / RPC, 256, 0, (cudaStream_t)stream>>>(
        (const bf16*)x, ldx, (bf16*)y, ldy, (const bf16*)shift, (const bf16*)scale, ldmod, rows_per_batch, mean, rstd, M, eps, split,
        (const bf16*)shift1, (const bf16*)scale1, rows_per_batch1);
    LAUNCH_OK();
  });
}

extern "C" int qfx_ln_modulate_fwd(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale,
                                   int64_t ldmod, int rows_per_batch, float* mean, float* rstd, int M, int D, float eps,
                                   void* stream) {
  return qfx_ln_modulate_fwd_pair(x, ldx, y, ldy, shift, scale, ldmod, rows_per_batch, mean, rstd, M, D, eps, M, nullptr, nullptr, 1,
                                  stream);
}

extern "C" int qfx_ln_modulate_bwd_pair(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                        const float* rstd, const void* scale, int64_t ldmod, int rows_per_batch, const void* dres,
                                        int64_t lddres, void* dx, int64_t lddx, const void* gate, int64_t ldgate, void* dx_gated,
                                        int64_t lddxg, int M, int D, int split, const void* scale1, const void* gate1,
                                        int rows_per_batch1, void* stream) {
  QFX_CHECK_ARG(D % 256 == 0, "qfx_ln_modulate_bwd: bad dims");
  QFX_CHECK_ARG(split >= M || (scale1 && rows_per_batch1 > 0 && ((gate1 != nullptr) == (gate != nullptr))),
                "qfx_ln_modulate_bwd_pair: second group needs scale (and a gate iff the first group has one)");
  // every operand is accessed in 16-byte vectors: 8-element leading dimensions and 16-byte aligned bases
  QFX_CHECK_ARG(lddy % 8 == 0 && ldx % 8 == 0 && ldmod % 8 == 0 && lddx % 8 == 0 && (!dres || lddres % 8 == 0) &&
                    (!dx_gated || (ldgate % 8 == 0 && lddxg % 8 == 0)),
                "qfx_ln_modulate_bwd_pair: leading dimensions must be multiples of 8 elements");
  QFX_CHECK_ARG(aligned(dy, 16) && aligned(x, 16) && aligned(scale, 16) && aligned(scale1, 16) && aligned(dres, 16) &&
                    aligned(dx, 16) && (!dx_gated || (aligned(gate, 16) && aligned(gate1, 16) && aligned(dx_gated, 16))),
                "qfx_ln_modulate_bwd_pair: operands must be 16-byte aligned");
  return dispatch_nv(D, [&](auto w, auto vpt) {
    constexpr int W = decltype(w)::value, RPC = 8 / W;
    ln_modulate_bwd_kernel<W, decltype(vpt)::value><<<(M + RPC - 1) / RPC, 256, 0, (cudaStream_t)stream>>>(
        (const bf16*)dy, lddy, (const bf16*)x, ldx, mean, rstd, (const bf16*)scale, ldmod, rows_per_batch, (const bf16*)dres,
        lddres, (bf16*)dx, lddx, (const bf16*)gate, ldgate, (bf16*)dx_gated, lddxg, M, split, (const bf16*)scale1,
        (const bf16*)gate1, rows_per_batch1);
    LAUNCH_OK();
  });
}

extern "C" int qfx_ln_modulate_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean,
                                   const float* rstd, const void* scale, int64_t ldmod, int rows_per_batch, const void* dres,
                                   int64_t lddres, void* dx, int64_t lddx, const void* gate, int64_t ldgate, void* dx_gated,
                                   int64_t lddxg, int M, int D, void* stream) {
  return qfx_ln_modulate_bwd_pair(dy, lddy, x, ldx, mean, rstd, scale, ldmod, rows_per_batch, dres, lddres, dx, lddx, gate, ldgate,
                                  dx_gated, lddxg, M, D, M, nullptr, nullptr, 1, stream);
}

extern "C" int qfx_mod_grad(const void* g, int64_t ldg, const void* m, int64_t ldm, const float* mean, const float* rstd,
                            int rows_per_batch, float* sum_out, float* prod_out, int64_t ldo, int M, int D, void* stream) {
  QFX_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && ldg % 8 == 0 && (m == nullptr || ldm % 8 == 0) && rows_per_batch > 0 &&
                    M % rows_per_batch == 0,
                "qfx_mod_grad: bad dims (D=%d, M=%d, rows_per_batch=%d)", D, M, rows_per_batch);
  QFX_CHECK_ARG((mean == nullptr) == (rstd == nullptr) && (mean == nullptr || m != nullptr), "qfx_mod_grad: mean/rstd need m");
  QFX_CHECK_ARG(aligned(g, 16) && aligned(m, 16), "qfx_mod_grad: g / m must be 16-byte aligned");
  const int B = M / rows_per_batch, cb = (D + 255) / 256;
  int splits = (4 * num_sms() + cb * B - 1) / (cb * B);  // about four CTAs per SM
  splits = splits < 1 ? 1 : (splits > (rows_per_batch + 31) / 32 ? (rows_per_batch + 31) / 32 : splits);
  mod_grad_kernel<<<dim3(cb, B, splits), 256, 0, (cudaStream_t)stream>>>((const bf16*)g, ldg, (const bf16*)m, ldm, mean, rstd,
                                                                        rows_per_batch, sum_out, prod_out, ldo, D);
  LAUNCH_OK();
}

extern "C" int qfx_gate_mul(const void* a, int64_t lda, const void* gate, int64_t ldg, int rows_per_batch, void* out,
                            int64_t ldo, int M, int D, void* stream) {
  QFX_CHECK_ARG(D % 8 == 0, "qfx_gate_mul: D %% 8");
  // a, gate and out are accessed in 16-byte vectors
  QFX_CHECK_ARG(lda % 8 == 0 && ldg % 8 == 0 && ldo % 8 == 0, "qfx_gate_mul: leading dimensions must be multiples of 8 elements");
  QFX_CHECK_ARG(aligned(a, 16) && aligned(gate, 16) && aligned(out, 16), "qfx_gate_mul: operands must be 16-byte aligned");
  gate_mul_kernel<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const bf16*)a, lda, (const bf16*)gate, ldg, rows_per_batch,
                                                                 (bf16*)out, ldo, M, D);
  LAUNCH_OK();
}

extern "C" int qfx_add_bf16(const void* a, const void* b, void* out, int64_t n, void* stream) {
  add_bf16_kernel<<<64, 256, 0, (cudaStream_t)stream>>>((const bf16*)a, (const bf16*)b, (bf16*)out, n);
  LAUNCH_OK();
}

extern "C" int qfx_rmsnorm_rows(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int M, int D, float eps,
                                void* stream) {
  QFX_CHECK_ARG(D % 8 == 0, "qfx_rmsnorm_rows: D %% 8");
  rmsnorm_rows_kernel<<<(M + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const bf16*)x, ldx, (const bf16*)w, (bf16*)y, ldy, M, D, eps);
  LAUNCH_OK();
}

extern "C" int qfx_qk_norm_rope_fwd_pair(const void* qkv, int64_t ldqkv, const void* wq, const void* wk, const float* rope,
                                         int64_t rope_bstride, void* Q, void* K, void* V, int tokens, int tokens_per_sample,
                                         int s_offset, int S, int H, float eps, int round_mid, int split, const void* wq1,
                                         const void* wk1, int tokens_per_sample1, int s_offset1, void* stream) {
  QFX_CHECK_ARG(split >= tokens || (wq1 && wk1 && tokens_per_sample1 > 0), "qfx_qk_norm_rope_fwd_pair: second group incomplete");
  QFX_CHECK_ARG(ldqkv % 4 == 0 && aligned(qkv, 8), "qfx_qk_norm_rope_fwd_pair: qkv needs an 8-byte aligned base and ldqkv %% 4 == 0");
  const int blocks = (tokens * H + 7) / 8;
  if (round_mid)
    qk_norm_rope_fwd_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        (const bf16*)qkv, ldqkv, (const bf16*)wq, (const bf16*)wk, (const float2*)rope, rope_bstride, (bf16*)Q, (bf16*)K, (bf16*)V,
        tokens, tokens_per_sample, s_offset, S, H, eps, split, (const bf16*)wq1, (const bf16*)wk1, tokens_per_sample1, s_offset1);
  else
    qk_norm_rope_fwd_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        (const bf16*)qkv, ldqkv, (const bf16*)wq, (const bf16*)wk, (const float2*)rope, rope_bstride, (bf16*)Q, (bf16*)K, (bf16*)V,
        tokens, tokens_per_sample, s_offset, S, H, eps, split, (const bf16*)wq1, (const bf16*)wk1, tokens_per_sample1, s_offset1);
  LAUNCH_OK();
}

extern "C" int qfx_qk_norm_rope_fwd(const void* qkv, int64_t ldqkv, const void* wq, const void* wk, const float* rope,
                                    int64_t rope_bstride, void* Q, void* K, void* V, int tokens, int tokens_per_sample,
                                    int s_offset, int S, int H, float eps, int round_mid, void* stream) {
  return qfx_qk_norm_rope_fwd_pair(qkv, ldqkv, wq, wk, rope, rope_bstride, Q, K, V, tokens, tokens_per_sample, s_offset, S, H, eps,
                                   round_mid, tokens, nullptr, nullptr, 1, 0, stream);
}

extern "C" int qfx_qk_norm_rope_bwd_pair(void* dQ, const void* dK, const void* dV, const void* qkv, int64_t ldqkv,
                                         const void* wq, const void* wk, const float* rope, int64_t rope_bstride, void* dqkv,
                                         int64_t lddqkv, int tokens, int tokens_per_sample, int s_offset, int S, int H, float eps,
                                         int round_mid, int split, const void* wq1, const void* wk1, int tokens_per_sample1,
                                         int s_offset1, int clear_dq, void* stream) {
  QFX_CHECK_ARG(split >= tokens || (wq1 && wk1 && tokens_per_sample1 > 0), "qfx_qk_norm_rope_bwd_pair: second group incomplete");
  QFX_CHECK_ARG(ldqkv % 4 == 0 && lddqkv % 4 == 0 && aligned(qkv, 8) && aligned(dqkv, 8) && aligned(dQ, 16),
                "qfx_qk_norm_rope_bwd_pair: qkv / dqkv need 8-byte aligned bases and leading dimensions %% 4 == 0");
  const int blocks = (tokens * H + 7) / 8;
  if (round_mid)
    qk_norm_rope_bwd_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        (float*)dQ, (const bf16*)dK, (const bf16*)dV, (const bf16*)qkv, ldqkv, (const bf16*)wq, (const bf16*)wk,
        (const float2*)rope, rope_bstride, (bf16*)dqkv, lddqkv, tokens, tokens_per_sample, s_offset, S, H, eps, split,
        (const bf16*)wq1, (const bf16*)wk1, tokens_per_sample1, s_offset1, clear_dq);
  else
    qk_norm_rope_bwd_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(
        (float*)dQ, (const bf16*)dK, (const bf16*)dV, (const bf16*)qkv, ldqkv, (const bf16*)wq, (const bf16*)wk,
        (const float2*)rope, rope_bstride, (bf16*)dqkv, lddqkv, tokens, tokens_per_sample, s_offset, S, H, eps, split,
        (const bf16*)wq1, (const bf16*)wk1, tokens_per_sample1, s_offset1, clear_dq);
  LAUNCH_OK();
}

extern "C" int qfx_qk_norm_rope_bwd(const void* dQ, const void* dK, const void* dV, const void* qkv, int64_t ldqkv,
                                    const void* wq, const void* wk, const float* rope, int64_t rope_bstride, void* dqkv,
                                    int64_t lddqkv, int tokens, int tokens_per_sample, int s_offset, int S, int H, float eps,
                                    int round_mid, void* stream) {
  return qfx_qk_norm_rope_bwd_pair(const_cast<void*>(dQ), dK, dV, qkv, ldqkv, wq, wk, rope, rope_bstride, dqkv, lddqkv, tokens,
                                   tokens_per_sample, s_offset, S, H, eps, round_mid, tokens, nullptr, nullptr, 1, 0, 0, stream);
}

extern "C" int qfx_gemv_act(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* y, int64_t ldy,
                            int B, int N, int K, int act, void* stream) {
  QFX_CHECK_ARG(B >= 1 && B <= 8 && K % 8 == 0 && ldw % 8 == 0, "qfx_gemv_act: B=%d K=%d", B, K);
  QFX_CHECK_ARG(((uintptr_t)x % 16) == 0 && ((uintptr_t)W % 16) == 0 && ldx % 8 == 0, "qfx_gemv_act: x / W must be 16-byte aligned");
  int grid = (N + GEMV_ROWS * 16 - 1) / (GEMV_ROWS * 16);  // 16 warps x GEMV_ROWS rows per CTA pass; persistent beyond one CTA per SM
  if (grid > num_sms()) grid = num_sms();
  size_t sm = (size_t)B * K * sizeof(float);
  QFX_CHECK_ARG(sm <= 200 * 1024, "qfx_gemv_act: K too large");
#define GEMV(NB)                                                                                                             \
  case NB: {                                                                                                                 \
    static bool done = false;                                                                                                \
    if (!done) {                                                                                                             \
      QFX_CUDA(cudaFuncSetAttribute(gemv_act_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));          \
      done = true;                                                                                                           \
    }                                                                                                                        \
    gemv_act_kernel<NB><<<grid, 512, sm, (cudaStream_t)stream>>>((const bf16*)x, ldx, (const bf16*)W, ldw, (const bf16*)bias, \
                                                                 (bf16*)y, ldy, N, K, act);                                 \
  } break;
  switch (B) {
    GEMV(1) GEMV(2) GEMV(3) GEMV(4) GEMV(5) GEMV(6) GEMV(7) GEMV(8)
  }
#undef GEMV
  LAUNCH_OK();
}

extern "C" int qfx_timestep_sinusoid(const float* t, float scale, void* out, int B, int dim, void* stream) {
  timestep_sinusoid_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(t, scale, (bf16*)out, B, dim);
  LAUNCH_OK();
}

extern "C" int qfx_flow_noisy_input(const void* x0, const void* noise, const void* control, const float* sigma, void* packed,
                                    int B, int L, int Lc, int C, void* stream) {
  flow_noisy_input_kernel<<<296, 256, 0, (cudaStream_t)stream>>>((const bf16*)x0, (const bf16*)noise, (const bf16*)control, sigma,
                                                                 (bf16*)packed, B, L, Lc, C);
  LAUNCH_OK();
}

extern "C" int qfx_flow_noisy_input_var(const void* x0, const void* noise, const void* control, const float* sigma, const int* Lt,
                                        const int* Lc, void* packed, int B, int Ltmax, int Lcmax, int Ltot, int C, void* stream) {
  flow_noisy_input_var_kernel<<<296, 256, 0, (cudaStream_t)stream>>>((const bf16*)x0, (const bf16*)noise, (const bf16*)control, sigma,
                                                                     Lt, Lc, (bf16*)packed, B, Ltmax, Lcmax, Ltot, C);
  LAUNCH_OK();
}

extern "C" int qfx_flow_loss(const void* pred, const void* x0, const void* noise, const float* w, float norm, float grad_scale,
                             float* loss, void* dpred, int B, int L, int Ltot, int C, void* stream) {
  QFX_CHECK_ARG(loss && B > 0 && L > 0 && Ltot >= L && C > 0, "qfx_flow_loss: bad arguments");
  QFX_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), (cudaStream_t)stream));
  flow_loss_kernel<<<296, 256, 0, (cudaStream_t)stream>>>((const bf16*)pred, (const bf16*)x0, (const bf16*)noise, w, norm,
                                                          grad_scale, loss, (bf16*)dpred, B, L, Ltot, C);
  LAUNCH_OK();
}

extern "C" int qfx_lora_wgrad(const void* P, int64_t ldp, const void* Q, int64_t ldq, float* G, int64_t gs_i, int64_t gs_j,
                              int M, int Dp, int r, void* stream) {
  QFX_CHECK_ARG(r == 4 || r == 8 || r == 16 || r == 32 || r == 64, "qfx_lora_wgrad: rank %d unsupported (4/8/16/32/64)", r);
  QFX_CHECK_ARG(G && M > 0 && Dp > 0, "qfx_lora_wgrad: bad arguments");
  int splits = (M + 511) / 512;
  int rows = ((M + splits - 1) / splits + 63) / 64 * 64;
  dim3 grid((Dp + 127) / 128, (M + rows - 1) / rows);
#define WG(R)                                                                                                                  \
  case R:                                                                                                                      \
    lora_wgrad_kernel<R><<<grid, 128, 0, (cudaStream_t)stream>>>((const bf16*)P, ldp, (const bf16*)Q, ldq, G, gs_i, gs_j, M, Dp, \
                                                                 rows);                                                        \
    break;
  switch (r) {
    WG(4) WG(8) WG(16) WG(32) WG(64)
    default:
      set_error("qfx_lora_wgrad: rank %d unsupported (4/8/16/32/64)", r);
      return -1;
  }
#undef WG
  LAUNCH_OK();
}

extern "C" int qfx_attn_delta_pair(const void* O, int64_t ldo, const void* dO, int64_t lddo, float* delta, void* dO_joint,
                                   int tokens, int tokens_per_sample, int s_offset, int S, int H, int split, int tokens_per_sample1,
                                   int s_offset1, void* stream) {
  QFX_CHECK_ARG(split >= tokens || tokens_per_sample1 > 0, "qfx_attn_delta_pair: second group incomplete");
  QFX_CHECK_ARG(ldo % 4 == 0 && lddo % 4 == 0 && aligned(O, 8) && aligned(dO, 8),
                "qfx_attn_delta_pair: O / dO need 8-byte aligned bases and leading dimensions %% 4 == 0");
  attn_delta_kernel<<<(tokens * H + 7) / 8, 256, 0, (cudaStream_t)stream>>>((const bf16*)O, ldo, (const bf16*)dO, lddo, delta,
                                                                            (bf16*)dO_joint, tokens, tokens_per_sample, s_offset,
                                                                            S, H, split, tokens_per_sample1, s_offset1);
  LAUNCH_OK();
}

extern "C" int qfx_attn_delta(const void* O, int64_t ldo, const void* dO, int64_t lddo, float* delta, void* dO_joint,
                              int tokens, int tokens_per_sample, int s_offset, int S, int H, void* stream) {
  return qfx_attn_delta_pair(O, ldo, dO, lddo, delta, dO_joint, tokens, tokens_per_sample, s_offset, S, H, tokens, 1, 0, stream);
}

extern "C" int qfx_grad_finalize(const float* g, int64_t n, float pre_scale, float max_norm, float* sumsq, void* out_bf16,
                                 void* stream) {
  QFX_CHECK_ARG(g && n > 0 && sumsq && out_bf16, "qfx_grad_finalize: bad arguments");
  QFX_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float), (cudaStream_t)stream));
  sumsq_kernel<<<592, 256, 0, (cudaStream_t)stream>>>(g, n, pre_scale, sumsq);
  clip_cast_kernel<<<592, 256, 0, (cudaStream_t)stream>>>(g, n, pre_scale, sumsq, max_norm, (bf16*)out_bf16);
  LAUNCH_OK();
}

// ---------------------------------------------------------------------------------------------------------------------
// Zero-fill of the padding rows a ragged GEMM skips (qfx_gemm_problem.row_tiles): keeps "every padded row of a gradient buffer is
// exactly zero", which the LoRA weight-gradient and modulation-gradient reductions over all rows rely on.
__global__ void zero_rows_kernel(bf16* __restrict__ out, int64_t ld, int ncols, const int* __restrict__ ranges, int n_ranges) {
  const int vec_per_row = ncols >> 3;
  for (int r = 0; r < n_ranges; ++r) {
    const int lo = ranges[2 * r], hi = ranges[2 * r + 1];
    const int64_t total = (int64_t)(hi - lo) * vec_per_row;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
      const int row = lo + (int)(i / vec_per_row), c = (int)(i % vec_per_row);
      *reinterpret_cast<uint4*>(out + (int64_t)row * ld + 8 * c) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

extern "C" int qfx_zero_rows(void* out, int64_t ld, int ncols, const int* ranges, int n_ranges, void* stream) {
  QFX_CHECK_ARG(out && ranges && n_ranges > 0 && ncols % 8 == 0 && ld % 8 == 0, "qfx_zero_rows: bad arguments (ncols=%d)", ncols);
  zero_rows_kernel<<<2 * qfx::num_sms(), 256, 0, (cudaStream_t)stream>>>((bf16*)out, ld, ncols, ranges, n_ranges);
  LAUNCH_OK();
}

// ---------------------------------------------------------------------------------------------------------------------
// Deterministic variants (qfx.h): per-CTA partials into caller-owned scratch, then one fixed-order pass (launch_split_sum).
extern "C" int qfx_mod_grad_det(const void* g, int64_t ldg, const void* m, int64_t ldm, const float* mean, const float* rstd,
                                int rows_per_batch, float* sum_out, float* prod_out, int64_t ldo, int M, int D, float* scratch,
                                int64_t scratch_floats, void* stream) {
  QFX_CHECK_ARG(M > 0 && D > 0 && D % 8 == 0 && ldg % 8 == 0 && (m == nullptr || ldm % 8 == 0) && rows_per_batch > 0 &&
                    M % rows_per_batch == 0,
                "qfx_mod_grad_det: bad dims (D=%d, M=%d, rows_per_batch=%d)", D, M, rows_per_batch);
  QFX_CHECK_ARG((mean == nullptr) == (rstd == nullptr) && (mean == nullptr || m != nullptr), "qfx_mod_grad_det: mean/rstd need m");
  QFX_CHECK_ARG(aligned(g, 16) && aligned(m, 16), "qfx_mod_grad_det: g / m must be 16-byte aligned");
  const int B = M / rows_per_batch, cb = (D + 255) / 256;
  int splits = (QFX_DET_MODGRAD_CTAS + cb * B - 1) / (cb * B);
  splits = splits < 1 ? 1 : (splits > (rows_per_batch + 31) / 32 ? (rows_per_batch + 31) / 32 : splits);
  const int64_t need = (int64_t)splits * 2 * B * D;
  QFX_CHECK_ARG(scratch && scratch_floats >= need, "qfx_mod_grad_det: scratch holds %lld floats, needs %lld", (long long)scratch_floats,
                (long long)need);
  mod_grad_kernel<true><<<dim3(cb, B, splits), 256, 0, (cudaStream_t)stream>>>((const bf16*)g, ldg, (const bf16*)m, ldm, mean, rstd,
                                                                              rows_per_batch, scratch, scratch, D, D);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 2LL * B * D; S.splits = splits; S.rows = 2 * B; S.cols = D;
  S.dst[0] = sum_out; S.dst[1] = m != nullptr ? prod_out : nullptr;
  S.rows_per_dst = B; S.cols_per_dst = D; S.ld_row = ldo; S.ld_col = 1; S.accumulate = 1;
  return launch_split_sum(S, (cudaStream_t)stream);
}

extern "C" int qfx_flow_loss_det(const void* pred, const void* x0, const void* noise, const float* w, float norm, float grad_scale,
                                 float* loss, void* dpred, int B, int L, int Ltot, int C, float* scratch, int64_t scratch_floats,
                                 void* stream) {
  QFX_CHECK_ARG(loss && B > 0 && L > 0 && Ltot >= L && C > 0, "qfx_flow_loss_det: bad arguments");
  QFX_CHECK_ARG(scratch && scratch_floats >= QFX_DET_LOSS_PARTIALS, "qfx_flow_loss_det: scratch holds %lld floats, needs %d",
                (long long)scratch_floats, QFX_DET_LOSS_PARTIALS);
  flow_loss_kernel<true><<<QFX_DET_LOSS_PARTIALS, 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)pred, (const bf16*)x0, (const bf16*)noise, w, norm, grad_scale, scratch, (bf16*)dpred, B, L, Ltot, C);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_LOSS_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = loss; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  return launch_split_sum(S, (cudaStream_t)stream);
}

extern "C" int qfx_lora_wgrad_det(const void* P, int64_t ldp, const void* Q, int64_t ldq, float* G, int64_t gs_i, int64_t gs_j, int M,
                                  int Dp, int r, float* scratch, int64_t scratch_floats, void* stream) {
  QFX_CHECK_ARG(r == 4 || r == 8 || r == 16 || r == 32 || r == 64, "qfx_lora_wgrad_det: rank %d unsupported (4/8/16/32/64)", r);
  QFX_CHECK_ARG(G && M > 0 && Dp > 0, "qfx_lora_wgrad_det: bad arguments");
  const int splits0 = (M + 511) / 512;
  const int rows = ((M + splits0 - 1) / splits0 + 63) / 64 * 64;
  const int splits = (M + rows - 1) / rows;
  const int64_t need = (int64_t)splits * Dp * r;
  QFX_CHECK_ARG(scratch && scratch_floats >= need, "qfx_lora_wgrad_det: scratch holds %lld floats, needs %lld", (long long)scratch_floats,
                (long long)need);
  dim3 grid((Dp + 127) / 128, splits);
#define WGD(R)                                                                                                                    \
  case R:                                                                                                                         \
    lora_wgrad_kernel<R, true><<<grid, 128, 0, (cudaStream_t)stream>>>((const bf16*)P, ldp, (const bf16*)Q, ldq, scratch, 0, 0, M, \
                                                                       Dp, rows);                                                 \
    break;
  switch (r) { WGD(4) WGD(8) WGD(16) WGD(32) WGD(64) }
#undef WGD
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = (int64_t)Dp * r; S.splits = splits; S.rows = Dp; S.cols = r;
  S.dst[0] = G; S.rows_per_dst = Dp; S.cols_per_dst = r; S.ld_row = gs_i; S.ld_col = gs_j; S.accumulate = 1;
  return launch_split_sum(S, (cudaStream_t)stream);
}

extern "C" int qfx_grad_finalize_det(const float* g, int64_t n, float pre_scale, float max_norm, float* sumsq, void* out_bf16,
                                     float* scratch, int64_t scratch_floats, void* stream) {
  QFX_CHECK_ARG(g && n > 0 && sumsq && out_bf16, "qfx_grad_finalize_det: bad arguments");
  QFX_CHECK_ARG(scratch && scratch_floats >= QFX_DET_NORM_PARTIALS, "qfx_grad_finalize_det: scratch holds %lld floats, needs %d",
                (long long)scratch_floats, QFX_DET_NORM_PARTIALS);
  sumsq_kernel<true><<<QFX_DET_NORM_PARTIALS, 256, 0, (cudaStream_t)stream>>>(g, n, pre_scale, scratch);
  QFX_CUDA(cudaGetLastError());
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = 1; S.splits = QFX_DET_NORM_PARTIALS; S.rows = S.cols = 1;
  S.dst[0] = sumsq; S.rows_per_dst = S.cols_per_dst = 1; S.accumulate = 0;
  int rc = launch_split_sum(S, (cudaStream_t)stream);
  if (rc) return rc;
  clip_cast_kernel<<<592, 256, 0, (cudaStream_t)stream>>>(g, n, pre_scale, sumsq, max_norm, (bf16*)out_bf16);
  LAUNCH_OK();
}
