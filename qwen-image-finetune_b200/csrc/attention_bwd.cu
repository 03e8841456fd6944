// Joint attention backward for sm_90a (head_dim 128): dQ, dK, dV from Q, K, V, dO, logsumexp and delta = rowsum(dO*O).
// This is the autograd backward of F.scaled_dot_product_attention as the reference runs it
// (/root/reference/src/qflux/models/transformer_qwenimage.py:329-337 under loss.backward(), base_trainer.py:528).
//
// One CTA per (128-key tile, batch*head), two warpgroups of 64 key rows each; thread 0 also issues the TMA loads (K and V once,
// a two-stage ring of 64-query tiles of Q and dO).  Scores are TRANSPOSED (row = key), so dK and dV stay in registers:
//     S^T  = K Q_i^T           wgmma SS   A = K (K-major)                 B = Q_i  (K-major)
//     dP^T = V dO_i^T          wgmma SS   A = V (K-major)                 B = dO_i (K-major)
//     P^T  = exp2(S^T c - L_q) ;  dS^T = P^T o (dP^T - delta_q) * scale      (registers; per-query L and delta are per column)
//     dV  += P^T dO_i          wgmma RS   A = P^T from registers          B = dO_i read MN-major
//     dK  += dS^T Q_i          wgmma RS   A = dS^T from registers         B = Q_i  read MN-major
//     dQ_i = dS K              wgmma SS   A = dS^T in shared memory read MN-major, B = K read MN-major; warpgroup w computes
//                              head-dim columns [64 w, 64 w + 64) over all 128 keys and adds them to the fp32 dQ accumulator with
//                              8-byte vector reductions (red.global.add.v2.f32) of adjacent column pairs.
// Keys >= kv_len[b] and text padding [txt_len[b], split) are masked per key ROW; queries past S get L = +inf (P = 0).
#include <stdlib.h>
#include <string.h>

#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"

namespace qfx {

struct AttnBwdParams {
  CUtensorMap tmK, tmV;    // bf16 [B*H, S, 128], box {64, 128, 1}
  CUtensorMap tmQ, tmdO;   // bf16 [B*H, S, 128], box {64, 64, 1}
  float* dQ;               // [B*H, S, 128] fp32, zeroed by the caller: every key tile adds its partial dQ
  bf16* dK;
  bf16* dV;
  const float* lse;        // log2 domain
  const float* delta;
  const int* kv_len;
  const int* txt_len;
  int split, S, H;
  float scale, scale_log2;
};

constexpr int BW_KV = 128 * 128 * 2;  // 32 KB: K or V tile, two 64-column swizzle atoms of 16 KB
constexpr int BW_KV_ATOM = 128 * 128;
constexpr int BW_Q = 64 * 128 * 2;    // 16 KB: Q_i or dO_i tile, two atoms of 8 KB
constexpr int BW_Q_ATOM = 64 * 128;
constexpr int BW_DS = 128 * 64 * 2;   // dS^T [128 keys x 64 queries] bf16, one atom per key row
constexpr int BW_SMEM = 2 * BW_KV + 4 * BW_Q + BW_DS + 1024 /*align slack*/ + 256;

__device__ __forceinline__ uint32_t mul_bf16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

__global__ void __launch_bounds__(256, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = smem_base, sV = smem_base + BW_KV;
  auto sQ = [&](int st) { return smem_base + 2 * BW_KV + st * BW_Q; };
  auto sdO = [&](int st) { return smem_base + 2 * BW_KV + (2 + st) * BW_Q; };
  const uint32_t sdS = smem_base + 2 * BW_KV + 4 * BW_Q;
  const uint32_t bar_base = sdS + BW_DS;
  const uint32_t kv_full = bar_base;
  auto q_full = [&](int st) { return bar_base + 8u * (1 + st); };

  const int kv0 = blockIdx.x * 128;
  const int bh = blockIdx.y;
  const int b = bh / P.H;
  const int kv_len = P.kv_len ? P.kv_len[b] : P.S;
  const int txt_len = P.txt_len ? P.txt_len[b] : P.split;
  // query tiles that hold only padding rows of a pad-to-max batch (positions >= kv_len[b]) carry dO = 0: nothing to add, skip them
  const int n_q = ((kv_len < P.S ? kv_len : P.S) + 63) / 64;
  // a fully masked key tile (beyond kv_len, or entirely inside the text padding) contributes nothing: it writes zeros
  const bool active = kv0 < kv_len && !(kv0 >= txt_len && kv0 + 128 <= P.split);

  const int cw = threadIdx.x >> 7;
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  float dk[64], dv[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) dk[e] = dv[e] = 0.f;

  if (active) {
    if (threadIdx.x == 0) {
      mbar_init(kv_full, 1);
      mbar_init(q_full(0), 1);
      mbar_init(q_full(1), 1);
      fence_barrier_init();
    }
    __syncthreads();
    auto load_q = [&](int i) {
      const int st = i & 1;
      mbar_expect_tx(q_full(st), 2 * BW_Q);
      tma_load_3d(sQ(st), &P.tmQ, q_full(st), 0, i * 64, bh);
      tma_load_3d(sQ(st) + BW_Q_ATOM, &P.tmQ, q_full(st), 64, i * 64, bh);
      tma_load_3d(sdO(st), &P.tmdO, q_full(st), 0, i * 64, bh);
      tma_load_3d(sdO(st) + BW_Q_ATOM, &P.tmdO, q_full(st), 64, i * 64, bh);
    };
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, 2 * BW_KV);
      tma_load_3d(sK, &P.tmK, kv_full, 0, kv0, bh);
      tma_load_3d(sK + BW_KV_ATOM, &P.tmK, kv_full, 64, kv0, bh);
      tma_load_3d(sV, &P.tmV, kv_full, 0, kv0, bh);
      tma_load_3d(sV + BW_KV_ATOM, &P.tmV, kv_full, 64, kv0, bh);
      load_q(0);
      if (n_q > 1) load_q(1);
    }
    bool key_ok[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int key = kv0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
      key_ok[hh] = key < kv_len && !(key >= txt_len && key < P.split);
    }
    const uint32_t aK = sK + cw * 64 * 128, aV = sV + cw * 64 * 128;
    mbar_wait(kv_full, 0);
    for (int i = 0; i < n_q; ++i) {
      const int st = i & 1;
      const int q0 = i * 64;
      float sc[32], dp[32];
      mbar_wait(q_full(st), (i >> 1) & 1);
      reg_fence(sc, 32);
      reg_fence(dp, 32);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_ss_n64<0, 0>(sc, sdesc_sw128(aK + (k >> 2) * BW_KV_ATOM + (k & 3) * 32, 16, 1024),
                           sdesc_sw128(sQ(st) + (k >> 2) * BW_Q_ATOM + (k & 3) * 32, 16, 1024), k != 0);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        wgmma_ss_n64<0, 0>(dp, sdesc_sw128(aV + (k >> 2) * BW_KV_ATOM + (k & 3) * 32, 16, 1024),
                           sdesc_sw128(sdO(st) + (k >> 2) * BW_Q_ATOM + (k & 3) * 32, 16, 1024), k != 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(sc, 32);
      reg_fence(dp, 32);
      // P^T and dS^T, packed as bf16 pairs in the accumulator layout (= the A fragments of the next contractions)
      uint32_t pa[16], da[16];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int q = q0 + 8 * jj + 2 * (l & 3);
        float2 L = make_float2(INFINITY, INFINITY), D = make_float2(0.f, 0.f);
        if (q < P.S) {
          L.x = P.lse[(int64_t)bh * P.S + q];
          D.x = P.delta[(int64_t)bh * P.S + q];
        }
        if (q + 1 < P.S) {
          L.y = P.lse[(int64_t)bh * P.S + q + 1];
          D.y = P.delta[(int64_t)bh * P.S + q + 1];
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = 4 * jj + 2 * hh;
          uint32_t p = pack_bf16(exp2f(sc[r] * P.scale_log2 - L.x), exp2f(sc[r + 1] * P.scale_log2 - L.y));
          if (!key_ok[hh]) p = 0u;
          // dS = P o (dP c - delta c): the bracket in fp32, rounded to bf16 and multiplied by the bf16 P as a packed pair
          const uint32_t d = mul_bf16x2(p, pack_bf16(dp[r] * P.scale - D.x * P.scale, dp[r + 1] * P.scale - D.y * P.scale));
          pa[2 * jj + hh] = p;
          da[2 * jj + hh] = d;
        }
      }
      // dS^T to shared memory: [128 keys][64 queries], 128B-swizzled rows (the MN-major A operand of dQ)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int kr = cw * 64 + 16 * w + (l >> 2) + 8 * hh;
          const uint32_t addr = sdS + kr * 128 + ((uint32_t)(jj ^ (kr & 7)) << 4) + (l & 3) * 4;
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(da[2 * jj + hh]) : "memory");
        }
      fence_proxy_async_smem();
      // A fragment of k-chunk c (queries 16 c ..): {pair(jj = 2c, h 0), pair(2c, h 1), pair(2c + 1, h 0), pair(2c + 1, h 1)}
      reg_fence(dv, 64);
      reg_fence(dk, 64);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 4; ++c) wgmma_rs_n128<1>(dv, pa + 4 * c, sdesc_sw128(sdO(st) + c * 2048, BW_Q_ATOM, 1024), 1);
#pragma unroll
      for (int c = 0; c < 4; ++c) wgmma_rs_n128<1>(dk, da + 4 * c, sdesc_sw128(sQ(st) + c * 2048, BW_Q_ATOM, 1024), 1);
      wgmma_commit();
      named_bar(1, 256);  // dS^T of both warpgroups is in shared memory
      float dq[32];
      reg_fence(dq, 32);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 8; ++c)
        wgmma_ss_n64<1, 1>(dq, sdesc_sw128(sdS + c * 2048, BW_Q_ATOM, 1024), sdesc_sw128(sK + cw * BW_KV_ATOM + c * 2048, BW_KV_ATOM, 1024),
                           c != 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dq, 32);
      reg_fence(dv, 64);
      reg_fence(dk, 64);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int q = q0 + 16 * w + (l >> 2) + 8 * hh;
        if (q < P.S) {
          float* dst = P.dQ + ((int64_t)bh * P.S + q) * 128 + cw * 64 + 2 * (l & 3);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) red_add_v2(dst + 8 * jj, dq[4 * jj + 2 * hh], dq[4 * jj + 2 * hh + 1]);
        }
      }
      named_bar(1, 256);  // stage st and the dS^T buffer are free
      if (threadIdx.x == 0 && i + 2 < n_q) load_q(i + 2);
    }
  }
  // epilogue: dK, dV rows of this warpgroup's 64 keys (zeros for a fully masked key tile)
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int key = kv0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
    if (key >= P.S) continue;
    bf16* dK = P.dK + ((int64_t)bh * P.S + key) * 128 + 2 * (l & 3);
    bf16* dV = P.dV + ((int64_t)bh * P.S + key) * 128 + 2 * (l & 3);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      *reinterpret_cast<uint32_t*>(dK + 8 * jj) = pack_bf16(dk[4 * jj + 2 * hh], dk[4 * jj + 2 * hh + 1]);
      *reinterpret_cast<uint32_t*>(dV + 8 * jj) = pack_bf16(dv[4 * jj + 2 * hh], dv[4 * jj + 2 * hh + 1]);
    }
  }
}

int make_qkv_tmap(CUtensorMap* m, const void* base, int BH, int S);  // attention_fwd.cu

static int make_q64_tmap(CUtensorMap* m, const void* base, int BH, int S) {
  uint64_t dims[3] = {128, (uint64_t)S, (uint64_t)BH};
  uint64_t strides[2] = {128 * 2, (uint64_t)S * 128 * 2};
  uint32_t box[3] = {64, 64, 1};
  return make_tmap_bf16(m, base, 3, dims, strides, box);
}

}  // namespace qfx

using namespace qfx;

/* All of Q, K, V, dO, dK, dV: [B, H, S, 128] bf16; dQ_accum: [B, H, S, 128] fp32, MUST be zeroed by the caller (every key tile
 * adds its partial dQ into it).  lse: log2-domain logsumexp from qfx_attn_fwd; delta = rowsum(dO*O). */
extern "C" int qfx_attn_bwd(const void* Q, const void* K, const void* V, const void* dO, const float* lse, const float* delta,
                            float* dQ_accum, void* dK, void* dV, const int* kv_len, const int* txt_len, int split, int B, int H,
                            int S, float softmax_scale, void* stream) {
  QFX_CHECK_ARG(B > 0 && H > 0 && S > 0 && dQ_accum && dK && dV && lse && delta, "qfx_attn_bwd: bad arguments");
  QFX_CHECK_ARG(!txt_len || (split > 0 && split <= S), "qfx_attn_bwd: txt_len needs 0 < split <= S (split=%d S=%d)", split, S);
  // dQ is reduced into as 8-byte pairs, dK / dV are stored as 4-byte pairs
  QFX_CHECK_ARG(((uintptr_t)dQ_accum & 7) == 0 && ((uintptr_t)dK & 3) == 0 && ((uintptr_t)dV & 3) == 0,
                "qfx_attn_bwd: dQ_accum must be 8-byte aligned, dK / dV 4-byte aligned");
  AttnBwdParams P;
  memset(&P, 0, sizeof(P));
  int rc;
  if ((rc = make_qkv_tmap(&P.tmK, K, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&P.tmV, V, B * H, S))) return rc;
  if ((rc = make_q64_tmap(&P.tmQ, Q, B * H, S))) return rc;
  if ((rc = make_q64_tmap(&P.tmdO, dO, B * H, S))) return rc;
  P.dQ = dQ_accum; P.dK = (bf16*)dK; P.dV = (bf16*)dV; P.lse = lse; P.delta = delta; P.kv_len = kv_len; P.txt_len = txt_len;
  P.split = txt_len ? split : 0; P.S = S; P.H = H;
  P.scale = softmax_scale;
  P.scale_log2 = softmax_scale * 1.4426950408889634f;
  static bool attr_done = false;
  if (!attr_done) {
    QFX_CUDA(cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM));
    attr_done = true;
  }
  dim3 grid((S + 127) / 128, B * H);
  attn_bwd_kernel<<<grid, 256, BW_SMEM, (cudaStream_t)stream>>>(P);
  QFX_CUDA(cudaGetLastError());
  return 0;
}
