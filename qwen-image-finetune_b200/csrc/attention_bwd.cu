// Joint attention backward for sm_90a (head_dim 128): dQ, dK, dV from Q, K, V, dO, logsumexp and delta = rowsum(dO*O).
// This is the autograd backward of F.scaled_dot_product_attention as the reference runs it
// (/root/reference/src/qflux/models/transformer_qwenimage.py:329-337 under loss.backward(), base_trainer.py:528).
//
// One CTA per (128-key tile, batch*head), two warpgroups of 64 key rows each; thread 0 also issues the TMA loads (K and V once,
// a three-stage ring of 64-query tiles of Q and dO).  Scores are TRANSPOSED (row = key), so dK and dV stay in registers:
//     S^T  = K Q_i^T           wgmma SS   A = K (K-major)                 B = Q_i  (K-major)
//     dP^T = V dO_i^T          wgmma SS   A = V (K-major)                 B = dO_i (K-major)
//     P^T  = exp2(S^T c - L_q) ;  dS^T = P^T o (dP^T - delta_q) * scale      (registers; per-query L and delta are per column)
//     dV  += P^T dO_i          wgmma RS   A = P^T from registers          B = dO_i read MN-major
//     dK  += dS^T Q_i          wgmma RS   A = dS^T from registers         B = Q_i  read MN-major
//     dQ_i = dS K              wgmma SS   A = dS^T in shared memory read MN-major, B = K read MN-major; warpgroup w computes
//                              head-dim columns [64 w, 64 w + 64) over all 128 keys, stages them in shared memory and adds them
//                              to the fp32 dQ accumulator with one TMA reduction (cp.reduce.async.bulk.tensor .add.f32).
// The warpgroups meet once per tile, at the dS^T hand-off: each arrives on ds_full[i & 1] after writing its dS^T rows and waits on
// it only before the dQ product, with its dK / dV products already issued.  dS^T is double-buffered, so a warpgroup that runs ahead
// never overwrites rows the other still reads.  lse and delta of tile i + 1 are read from global memory by warpgroup 0 while tile
// i's S^T / dP^T run, and published to shared memory through the same barrier.  A Q / dO stage is released to the loader by an
// mbarrier (q_empty, one arrival per warpgroup) once both warpgroups' products on it have completed.
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
  CUtensorMap tmdQ;        // fp32 [B*H, S, 128], box {32, 64, 1}, 128B swizzle: the dQ reduction (attn_bwd_kernel<true>)
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
constexpr int BW_STAGES = 3;          // Q / dO ring depth
constexpr int BW_DS = 128 * 64 * 2;   // dS^T [128 keys x 64 queries] bf16, one atom per key row; two buffers
constexpr int BW_DQ = 64 * 64 * 4;    // one warpgroup's fp32 dQ tile [64 queries x 64 columns]: two 128B-swizzled boxes of 32 columns
constexpr int BW_LD = 2 * 64 * 4;     // lse[64] then delta[64] of one query tile; two buffers
constexpr int BW_OFF_Q = 2 * BW_KV;
constexpr int BW_OFF_DS = BW_OFF_Q + 2 * BW_STAGES * BW_Q;
constexpr int BW_OFF_DQ = BW_OFF_DS + 2 * BW_DS;
constexpr int BW_OFF_LD = BW_OFF_DQ + 2 * BW_DQ;
constexpr int BW_OFF_BAR = BW_OFF_LD + 2 * BW_LD;
constexpr int BW_SMEM = BW_OFF_BAR + 128 /*barriers*/ + 1024 /*align slack*/;
static_assert(BW_SMEM <= 227 * 1024, "attn_bwd_kernel: shared memory over the sm_90 opt-in limit");

__device__ __forceinline__ uint32_t mul_bf16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  return r;
}

// kDQ = false: dK and dV only (the deterministic backward; its dQ comes from attn_bwd_dq_kernel below).
template <bool kDQ = true>
__global__ void __launch_bounds__(256, 1) attn_bwd_kernel(const __grid_constant__ AttnBwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = smem_base, sV = smem_base + BW_KV;
  auto sQ = [&](int st) { return smem_base + BW_OFF_Q + st * 2 * BW_Q; };
  auto sdO = [&](int st) { return smem_base + BW_OFF_Q + st * 2 * BW_Q + BW_Q; };
  auto sdS = [&](int b) { return smem_base + BW_OFF_DS + b * BW_DS; };
  auto sLD = [&](int b) { return smem_base + BW_OFF_LD + b * BW_LD; };
  const uint32_t bar_base = smem_base + BW_OFF_BAR;
  const uint32_t kv_full = bar_base;
  auto q_full = [&](int st) { return bar_base + 8u * (1 + st); };
  auto q_empty = [&](int st) { return bar_base + 8u * (1 + BW_STAGES + st); };
  auto ds_full = [&](int b) { return bar_base + 8u * (1 + 2 * BW_STAGES + b); };

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
    // warpgroup 0 thread t reads lse (t < 64) or delta (t >= 64) of query 64 i + (t & 63); queries past S get L = +inf, delta = 0
    auto load_ld = [&](int i) {
      const int q = i * 64 + (t & 63);
      return q < P.S ? (t < 64 ? P.lse : P.delta)[(int64_t)bh * P.S + q] : (t < 64 ? INFINITY : 0.f);
    };
    if (threadIdx.x == 0) {
      mbar_init(kv_full, 1);
      for (int st = 0; st < BW_STAGES; ++st) {
        mbar_init(q_full(st), 1);
        mbar_init(q_empty(st), 2);
      }
      mbar_init(ds_full(0), 256);
      mbar_init(ds_full(1), 256);
      fence_barrier_init();
    }
    if (cw == 0) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sLD(0) + 4 * t), "f"(load_ld(0)) : "memory");
    __syncthreads();
    auto load_q = [&](int i) {
      const int st = i % BW_STAGES;
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
      for (int i = 0; i < BW_STAGES && i < n_q; ++i) load_q(i);
    }
    bool key_ok[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int key = kv0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
      key_ok[hh] = key < kv_len && !(key >= txt_len && key < P.split);
    }
    const uint32_t aK = sK + cw * 64 * 128, aV = sV + cw * 64 * 128;
    const uint32_t sdQ = smem_base + BW_OFF_DQ + cw * BW_DQ;
    mbar_wait(kv_full, 0);
    for (int i = 0; i < n_q; ++i) {
      const int st = i % BW_STAGES, db = i & 1;
      const int q0 = i * 64;
      float sc[32], dp[32];
      mbar_wait(q_full(st), (i / BW_STAGES) & 1);
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
      // the next tile's lse / delta, read while the tensor cores run this tile's products
      const bool ld_next = cw == 0 && i + 1 < n_q;
      const float ld_val = ld_next ? load_ld(i + 1) : 0.f;
      wgmma_wait<0>();
      reg_fence(sc, 32);
      reg_fence(dp, 32);
      // P^T and dS^T, packed as bf16 pairs in the accumulator layout (= the A fragments of the next contractions)
      uint32_t pa[16], da[16];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const uint32_t lq = sLD(db) + 4 * (8 * jj + 2 * (l & 3));
        float2 L, D;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(L.x), "=f"(L.y) : "r"(lq) : "memory");
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(D.x), "=f"(D.y) : "r"(lq + 256) : "memory");
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
      if constexpr (kDQ) {
        // dS^T to shared memory: [128 keys][64 queries], 128B-swizzled rows (the MN-major A operand of dQ)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int kr = cw * 64 + 16 * w + (l >> 2) + 8 * hh;
            const uint32_t addr = sdS(db) + kr * 128 + ((uint32_t)(jj ^ (kr & 7)) << 4) + (l & 3) * 4;
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(da[2 * jj + hh]) : "memory");
          }
        fence_proxy_async_smem();
      }
      // buffer db ^ 1 was last read in tile i - 1, before this warpgroup's wait on ds_full[db ^ 1]
      if (ld_next) asm volatile("st.shared.f32 [%0], %1;" ::"r"(sLD(db ^ 1) + 4 * t), "f"(ld_val) : "memory");
      mbar_arrive(ds_full(db));
      // A fragment of k-chunk c (queries 16 c ..): {pair(jj = 2c, h 0), pair(2c, h 1), pair(2c + 1, h 0), pair(2c + 1, h 1)}
      reg_fence(dv, 64);
      reg_fence(dk, 64);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 4; ++c) wgmma_rs_n128<1>(dv, pa + 4 * c, sdesc_sw128(sdO(st) + c * 2048, BW_Q_ATOM, 1024), 1);
#pragma unroll
      for (int c = 0; c < 4; ++c) wgmma_rs_n128<1>(dk, da + 4 * c, sdesc_sw128(sQ(st) + c * 2048, BW_Q_ATOM, 1024), 1);
      wgmma_commit();
      // dS^T of both warpgroups is in shared memory, and lse / delta of tile i + 1 are published
      mbar_wait(ds_full(db), (i >> 1) & 1);
      if constexpr (kDQ) {
        float dq[32];
        reg_fence(dq, 32);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < 8; ++c)
          wgmma_ss_n64<1, 1>(dq, sdesc_sw128(sdS(db) + c * 2048, BW_Q_ATOM, 1024),
                             sdesc_sw128(sK + cw * BW_KV_ATOM + c * 2048, BW_KV_ATOM, 1024), c != 0);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(dq, 32);
        reg_fence(dv, 64);
        reg_fence(dk, 64);
        if (t == 0) {
          mbar_arrive(q_empty(st));
          tma_store_wait_read<0>();  // the previous tile's dQ reduction has read the staging tile
        }
        named_bar(1 + cw, 128);
        // dQ_i columns [64 cw, 64 cw + 64) to the staging tile: box jj / 4 holds columns 8 jj .. 8 jj + 7 of query rows 0..63,
        // 128 B per row, its 16-byte chunks swizzled by row % 8 (the layout the tensor map's 128B swizzle reads)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = 16 * w + (l >> 2) + 8 * hh;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const uint32_t chunk = 2 * (jj & 3) + ((l & 3) >> 1);
            const uint32_t addr = sdQ + (jj >> 2) * (BW_DQ / 2) + row * 128 + ((chunk ^ (row & 7)) << 4) + (l & 1) * 8;
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(dq[4 * jj + 2 * hh]), "f"(dq[4 * jj + 2 * hh + 1])
                         : "memory");
          }
        }
        fence_proxy_async_smem();
        named_bar(1 + cw, 128);
        if (t == 0) {
          tma_reduce_add_3d(&P.tmdQ, sdQ, cw * 64, q0, bh);
          tma_reduce_add_3d(&P.tmdQ, sdQ + BW_DQ / 2, cw * 64 + 32, q0, bh);
          tma_store_commit();
        }
      } else {
        wgmma_wait<0>();
        reg_fence(dv, 64);
        reg_fence(dk, 64);
        if (t == 0) mbar_arrive(q_empty(st));
      }
      // stage st is refilled once both warpgroups' products on it have completed
      if (threadIdx.x == 0 && i + BW_STAGES < n_q) {
        mbar_wait(q_empty(st), (i / BW_STAGES) & 1);
        load_q(i + BW_STAGES);
      }
    }
    if (kDQ && t == 0) tma_store_wait<0>();
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

// Deterministic dQ: query-major, one CTA per (128-query tile, batch*head), two warpgroups of 64 query rows each; thread 0 issues
// the TMA loads (Q and dO once, a two-stage ring of 64-key tiles of K and V).  Per key tile j the scores are recomputed:
//     S   = Q K_j^T            wgmma SS   A = Q  (K-major)     B = K_j (K-major)
//     dP  = dO V_j^T           wgmma SS   A = dO (K-major)     B = V_j (K-major)
//     P   = exp2(S c - L_q) ;  dS = P o (dP - delta_q) * scale     (registers; the same bf16 rounding points as attn_bwd_kernel)
//     dQ += dS K_j             wgmma RS   A = dS from registers     B = K_j read MN-major
// over the key tiles in ascending order, so every dQ element is one register sum in a fixed order, added ONCE to the caller's buffer.
// 64-key tiles keep the three accumulators (S, dP: 32 registers each, dQ: 64) well inside the register file.
constexpr int DQ_KT = 64 * 128 * 2;     // 16 KB: K_j or V_j tile, two atoms of 8 KB
constexpr int DQ_KT_ATOM = 64 * 128;
constexpr int DQ_QT = 128 * 128 * 2;    // 32 KB: Q or dO tile, two atoms of 16 KB
constexpr int DQ_QT_ATOM = 128 * 128;
constexpr int DQ_SMEM = 2 * DQ_QT + 4 * DQ_KT + 1024 /*align slack*/ + 256;

__global__ void __launch_bounds__(256, 1) attn_bwd_dq_kernel(const __grid_constant__ AttnBwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = smem_base, sdO = smem_base + DQ_QT;
  auto sK = [&](int st) { return smem_base + 2 * DQ_QT + st * DQ_KT; };
  auto sV = [&](int st) { return smem_base + 2 * DQ_QT + (2 + st) * DQ_KT; };
  const uint32_t bar_base = smem_base + 2 * DQ_QT + 4 * DQ_KT;
  const uint32_t q_full = bar_base;
  auto kv_full = [&](int st) { return bar_base + 8u * (1 + st); };

  const int q0 = blockIdx.x * 128;
  const int bh = blockIdx.y;
  const int b = bh / P.H;
  const int kv_len = min(P.kv_len ? P.kv_len[b] : P.S, P.S);
  const int txt_len = P.txt_len ? P.txt_len[b] : P.split;
  // query tiles of only padding rows (>= kv_len[b]) add nothing; key tiles wholly inside the text padding [txt_len, split) are
  // skipped: the live tiles are [0, n_txt) and [img0, n_k)
  const int n_k = (kv_len + 63) / 64;
  const int n_txt = min((txt_len + 63) / 64, n_k);
  const int img0 = max(P.split / 64, n_txt);
  const int n_live = n_txt + max(0, n_k - img0);
  if (q0 >= kv_len || n_live == 0) return;
  auto tile = [&](int i) { return i < n_txt ? i : img0 + (i - n_txt); };

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_kv = [&](int i) {
    const int st = i & 1, k0 = tile(i) * 64;
    mbar_expect_tx(kv_full(st), 2 * DQ_KT);
    tma_load_3d(sK(st), &P.tmK, kv_full(st), 0, k0, bh);
    tma_load_3d(sK(st) + DQ_KT_ATOM, &P.tmK, kv_full(st), 64, k0, bh);
    tma_load_3d(sV(st), &P.tmV, kv_full(st), 0, k0, bh);
    tma_load_3d(sV(st) + DQ_KT_ATOM, &P.tmV, kv_full(st), 64, k0, bh);
  };
  if (threadIdx.x == 0) {
    mbar_expect_tx(q_full, 2 * DQ_QT);
    tma_load_3d(sQ, &P.tmQ, q_full, 0, q0, bh);
    tma_load_3d(sQ + DQ_QT_ATOM, &P.tmQ, q_full, 64, q0, bh);
    tma_load_3d(sdO, &P.tmdO, q_full, 0, q0, bh);
    tma_load_3d(sdO + DQ_QT_ATOM, &P.tmdO, q_full, 64, q0, bh);
    load_kv(0);
    if (n_live > 1) load_kv(1);
  }

  const int cw = threadIdx.x >> 7;
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  float L[2], D[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = q0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
    L[hh] = q < P.S ? P.lse[(int64_t)bh * P.S + q] : INFINITY;  // queries past S: P = 0
    D[hh] = q < P.S ? P.delta[(int64_t)bh * P.S + q] * P.scale : 0.f;
  }
  float dq[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) dq[e] = 0.f;
  const uint32_t aQ = sQ + cw * 64 * 128, adO = sdO + cw * 64 * 128;
  mbar_wait(q_full, 0);
  for (int i = 0; i < n_live; ++i) {
    const int st = i & 1, k0 = tile(i) * 64;
    float sc[32], dp[32];
    mbar_wait(kv_full(st), (i >> 1) & 1);
    reg_fence(sc, 32);
    reg_fence(dp, 32);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma_ss_n64<0, 0>(sc, sdesc_sw128(aQ + (k >> 2) * DQ_QT_ATOM + (k & 3) * 32, 16, 1024),
                         sdesc_sw128(sK(st) + (k >> 2) * DQ_KT_ATOM + (k & 3) * 32, 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma_ss_n64<0, 0>(dp, sdesc_sw128(adO + (k >> 2) * DQ_QT_ATOM + (k & 3) * 32, 16, 1024),
                         sdesc_sw128(sV(st) + (k >> 2) * DQ_KT_ATOM + (k & 3) * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sc, 32);
    reg_fence(dp, 32);
    // keys >= kv_len[b] and the text padding [txt_len[b], split) get P = 0 (only tiles that contain such keys pay for the test)
    const bool partial = k0 + 64 > kv_len || (txt_len < P.split && k0 < P.split && k0 + 64 > txt_len);
    uint32_t da[16];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = 4 * jj + 2 * hh;
        float p0 = exp2f(sc[r] * P.scale_log2 - L[hh]), p1 = exp2f(sc[r + 1] * P.scale_log2 - L[hh]);
        if (partial) {
          const int key = k0 + 8 * jj + 2 * (l & 3);
          if (key >= kv_len || (key >= txt_len && key < P.split)) p0 = 0.f;
          if (key + 1 >= kv_len || (key + 1 >= txt_len && key + 1 < P.split)) p1 = 0.f;
        }
        da[2 * jj + hh] = mul_bf16x2(pack_bf16(p0, p1), pack_bf16(dp[r] * P.scale - D[hh], dp[r + 1] * P.scale - D[hh]));
      }
    reg_fence(dq, 64);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 4; ++c) wgmma_rs_n128<1>(dq, da + 4 * c, sdesc_sw128(sK(st) + c * 2048, DQ_KT_ATOM, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dq, 64);
    named_bar(1, 256);  // both warpgroups are done with stage st
    if (threadIdx.x == 0 && i + 2 < n_live) load_kv(i + 2);
  }
  // epilogue: one read-modify-write per element of the rows < kv_len[b]
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = q0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
    if (q >= kv_len) continue;
    float2* dst = reinterpret_cast<float2*>(P.dQ + ((int64_t)bh * P.S + q) * 128 + 2 * (l & 3));
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      float2 v = dst[4 * jj];
      v.x += dq[4 * jj + 2 * hh];
      v.y += dq[4 * jj + 2 * hh + 1];
      dst[4 * jj] = v;
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

// fp32 dQ [B*H, S, 128] as the reduction target of attn_bwd_kernel<true>: boxes of 32 columns x 64 query rows, 128B-swizzled
static int make_dq_tmap(CUtensorMap* m, const void* base, int BH, int S) {
  uint64_t dims[3] = {128, (uint64_t)S, (uint64_t)BH};
  uint64_t strides[2] = {128 * 4, (uint64_t)S * 128 * 4};
  uint32_t box[3] = {32, 64, 1};
  return make_tmap_f32(m, base, 3, dims, strides, box);
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
  // ... and through a tensor map, whose base address must be 16-byte aligned
  QFX_CHECK_ARG(((uintptr_t)dQ_accum & 15) == 0, "qfx_attn_bwd: dQ_accum must be 16-byte aligned");
  AttnBwdParams P;
  memset(&P, 0, sizeof(P));
  int rc;
  if ((rc = make_dq_tmap(&P.tmdQ, dQ_accum, B * H, S))) return rc;
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
    QFX_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM));
    attr_done = true;
  }
  dim3 grid((S + 127) / 128, B * H);
  attn_bwd_kernel<true><<<grid, 256, BW_SMEM, (cudaStream_t)stream>>>(P);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

/* Deterministic variant (see qfx.h): the same arguments and the same dQ_accum contract, but dK / dV come from attn_bwd_kernel<false>
 * and dQ from attn_bwd_dq_kernel, which adds each element once — no floating-point atomics, bit-reproducible run to run. */
extern "C" int qfx_attn_bwd_det(const void* Q, const void* K, const void* V, const void* dO, const float* lse, const float* delta,
                                float* dQ_accum, void* dK, void* dV, const int* kv_len, const int* txt_len, int split, int B, int H,
                                int S, float softmax_scale, void* stream) {
  QFX_CHECK_ARG(B > 0 && H > 0 && S > 0 && dQ_accum && dK && dV && lse && delta, "qfx_attn_bwd_det: bad arguments");
  QFX_CHECK_ARG(!txt_len || (split > 0 && split <= S), "qfx_attn_bwd_det: txt_len needs 0 < split <= S (split=%d S=%d)", split, S);
  // dQ is read and written as 8-byte pairs, dK / dV are stored as 4-byte pairs
  QFX_CHECK_ARG(((uintptr_t)dQ_accum & 7) == 0 && ((uintptr_t)dK & 3) == 0 && ((uintptr_t)dV & 3) == 0,
                "qfx_attn_bwd_det: dQ_accum must be 8-byte aligned, dK / dV 4-byte aligned");
  AttnBwdParams P, Pq;
  memset(&P, 0, sizeof(P));
  memset(&Pq, 0, sizeof(Pq));
  int rc;
  if ((rc = make_qkv_tmap(&P.tmK, K, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&P.tmV, V, B * H, S))) return rc;
  if ((rc = make_q64_tmap(&P.tmQ, Q, B * H, S))) return rc;
  if ((rc = make_q64_tmap(&P.tmdO, dO, B * H, S))) return rc;
  // the dQ kernel's roles are swapped: 128-row Q / dO tiles, 64-row K / V tiles
  if ((rc = make_q64_tmap(&Pq.tmK, K, B * H, S))) return rc;
  if ((rc = make_q64_tmap(&Pq.tmV, V, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&Pq.tmQ, Q, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&Pq.tmdO, dO, B * H, S))) return rc;
  P.dQ = dQ_accum; P.dK = (bf16*)dK; P.dV = (bf16*)dV; P.lse = lse; P.delta = delta; P.kv_len = kv_len; P.txt_len = txt_len;
  P.split = txt_len ? split : 0; P.S = S; P.H = H;
  P.scale = softmax_scale;
  P.scale_log2 = softmax_scale * 1.4426950408889634f;
  Pq.dQ = P.dQ; Pq.lse = lse; Pq.delta = delta; Pq.kv_len = kv_len; Pq.txt_len = txt_len;
  Pq.split = P.split; Pq.S = S; Pq.H = H; Pq.scale = P.scale; Pq.scale_log2 = P.scale_log2;
  static bool attr_done = false;
  if (!attr_done) {
    QFX_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BW_SMEM));
    QFX_CUDA(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
    attr_done = true;
  }
  attn_bwd_kernel<false><<<dim3((S + 127) / 128, B * H), 256, BW_SMEM, (cudaStream_t)stream>>>(P);
  QFX_CUDA(cudaGetLastError());
  attn_bwd_dq_kernel<<<dim3((S + 127) / 128, B * H), 256, DQ_SMEM, (cudaStream_t)stream>>>(Pq);
  QFX_CUDA(cudaGetLastError());
  return 0;
}
