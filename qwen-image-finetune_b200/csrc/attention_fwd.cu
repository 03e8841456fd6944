// Joint (text+image) non-causal attention forward for sm_90a, head_dim 128, bf16 in / fp32 softmax.
// Replaces `dispatch_attention_fn` -> F.scaled_dot_product_attention on the concatenated [txt; img] sequence
// (/root/reference/src/qflux/models/transformer_qwenimage.py:322-345, transformer_flux.py:149-156).
//
// One CTA per (128-query tile, batch*head), two warpgroups of 64 query rows each; thread 0 also issues the TMA loads of a
// two-stage K / V ring.  Per 128-key tile j:
//     S   = Q K_j^T          wgmma SS, both operands K-major (d contiguous), fp32 accumulator in registers
//     P   = exp2(S*c - m)    in registers; row max / sum reduced over the four threads of a quad
//     O  += P V_j            wgmma RS: A = P straight from the accumulator registers (bf16), B = V (MN-major: d contiguous)
#include <stdlib.h>
#include <string.h>

#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"

namespace qfx {

constexpr int ATT_D = 128;
constexpr int ATT_BQ = 128;
constexpr int ATT_BK = 128;
constexpr int TILE_BYTES = 128 * 128 * 2;  // 32 KB: two 64-wide 128B-swizzle atoms of [128 rows x 128 B]
constexpr int ATOM_BYTES = 128 * 128;      // 16 KB

struct AttnFwdParams {
  CUtensorMap tmQ, tmK, tmV;  // [B*H, S, 128] bf16, box {64, 128, 1}
  bf16* out0;                 // rows with joint position s < split  -> out0[(b*rows0 + s) * ld0 + h*128 ..]
  bf16* out1;                 // rows with s >= split               -> out1[(b*rows1 + s - split) * ld1 + h*128 ..]
  int64_t ld0, ld1;
  int rows0, rows1, split;
  float* lse;          // [B*H, S] log2-domain logsumexp:  m + log2(l)
  const int* kv_len;   // [B] end of the valid joint sequence per sample (NULL: S): keys >= kv_len[b] are masked
  const int* txt_len;  // [B] valid text tokens per sample (NULL: split): keys in [txt_len[b], split) are masked too
  int S, H;
  float scale_log2;    // (1/sqrt(d)) * log2(e)
};

constexpr int ATT_SMEM = 5 * TILE_BYTES + 1024 /*align slack*/ + 256;  // Q, K x2, V x2, barriers

// A query tile that holds only padding rows of a pad-to-max batch (every query position >= kv_len[b], all of them image rows): the
// output rows become zeros (they feed row-wise kernels and must stay finite) and no attention math runs.
__device__ __forceinline__ bool attn_fwd_skip_padding_tile(const AttnFwdParams& P, int q0, int b, int h, int bh, int kv_len) {
  if (q0 < kv_len || q0 < P.split) return false;
  for (int idx = threadIdx.x; idx < ATT_BQ * 16; idx += blockDim.x) {
    const int sq = q0 + (idx >> 4), c = idx & 15;
    if (sq < P.S) {
      bf16* dst = P.out1 + ((int64_t)b * P.rows1 + (sq - P.split)) * P.ld1 + h * ATT_D + c * 8;
      *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
      if (P.lse && c == 0) P.lse[(int64_t)bh * P.S + sq] = 0.f;
    }
  }
  return true;
}

__global__ void __launch_bounds__(256, 1) attn_fwd_kernel(const __grid_constant__ AttnFwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;  // 128B-swizzle atoms need 1024 B alignment
  const uint32_t sQ = smem_base;
  auto sK = [&](int s) { return smem_base + TILE_BYTES * (1 + s); };
  auto sV = [&](int s) { return smem_base + TILE_BYTES * (3 + s); };
  const uint32_t bar_base = smem_base + 5 * TILE_BYTES;
  const uint32_t q_full = bar_base;
  auto kv_full = [&](int s) { return bar_base + 8u * (1 + s); };

  const int q0 = blockIdx.x * ATT_BQ;
  const int bh = blockIdx.y;
  const int b = bh / P.H, h = bh - b * P.H;
  const int kv_len = P.kv_len ? P.kv_len[b] : P.S;
  const int txt_len = P.txt_len ? P.txt_len[b] : P.split;
  const int n_tiles = (kv_len + ATT_BK - 1) / ATT_BK;
  if (attn_fwd_skip_padding_tile(P, q0, b, h, bh, kv_len)) return;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    mbar_init(kv_full(0), 1);
    mbar_init(kv_full(1), 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(kv_full(s), 2 * TILE_BYTES);
    tma_load_3d(sK(s), &P.tmK, kv_full(s), 0, j * ATT_BK, bh);
    tma_load_3d(sK(s) + ATOM_BYTES, &P.tmK, kv_full(s), 64, j * ATT_BK, bh);
    tma_load_3d(sV(s), &P.tmV, kv_full(s), 0, j * ATT_BK, bh);
    tma_load_3d(sV(s) + ATOM_BYTES, &P.tmV, kv_full(s), 64, j * ATT_BK, bh);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&P.tmQ);
    tma_prefetch_desc(&P.tmK);
    tma_prefetch_desc(&P.tmV);
    mbar_expect_tx(q_full, TILE_BYTES);
    tma_load_3d(sQ, &P.tmQ, q_full, 0, q0, bh);
    tma_load_3d(sQ + ATOM_BYTES, &P.tmQ, q_full, 64, q0, bh);
    load_kv(0);
    if (n_tiles > 1) load_kv(1);
  }

  const int cw = threadIdx.x >> 7;  // warpgroup: query rows 64 cw .. + 63 of the tile
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  float o[64], sc[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) o[e] = 0.f;
  float m_used[2] = {-INFINITY, -INFINITY}, lsum[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);
  const uint32_t aQ = sQ + cw * 64 * 128;
  for (int j = 0; j < n_tiles; ++j) {
    const int s = j & 1;
    mbar_wait(kv_full(s), (j >> 1) & 1);
    reg_fence(sc, 64);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)
      wgmma_ss_n128<0, 0>(sc, sdesc_sw128(aQ + (k >> 2) * ATOM_BYTES + (k & 3) * 32, 16, 1024),
                          sdesc_sw128(sK(s) + (k >> 2) * ATOM_BYTES + (k & 3) * 32, 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sc, 64);
    // keys >= kv_len[b] and the text padding [txt_len[b], split) are masked (only tiles that contain such keys pay for the test)
    const int k0 = j * ATT_BK;
    if (k0 + ATT_BK > kv_len || (txt_len < P.split && k0 < P.split && k0 + ATT_BK > txt_len)) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = k0 + 8 * jj + 2 * (l & 3) + e;
          if (key >= kv_len || (key >= txt_len && key < P.split)) sc[4 * jj + e] = sc[4 * jj + 2 + e] = -INFINITY;
        }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * hh], sc[4 * jj + 2 * hh + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_used[hh], mx * P.scale_log2);
      const float m_safe = m_new == -INFINITY ? 0.f : m_new;  // a row with no valid key so far: all its p are 0
      const float alpha = exp2f(m_used[hh] - m_safe);
      m_used[hh] = m_new;
      lsum[hh] *= alpha;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        o[4 * jj + 2 * hh] *= alpha;
        o[4 * jj + 2 * hh + 1] *= alpha;
        const float p0 = exp2f(sc[4 * jj + 2 * hh] * P.scale_log2 - m_safe);
        const float p1 = exp2f(sc[4 * jj + 2 * hh + 1] * P.scale_log2 - m_safe);
        sc[4 * jj + 2 * hh] = p0;
        sc[4 * jj + 2 * hh + 1] = p1;
        lsum[hh] += p0 + p1;
      }
    }
    uint32_t pa[32];
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) pa[4 * c + e] = pack_bf16(sc[8 * c + 2 * e], sc[8 * c + 2 * e + 1]);
    reg_fence(o, 64);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < 8; ++c) wgmma_rs_n128<1>(o, pa + 4 * c, sdesc_sw128(sV(s) + c * 2048, ATOM_BYTES, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o, 64);
    named_bar(1, 256);  // both warpgroups are done with stage s
    if (threadIdx.x == 0 && j + 2 < n_tiles) load_kv(j + 2);
  }
  // ----------------------------------------------------------------- epilogue
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    float ls = lsum[hh];
    ls += __shfl_xor_sync(0xffffffffu, ls, 1);
    ls += __shfl_xor_sync(0xffffffffu, ls, 2);
    const int sq = q0 + cw * 64 + 16 * w + (l >> 2) + 8 * hh;
    if (sq >= P.S) continue;
    const float inv = 1.f / ls;
    bf16* dst = sq < P.split ? P.out0 + ((int64_t)b * P.rows0 + sq) * P.ld0 + h * ATT_D
                             : P.out1 + ((int64_t)b * P.rows1 + (sq - P.split)) * P.ld1 + h * ATT_D;
    if (P.lse && (l & 3) == 0) P.lse[(int64_t)bh * P.S + sq] = m_used[hh] + log2f(ls);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj + 2 * (l & 3)) = pack_bf16(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
  }
}

int make_qkv_tmap(CUtensorMap* m, const void* base, int BH, int S) {
  uint64_t dims[3] = {128, (uint64_t)S, (uint64_t)BH};
  uint64_t strides[2] = {128 * 2, (uint64_t)S * 128 * 2};
  uint32_t box[3] = {64, 128, 1};
  return make_tmap_bf16(m, base, 3, dims, strides, box);
}

}  // namespace qfx

using namespace qfx;

/* Q,K,V: [B, H, S, 128] bf16 (head-major joint sequence, text tokens first).  Output is written token-major into two
 * row groups (text rows -> out0, image rows -> out1) so the output projections consume it without a split/copy. */
extern "C" int qfx_attn_fwd(const void* Q, const void* K, const void* V, void* out0, int64_t ld0, int rows0, void* out1,
                            int64_t ld1, int rows1, int split, float* lse, const int* kv_len, const int* txt_len, int B, int H,
                            int S, float softmax_scale, void* stream) {
  QFX_CHECK_ARG(B > 0 && H > 0 && S > 0 && out0 && (split >= S || out1), "qfx_attn_fwd: bad arguments");
  QFX_CHECK_ARG(split >= 0 && rows0 >= (split < S ? split : S) && (split >= S || rows1 >= S - split),
                "qfx_attn_fwd: row groups too short (split=%d S=%d rows0=%d rows1=%d)", split, S, rows0, rows1);
  QFX_CHECK_ARG(!txt_len || (split > 0 && split <= S), "qfx_attn_fwd: txt_len needs 0 < split <= S (split=%d S=%d)", split, S);
  // rows are stored as 4-byte pairs and, in padding query tiles, as 16-byte vectors
  QFX_CHECK_ARG(ld0 % 8 == 0 && ld0 >= (int64_t)H * ATT_D && ((uintptr_t)out0 & 15) == 0 &&
                    (split >= S || (ld1 % 8 == 0 && ld1 >= (int64_t)H * ATT_D && ((uintptr_t)out1 & 15) == 0)),
                "qfx_attn_fwd: out0 / out1 must be 16-byte aligned with leading dimensions >= H*128 and multiples of 8 (ld0=%lld ld1=%lld)",
                (long long)ld0, (long long)ld1);
  AttnFwdParams P;
  memset(&P, 0, sizeof(P));
  int rc;
  if ((rc = make_qkv_tmap(&P.tmQ, Q, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&P.tmK, K, B * H, S))) return rc;
  if ((rc = make_qkv_tmap(&P.tmV, V, B * H, S))) return rc;
  P.out0 = (bf16*)out0; P.out1 = (bf16*)out1;
  P.ld0 = ld0; P.ld1 = ld1; P.rows0 = rows0; P.rows1 = rows1; P.split = split;
  P.lse = lse; P.kv_len = kv_len; P.txt_len = txt_len; P.S = S; P.H = H;
  P.scale_log2 = softmax_scale * 1.4426950408889634f;
  static bool attr_done = false;
  if (!attr_done) {
    QFX_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM));
    attr_done = true;
  }
  dim3 grid((S + ATT_BQ - 1) / ATT_BQ, B * H);
  attn_fwd_kernel<<<grid, 256, ATT_SMEM, (cudaStream_t)stream>>>(P);
  QFX_CUDA(cudaGetLastError());
  return 0;
}
