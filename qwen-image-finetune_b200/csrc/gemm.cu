// Fused LoRA projection GEMM for sm_90a: persistent, warp-specialised, TMA -> 128B-swizzled smem ring ->
// wgmma (two consumer warpgroups, each M=64 x N=BN x K=16 with fp32 accumulators in registers) -> fused epilogue.
//
// Replaces the reference's `peft` LoRA Linear forward / backward-dgrad on the MMDiT block projections
// (/root/reference/src/qflux/models/transformer_qwenimage.py:286-293,348-352 and FeedForward :408,418; LoRA injected
// at /root/reference/src/qflux/trainer/base_trainer.py:929-941).  The low-rank term is appended to the K loop of the
// same contraction as extra 64-wide k-blocks taken from a second pair of tensor maps, so each projection is ONE
// tensor-core contraction:   acc = X.W^T + (s X A^T).B^T   (forward)   |   acc = dY.W + (s dY B).A   (dgrad).
//
// Roles (384 threads, 1 CTA / SM): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers: rows 64*(wg-1) .. +63
// of the 128-row tile.  The producer runs ahead into the next tile's k-blocks while the consumers run the epilogue.
#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"
#include <stdlib.h>
#include <string.h>

namespace qfx {

constexpr int BM = 128;
constexpr int BK = 64;

struct GemmProb {
  CUtensorMap tmA, tmB, tmA2, tmB2;
  int M, kb2, a2_col0, rows_per_batch;
  const bf16* bias;
  bf16* out;
  bf16* out2;
  const bf16* resid;
  const bf16* gate;
  const bf16* aux;
  const int* row_tiles;  // ragged rows: start row of each computed 256-row band (NULL: dense)
  int64_t ldo, ldo2, ldr, ldg, ldaux;
  int s_offset, pad_;    // ATTN_DO epilogue: joint position of this row group's first token
};

struct GemmParams {  // passed by value as a __grid_constant__ kernel parameter: must stay below the 4 KB parameter space
  GemmProb p[QFX_MAX_PROBLEMS];
  int nprob, N, K, lora_group_n;
  float* delta;          // ATTN_DO epilogue (shared by the row groups): rowsum(dO * O) per (b, h, s), and the [B, H, S, 128] geometry
  int attn_S, attn_H;
  int tiles_m_end[QFX_MAX_PROBLEMS];  // running sum of the problems' m-tile counts (problem i owns m-tiles [end[i-1], end[i]))
  int tiles_m_total, tiles_n, total_tiles;
  float alpha;
  int stream_out;  // epilogue stores bypass L2 residency (st.global.cs): set when the output is larger than L2, so that writing it does not
                   // evict the A operand every wave re-reads (ncu, round 1: 658 MB of DRAM reads for 210 MB of operands on the MLP-up GEMM)
};

static_assert(sizeof(GemmParams) <= 4090, "GemmParams must fit the kernel parameter space");

template <int BN>
struct GemmCfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 256 ? 4 : BN == 192 ? 5 : BN == 128 ? 6 : 8;
  static constexpr int EPI_LD = 33;  // fp32 staging row of one 32-column chunk, padded: row-per-thread reads are conflict-free
  static constexpr int EPI_BYTES = 2 * 64 * EPI_LD * 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");
};

__device__ __forceinline__ void st_out(uint4* p, uint4 v, bool stream) {
  if (stream) __stcs(p, v);
  else *p = v;
}

// Epilogue of one 32-column chunk of one output row: r = the 32 fp32 accumulators of columns [n, n + 32).
// ATTN_DO: the row is token (ab, as) of the joint sequence; dacc carries sum_d dO*O across the four 32-column chunks of a head,
// so a thread must walk the chunks of a head in order.
template <int EPI>
__device__ __forceinline__ void epilogue_chunk(const GemmProb& q, const GemmParams& P, uint32_t* r, int row, bool row_ok, int n,
                                               const bf16* gate_row, int ab, int as, float& dacc) {
  uint32_t o[16];
  uint4 bias4[4];
  if (q.bias != nullptr) {
#pragma unroll
  for (int v = 0; v < 4; ++v) bias4[v] = __ldg(reinterpret_cast<const uint4*>(q.bias + n) + v);
  } else {
#pragma unroll
  for (int v = 0; v < 4; ++v) bias4[v] = make_uint4(0, 0, 0, 0);
  }
  const uint32_t* bw = reinterpret_cast<const uint32_t*>(bias4);
  if (EPI == QFX_EPI_BIAS) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    float v0 = __uint_as_float(r[2 * i]) * P.alpha + bf16_lo(bw[i]);
    float v1 = __uint_as_float(r[2 * i + 1]) * P.alpha + bf16_hi(bw[i]);
    o[i] = pack_bf16(v0, v1);
  }
  } else if (EPI == QFX_EPI_GELU) {
  uint32_t u[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    u[i] = pack_bf16(__uint_as_float(r[2 * i]) + bf16_lo(bw[i]), __uint_as_float(r[2 * i + 1]) + bf16_hi(bw[i]));
    o[i] = pack_bf16(gelu_tanh(bf16_lo(u[i])), gelu_tanh(bf16_hi(u[i])));
  }
  if (row_ok) {
    uint4* dst2 = reinterpret_cast<uint4*>(q.out2 + (int64_t)row * q.ldo2 + n);
#pragma unroll
    for (int v = 0; v < 4; ++v) st_out(dst2 + v, make_uint4(u[4 * v], u[4 * v + 1], u[4 * v + 2], u[4 * v + 3]), P.stream_out);
  }
  } else if (EPI == QFX_EPI_RESID_GATE) {
  if (row_ok) {
    const uint4* rs = reinterpret_cast<const uint4*>(q.resid + (int64_t)row * q.ldr + n);
    const uint4* gs = reinterpret_cast<const uint4*>(gate_row + n);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      uint4 rr = rs[v];
      uint4 gg = __ldg(gs + v);
      const uint32_t* rw = reinterpret_cast<const uint32_t*>(&rr);
      const uint32_t* gw = reinterpret_cast<const uint32_t*>(&gg);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * v + e;
        // eager bf16 rounding points of the reference: y=Linear(x) -> gate*y -> resid + (.)
        float y0 = round_bf16(__uint_as_float(r[2 * i]) + bf16_lo(bw[i]));
        float y1 = round_bf16(__uint_as_float(r[2 * i + 1]) + bf16_hi(bw[i]));
        float z0 = round_bf16(bf16_lo(gw[e]) * y0);
        float z1 = round_bf16(bf16_hi(gw[e]) * y1);
        o[i] = pack_bf16(bf16_lo(rw[e]) + z0, bf16_hi(rw[e]) + z1);
        if (q.out2 != nullptr) r[i] = pack_bf16(y0, y1);  // un-gated branch output (the accumulator registers are dead now)
      }
    }
    if (q.out2 != nullptr) {  // kept when the gate's AdaLN linear carries LoRA: d gate = sum_t dOut * y
      uint4* dst2 = reinterpret_cast<uint4*>(q.out2 + (int64_t)row * q.ldo2 + n);
#pragma unroll
      for (int v = 0; v < 4; ++v) dst2[v] = make_uint4(r[4 * v], r[4 * v + 1], r[4 * v + 2], r[4 * v + 3]);
    }
  }
  } else if (EPI == QFX_EPI_ADD) {
  if (row_ok) {
    const uint4* rs = reinterpret_cast<const uint4*>(q.resid + (int64_t)row * q.ldr + n);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      uint4 rr = rs[v];
      const uint32_t* rw = reinterpret_cast<const uint32_t*>(&rr);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * v + e;
        o[i] = pack_bf16(bf16_lo(rw[e]) + round_bf16(__uint_as_float(r[2 * i]) * P.alpha),
                         bf16_hi(rw[e]) + round_bf16(__uint_as_float(r[2 * i + 1]) * P.alpha));
      }
    }
  }
  } else if (EPI == QFX_EPI_ATTN_DO) {
  if (row_ok) {
    const uint4* os = reinterpret_cast<const uint4*>(q.aux + (int64_t)row * q.ldaux + n);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      uint4 oo = os[v];
      const uint32_t* ow = reinterpret_cast<const uint32_t*>(&oo);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * v + e;
        const float g0 = round_bf16(__uint_as_float(r[2 * i]) * P.alpha), g1 = round_bf16(__uint_as_float(r[2 * i + 1]) * P.alpha);
        o[i] = pack_bf16(g0, g1);
        dacc += g0 * bf16_lo(ow[e]) + g1 * bf16_hi(ow[e]);
      }
    }
    const int h = n >> 7, cc = n & 127;
    const int64_t pos = ((int64_t)ab * P.attn_H + h) * P.attn_S + as;
    uint4* dj = reinterpret_cast<uint4*>(q.out + pos * 128 + cc);
#pragma unroll
    for (int v = 0; v < 4; ++v) dj[v] = make_uint4(o[4 * v], o[4 * v + 1], o[4 * v + 2], o[4 * v + 3]);
    if (cc == 96) {  // last chunk of this head
      P.delta[pos] = dacc;
      dacc = 0.f;
    }
    if (q.out2 != nullptr) {
      uint4* dst2 = reinterpret_cast<uint4*>(q.out2 + (int64_t)row * q.ldo2 + n);
#pragma unroll
      for (int v = 0; v < 4; ++v) dst2[v] = make_uint4(o[4 * v], o[4 * v + 1], o[4 * v + 2], o[4 * v + 3]);
    }
  }
  } else if (EPI == QFX_EPI_DGELU) {
  if (row_ok) {
    const uint4* us = reinterpret_cast<const uint4*>(q.aux + (int64_t)row * q.ldaux + n);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      uint4 uu = us[v];
      const uint32_t* uw = reinterpret_cast<const uint32_t*>(&uu);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * v + e;
        float g0 = round_bf16(__uint_as_float(r[2 * i]) * P.alpha);
        float g1 = round_bf16(__uint_as_float(r[2 * i + 1]) * P.alpha);
        o[i] = pack_bf16(g0 * gelu_tanh_grad(bf16_lo(uw[e])), g1 * gelu_tanh_grad(bf16_hi(uw[e])));
      }
    }
  }
  }
  if (row_ok && EPI != QFX_EPI_ATTN_DO) {
  uint4* dst = reinterpret_cast<uint4*>(q.out + (int64_t)row * q.ldo + n);
#pragma unroll
  for (int v = 0; v < 4; ++v) st_out(dst + v, make_uint4(o[4 * v], o[4 * v + 1], o[4 * v + 2], o[4 * v + 3]), P.stream_out);
  }
}

template <int BN, int TB>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t a, uint64_t b, int scale_d) {
  if constexpr (BN == 64) wgmma_ss_n64<0, TB>(d, a, b, scale_d);
  else if constexpr (BN == 128) wgmma_ss_n128<0, TB>(d, a, b, scale_d);
  else if constexpr (BN == 192) wgmma_ss_n192<0, TB>(d, a, b, scale_d);
  else wgmma_ss_n256<0, TB>(d, a, b, scale_d);
}

template <int BN, bool TRANS_B, int EPI>
__global__ void __launch_bounds__(384, 1) gemm_kernel(const __grid_constant__ GemmParams P) {
  using C = GemmCfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  float* epi_stage = reinterpret_cast<float*>(smem_gen + C::STAGES * C::STAGE_BYTES);
  const uint32_t bar_base = smem_base + C::STAGES * C::STAGE_BYTES + C::EPI_BYTES;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (C::STAGES + s); };

  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // lane 0 of each of the 8 consumer warps
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int nkb = P.K / BK;

  auto decode = [&](int tile, int& prob, int& m0, int& n0) {
    int n_blk = tile / P.tiles_m_total;
    int mm = tile - n_blk * P.tiles_m_total;
    prob = 0;
#pragma unroll
    for (int i = 0; i < QFX_MAX_PROBLEMS - 1; ++i) prob += (i + 1 < P.nprob && mm >= P.tiles_m_end[i]) ? 1 : 0;
    const int local = prob ? mm - P.tiles_m_end[prob - 1] : mm;
    const int* rt = P.p[prob].row_tiles;
    m0 = rt ? __ldg(rt + (local >> 1)) + (local & 1) * BM : local * BM;
    n0 = n_blk * BN;
  };

  if (wg == 0) {
    // =============================================================== TMA producer
    reg_dealloc<40>();  // one thread issues TMA: the consumers take its registers for the BN/2 accumulators + the epilogue
    if (threadIdx.x == 0) {
      for (int i = 0; i < P.nprob; ++i) {
        tma_prefetch_desc(&P.p[i].tmA);
        tma_prefetch_desc(&P.p[i].tmB);
        if (P.p[i].kb2) {
          tma_prefetch_desc(&P.p[i].tmA2);
          tma_prefetch_desc(&P.p[i].tmB2);
        }
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
        int prob, m0, n0;
        decode(tile, prob, m0, n0);
        const GemmProb& q = P.p[prob];
        const int kb_total = nkb + q.kb2;
        const int grp = (!TRANS_B && P.lora_group_n > 0) ? n0 / P.lora_group_n : 0;
        for (int kb = 0; kb < kb_total; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t a_dst = smem_base + stage * C::STAGE_BYTES;
          const uint32_t b_dst = a_dst + C::A_BYTES;
          mbar_expect_tx(full_bar(stage), C::STAGE_BYTES);
          if (kb < nkb) {
            tma_load_2d(a_dst, &q.tmA, full_bar(stage), kb * BK, m0);
            if (!TRANS_B) {
              tma_load_2d(b_dst, &q.tmB, full_bar(stage), kb * BK, n0);
            } else {
#pragma unroll
              for (int a = 0; a < BN / 64; ++a) tma_load_2d(b_dst + a * 8192, &q.tmB, full_bar(stage), n0 + a * 64, kb * BK);
            }
          } else {
            const int j = kb - nkb;
            tma_load_2d(a_dst, &q.tmA2, full_bar(stage), q.a2_col0 + (grp * q.kb2 + j) * 64, m0);
            if (!TRANS_B) {
              tma_load_2d(b_dst, &q.tmB2, full_bar(stage), j * 64, n0);
            } else {
#pragma unroll
              for (int a = 0; a < BN / 64; ++a) tma_load_2d(b_dst + a * 8192, &q.tmB2, full_bar(stage), n0 + a * 64, j * 64);
            }
          }
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // =============================================================== consumers: rows 64 * cw .. + 63 of each tile
    reg_alloc<232>();  // 128 x 40 + 256 x 232 = 64512 <= the 65536 registers of the SM
    const int cw = wg - 1;
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    float* stg = epi_stage + cw * 64 * C::EPI_LD;
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
      int prob, m0, n0;
      decode(tile, prob, m0, n0);
      const GemmProb& q = P.p[prob];
      const int kb_total = nkb + q.kb2;
      int prev = 0;
      reg_fence(acc, BN / 2);
      for (int kb = 0; kb < kb_total; ++kb) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t a_addr = smem_base + stage * C::STAGE_BYTES + cw * 64 * 128;
        const uint32_t b_addr = smem_base + stage * C::STAGE_BYTES + C::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t ad = sdesc_sw128(a_addr + k * 32, 16, 1024);
          const uint64_t bd = TRANS_B ? sdesc_sw128(b_addr + k * 2048, 8192, 1024) : sdesc_sw128(b_addr + k * 32, 16, 1024);
          wgmma_tile<BN, TRANS_B ? 1 : 0>(acc, ad, bd, (kb | k) != 0);
        }
        wgmma_commit();
        if (kb > 0) {  // the k-block before this one has been consumed: its stage goes back to the producer
          wgmma_wait<1>();
          if (l == 0) mbar_arrive(empty_bar(prev));
        }
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence(acc, BN / 2);
      if (l == 0) mbar_arrive(empty_bar(prev));

      // ---- epilogue: 32-column chunks staged through shared memory so that thread t < 64 owns output row t of the warpgroup
      const int row = m0 + cw * 64 + t;
      const bool row_ok = t < 64 && row < q.M;
      const bf16* gate_row = nullptr;
      if (EPI == QFX_EPI_RESID_GATE && row_ok) gate_row = q.gate + (int64_t)(row / q.rows_per_batch) * q.ldg;
      int ab = 0, as = 0;
      float dacc = 0.f;
      if (EPI == QFX_EPI_ATTN_DO) {
        ab = row / q.rows_per_batch;
        as = q.s_offset + row - ab * q.rows_per_batch;
      }
#pragma unroll
      for (int c = 0; c < BN; c += 32) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = c / 8 + jj;
          const int r0 = 16 * w + (l >> 2), cc = jj * 8 + 2 * (l & 3);
          stg[r0 * C::EPI_LD + cc] = acc[4 * j];
          stg[r0 * C::EPI_LD + cc + 1] = acc[4 * j + 1];
          stg[(r0 + 8) * C::EPI_LD + cc] = acc[4 * j + 2];
          stg[(r0 + 8) * C::EPI_LD + cc + 1] = acc[4 * j + 3];
        }
        named_bar(1 + cw, 128);
        if (t < 64) {
          uint32_t r[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) r[i] = __float_as_uint(stg[t * C::EPI_LD + i]);
          epilogue_chunk<EPI>(q, P, r, row, row_ok, n0 + c, gate_row, ab, as, dacc);
        }
        named_bar(1 + cw, 128);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------ host
static int make_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, int64_t ld_elems, uint32_t box_inner,
                   uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {(uint64_t)ld_elems * 2};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_bf16(m, base, 2, dims, strides, box);
}

template <int BN, bool TRANS_B, int EPI>
static int launch(const GemmParams& P, cudaStream_t stream) {
  using C = GemmCfg<BN>;
  auto kern = gemm_kernel<BN, TRANS_B, EPI>;
  static bool attr_done[64] = {};  // function attributes are per device
  int dev = 0;
  QFX_CUDA(cudaGetDevice(&dev));
  if (!attr_done[dev & 63]) {
    QFX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr_done[dev & 63] = true;
  }
  int grid = P.total_tiles < num_sms() ? P.total_tiles : num_sms();
  kern<<<grid, 384, C::SMEM_BYTES, stream>>>(P);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

template <int BN>
static int dispatch(const GemmParams& P, int trans_b, int epi, cudaStream_t s) {
  if (!trans_b) {
    switch (epi) {
      case QFX_EPI_BIAS: return launch<BN, false, QFX_EPI_BIAS>(P, s);
      case QFX_EPI_GELU: return launch<BN, false, QFX_EPI_GELU>(P, s);
      case QFX_EPI_RESID_GATE: return launch<BN, false, QFX_EPI_RESID_GATE>(P, s);
    }
  } else {
    switch (epi) {
      case QFX_EPI_BIAS: return launch<BN, true, QFX_EPI_BIAS>(P, s);
      case QFX_EPI_DGELU: return launch<BN, true, QFX_EPI_DGELU>(P, s);
      case QFX_EPI_ADD: return launch<BN, true, QFX_EPI_ADD>(P, s);
      case QFX_EPI_ATTN_DO:
        if (BN % 128 == 0) return launch<(BN % 128 == 0 ? BN : 128), true, QFX_EPI_ATTN_DO>(P, s);
        break;
    }
  }
  set_error("qfx_gemm_bf16: unsupported (trans_b=%d, epilogue=%d)", trans_b, epi);
  return -1;
}

}  // namespace qfx

using namespace qfx;

extern "C" int qfx_gemm_bf16(const qfx_gemm_problem* probs, int nprob, int N, int K, int trans_b, int epilogue, float alpha,
                             int lora_group_n, int block_n, void* stream) {
  QFX_CHECK_ARG(nprob >= 1 && nprob <= QFX_MAX_PROBLEMS, "qfx_gemm_bf16: nprob=%d", nprob);
  QFX_CHECK_ARG(K > 0 && K % BK == 0, "qfx_gemm_bf16: K=%d must be a positive multiple of 64", K);
  // block_n = 1000 + bn asks for 256-row tiles computed by a CTA pair; the sm_90a library has one kernel with 128-row tiles and
  // runs such a request as block_n = bn (the result is the same).
  if (block_n >= 1000) block_n -= 1000;
  int bn = block_n;
  if (bn == 0 && epilogue == QFX_EPI_ATTN_DO) bn = N % 256 == 0 ? 256 : 128;  // a tile must hold whole heads
  if (bn == 0) bn = N % 256 == 0 ? 256 : N % 192 == 0 ? 192 : N % 128 == 0 ? 128 : 64;
  QFX_CHECK_ARG(epilogue != QFX_EPI_ATTN_DO || (trans_b && N % 128 == 0 && bn % 128 == 0), "qfx_gemm_bf16: ATTN_DO needs trans_b=1, N %% 128 == 0");
  QFX_CHECK_ARG((bn == 64 || bn == 128 || bn == 192 || bn == 256) && N % bn == 0, "qfx_gemm_bf16: N=%d block_n=%d", N, bn);
  QFX_CHECK_ARG(!(trans_b && lora_group_n), "qfx_gemm_bf16: lora_group_n only with trans_b=0");
  QFX_CHECK_ARG(lora_group_n == 0 || lora_group_n % bn == 0, "qfx_gemm_bf16: lora_group_n %% block_n != 0");
  QFX_CHECK_ARG(alpha == 1.f || (epilogue != QFX_EPI_GELU && epilogue != QFX_EPI_RESID_GATE),
                "qfx_gemm_bf16: the GELU and RESID_GATE epilogues take alpha = 1 only (alpha=%g)", alpha);

  // Every problem is validated before any tensor map is encoded: a refusal never depends on the driver.  The epilogue operands are
  // read and written as 16-byte vectors, so their bases and leading dimensions must allow that.
  auto al16 = [](const void* p) { return ((uintptr_t)p & 15) == 0; };
  for (int i = 0; i < nprob; ++i) {
    const qfx_gemm_problem& s = probs[i];
    QFX_CHECK_ARG(s.M > 0 && s.A && s.B && s.out, "qfx_gemm_bf16: problem %d has null/empty operands", i);
    QFX_CHECK_ARG(s.lda % 8 == 0 && s.ldb % 8 == 0 && s.ldo % 8 == 0, "qfx_gemm_bf16: leading dims must be multiples of 8");
    QFX_CHECK_ARG(s.kb2 >= 0 && s.a2_col0 >= 0, "qfx_gemm_bf16: problem %d: kb2=%d a2_col0=%d", i, s.kb2, s.a2_col0);
    if (s.kb2 > 0) QFX_CHECK_ARG(s.A2 && s.B2 && s.lda2 % 8 == 0 && s.ldb2 % 8 == 0, "qfx_gemm_bf16: bad LoRA operands");
    QFX_CHECK_ARG(!s.row_tiles || s.n_row_tiles > 0, "qfx_gemm_bf16: row_tiles without n_row_tiles");
    if (epilogue == QFX_EPI_GELU) QFX_CHECK_ARG(s.out2 && s.ldo2 % 8 == 0, "qfx_gemm_bf16: GELU epilogue needs out2");
    if (epilogue == QFX_EPI_RESID_GATE) QFX_CHECK_ARG(s.resid && s.gate && s.ldr % 8 == 0 && s.ldg % 8 == 0, "qfx_gemm_bf16: RESID_GATE epilogue needs resid+gate");
    if (epilogue == QFX_EPI_ADD) QFX_CHECK_ARG(s.resid && s.ldr % 8 == 0, "qfx_gemm_bf16: ADD epilogue needs resid");
    if (epilogue == QFX_EPI_DGELU) QFX_CHECK_ARG(s.aux && s.ldaux % 8 == 0, "qfx_gemm_bf16: DGELU epilogue needs aux");
    if (epilogue == QFX_EPI_ATTN_DO) {
      QFX_CHECK_ARG(s.aux && s.ldaux % 8 == 0 && s.delta && s.attn_H * 128 == N && s.attn_S > 0 && s.rows_per_batch > 0 && !s.row_tiles,
                    "qfx_gemm_bf16: ATTN_DO epilogue needs aux (O), delta, attn_H*128 == N, attn_S, rows_per_batch (dense rows only)");
      QFX_CHECK_ARG(s.s_offset >= 0 && s.s_offset + s.rows_per_batch <= s.attn_S,
                    "qfx_gemm_bf16: ATTN_DO problem %d: joint positions [%d, %d) outside attn_S=%d", i, s.s_offset,
                    s.s_offset + s.rows_per_batch, s.attn_S);
      QFX_CHECK_ARG(i == 0 || (s.delta == probs[0].delta && s.attn_S == probs[0].attn_S && s.attn_H == probs[0].attn_H),
                    "qfx_gemm_bf16: ATTN_DO row groups must share delta / attn_S / attn_H");
    }
    const bool has_out2 = s.out2 && (epilogue == QFX_EPI_GELU || epilogue == QFX_EPI_RESID_GATE || epilogue == QFX_EPI_ATTN_DO);
    if (has_out2) QFX_CHECK_ARG(s.ldo2 % 8 == 0, "qfx_gemm_bf16: problem %d: ldo2=%lld must be a multiple of 8", i, (long long)s.ldo2);
    QFX_CHECK_ARG(al16(s.out) && al16(s.bias) && (!has_out2 || al16(s.out2)) &&
                      (!(epilogue == QFX_EPI_RESID_GATE || epilogue == QFX_EPI_ADD) || al16(s.resid)) &&
                      (epilogue != QFX_EPI_RESID_GATE || al16(s.gate)) &&
                      (!(epilogue == QFX_EPI_DGELU || epilogue == QFX_EPI_ATTN_DO) || al16(s.aux)),
                  "qfx_gemm_bf16: problem %d: out / out2 / bias / resid / gate / aux must be 16-byte aligned", i);
  }

  GemmParams P;
  memset(&P, 0, sizeof(P));
  P.nprob = nprob;
  P.N = N;
  P.K = K;
  P.lora_group_n = lora_group_n;
  P.alpha = alpha;
  P.tiles_n = N / bn;
  {
    // outputs larger than about the 50 MB L2 are streamed past it so that writing them does not evict the re-read A operand
    static const int force = getenv("QFX_GEMM_STREAM") ? atoi(getenv("QFX_GEMM_STREAM")) : -1;  // A/B switch
    double out_bytes = 0;
    for (int i = 0; i < nprob; ++i) out_bytes += 2.0 * probs[i].M * N * (epilogue == QFX_EPI_GELU ? 2 : 1);
    P.stream_out = force >= 0 ? force : (out_bytes > 48e6);
  }
  int tiles_m_total = 0;
  for (int i = 0; i < nprob; ++i) {
    const qfx_gemm_problem& s = probs[i];
    GemmProb& d = P.p[i];
    int rc = make_2d(&d.tmA, s.A, (uint64_t)K, (uint64_t)s.M, s.lda, BK, BM);
    if (rc) return rc;
    if (!trans_b)
      rc = make_2d(&d.tmB, s.B, (uint64_t)K, (uint64_t)N, s.ldb, BK, (uint32_t)bn);
    else
      rc = make_2d(&d.tmB, s.B, (uint64_t)N, (uint64_t)K, s.ldb, 64, BK);
    if (rc) return rc;
    d.kb2 = s.kb2;
    d.a2_col0 = s.a2_col0;
    if (s.kb2 > 0) {
      const int groups = lora_group_n ? N / lora_group_n : 1;
      rc = make_2d(&d.tmA2, s.A2, (uint64_t)(s.a2_col0 + 64 * s.kb2 * groups), (uint64_t)s.M, s.lda2, BK, BM);
      if (rc) return rc;
      if (!trans_b)
        rc = make_2d(&d.tmB2, s.B2, (uint64_t)(64 * s.kb2), (uint64_t)N, s.ldb2, BK, (uint32_t)bn);
      else
        rc = make_2d(&d.tmB2, s.B2, (uint64_t)N, (uint64_t)(64 * s.kb2), s.ldb2, 64, BK);
      if (rc) return rc;
    }
    d.M = s.M;
    d.rows_per_batch = s.rows_per_batch > 0 ? s.rows_per_batch : s.M;
    d.bias = (const bf16*)s.bias;
    d.out = (bf16*)s.out;
    d.out2 = (bf16*)s.out2;
    d.resid = (const bf16*)s.resid;
    d.gate = (const bf16*)s.gate;
    d.aux = (const bf16*)s.aux;
    d.ldo = s.ldo; d.ldo2 = s.ldo2; d.ldr = s.ldr; d.ldg = s.ldg; d.ldaux = s.ldaux;
    d.row_tiles = s.row_tiles;
    d.s_offset = s.s_offset;
    if (epilogue == QFX_EPI_ATTN_DO) {
      P.delta = s.delta; P.attn_S = s.attn_S; P.attn_H = s.attn_H;
    }
    int tm = (s.M + BM - 1) / BM;
    if (s.row_tiles) tm = 2 * s.n_row_tiles;
    tiles_m_total += tm;
    P.tiles_m_end[i] = tiles_m_total;
  }
  P.tiles_m_total = tiles_m_total;
  P.total_tiles = tiles_m_total * P.tiles_n;
  cudaStream_t st = (cudaStream_t)stream;
  switch (bn) {
    case 64: return dispatch<64>(P, trans_b, epilogue, st);
    case 128: return dispatch<128>(P, trans_b, epilogue, st);
    case 192: return dispatch<192>(P, trans_b, epilogue, st);
    default: return dispatch<256>(P, trans_b, epilogue, st);
  }
}
