// LoRA weight gradients on wgmma:  G += A^T B  reduced over the token dimension M (split across CTAs).
//   dB[out, r] = dY^T (s X A^T)        dA[r, in] = (s dY B)^T X         (autograd of peft's LoRA Linear,
//   injected at /root/reference/src/qflux/trainer/base_trainer.py:929-941)
// Both operands are row-major [M, cols] activations, i.e. the reduction dimension is the OUTER one — exactly the
// MN-major wgmma operand layout — so TMA tiles of the tensors as they lie in HBM feed the tensor core directly:
//   A tile [64 rows(m) x 128 cols] = 2 swizzle atoms   -> one M = 64 wgmma per consumer warpgroup and atom
//   B tile [64 rows(m) x 64*NG cols] = NG atoms        -> MMA "N" = 64*NG (one 64-wide rank chunk of each group)
// A group's B columns are Rp = 64*RB wide (the LoRA rank padded to 64 or 128).  Rank chunk c (grid z, c < RB) pairs the A tile
// with columns [g*Rp + 64c, g*Rp + 64c + 64) of every group g, so A is read once per chunk and the accumulator stays 64*NG wide.
// mode 0 (dA of a fused q|k|v site, or any single site): every A-column tile pairs with all NG groups of B.
// mode 1 (dB of a fused site): A columns [g*Dg, (g+1)*Dg) pair with B group g only.
// The [128 x 64*NG] fp32 accumulator lives in the registers of two consumer warpgroups; the epilogue adds the first r columns of each group into the flat
// fp32 LoRA-gradient buffer with red.global.add.f32 (a few thousand per CTA).
#include <string.h>

#include "../../include/qfx.h"
#include "host_common.h"
#include "sm90.cuh"

namespace qfx {

constexpr int WG_MAXG = 3;
constexpr int WG_MAXRB = 2;  // rank chunks per group: r <= 128

struct WgradParams {
  CUtensorMap tmA, tmB;
  float* G[WG_MAXG];
  int64_t gs_i, gs_j;
  int M, Na, ng, mode, Dg, r, rows_per_split;
  float* part;  // deterministic variant: split-major partial tiles [splits][Na][NG * r]
};

template <int NG>
__device__ __forceinline__ void wgmma_wgrad(float* d, uint64_t a, uint64_t b, int scale_d) {
  if constexpr (NG == 1) wgmma_ss_n64<1, 1>(d, a, b, scale_d);
  else if constexpr (NG == 2) wgmma_ss_n128<1, 1>(d, a, b, scale_d);
  else wgmma_ss_n192<1, 1>(d, a, b, scale_d);
}

// kPartial: each CTA stores its partial tile with plain stores into P.part (reduced in split order by launch_split_sum)
// RB: 64-wide rank chunks per group (1: r <= 64, 2: r <= 128)
template <int NG, bool kPartial = false, int RB = 1>
__global__ void __launch_bounds__(384, 1) wgrad_kernel(const __grid_constant__ WgradParams P) {
  constexpr int A_BYTES = 2 * 8192, B_BYTES = NG * 8192, STAGE = A_BYTES + B_BYTES, STAGES = 4;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + STAGES * STAGE;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  const int wg = threadIdx.x >> 7;

  const int i0 = blockIdx.x * 128;                       // first A column of this tile
  const int m_begin = blockIdx.y * P.rows_per_split;
  const int m_end = min(P.M, m_begin + P.rows_per_split);
  const int nkb = (m_end - m_begin + 63) / 64;
  const int grp = P.mode == 1 ? i0 / P.Dg : 0;           // mode 1: the single B group this tile pairs with
  const int c0 = RB > 1 ? (int)blockIdx.z * 64 : 0;     // first rank of this CTA's chunk
  const int b_col0 = (P.mode == 1 ? grp * 64 * RB : 0) + c0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 8);  // lane 0 of each consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      tma_prefetch_desc(&P.tmA);
      tma_prefetch_desc(&P.tmB);
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % STAGES;
        if (kb >= STAGES) mbar_wait(empty_bar(s), ((kb / STAGES) - 1) & 1);
        const uint32_t a_dst = smem_base + s * STAGE, b_dst = a_dst + A_BYTES;
        mbar_expect_tx(full_bar(s), STAGE);
        const int m0 = m_begin + kb * 64;
        tma_load_2d(a_dst, &P.tmA, full_bar(s), i0, m0);
        tma_load_2d(a_dst + 8192, &P.tmA, full_bar(s), i0 + 64, m0);
#pragma unroll
        for (int g = 0; g < NG; ++g) tma_load_2d(b_dst + g * 8192, &P.tmB, full_bar(s), b_col0 + g * 64 * RB, m0);
      }
    }
  } else {
    // consumer cw: A columns i0 + 64 cw .. + 63 (one MN-major swizzle atom of the A tile) x all 64*NG B columns
    const int cw = wg - 1;
    const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    float acc[NG * 32];
#pragma unroll
    for (int e = 0; e < NG * 32; ++e) acc[e] = 0.f;
    reg_fence(acc, NG * 32);
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % STAGES;
      mbar_wait(full_bar(s), (kb / STAGES) & 1);
      const uint32_t a_addr = smem_base + s * STAGE + cw * 8192, b_addr = smem_base + s * STAGE + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_wgrad<NG>(acc, sdesc_sw128(a_addr + k * 2048, 8192, 1024), sdesc_sw128(b_addr + k * 2048, 8192, 1024), 1);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc, NG * 32);
      if (l == 0) mbar_arrive(empty_bar(s));
    }
    if (nkb > 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int i = i0 + cw * 64 + 16 * w + (l >> 2) + 8 * h;  // A column == accumulator row
        if (i >= P.Na) continue;
#pragma unroll
        for (int jj = 0; jj < NG * 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * jj + 2 * (l & 3) + e;
            const int g = col >> 6, j = (col & 63) + c0;
            if (kPartial && j < P.r) {
              P.part[((int64_t)blockIdx.y * P.Na + i) * (NG * P.r) + g * P.r + j] = acc[4 * jj + 2 * h + e];
            } else if (j < P.r) {
              const int gg = P.mode == 1 ? grp : g;
              const int64_t ii = P.mode == 1 ? (int64_t)(i - grp * P.Dg) : (int64_t)i;
              atomicAdd(P.G[gg] + ii * P.gs_i + (int64_t)j * P.gs_j, acc[4 * jj + 2 * h + e]);
            }
          }
        }
      }
    }
  }
}

template <int NG, bool kPartial = false, int RB = 1>
static int launch_wgrad(const WgradParams& P, dim3 grid, cudaStream_t st) {
  constexpr int SMEM = 4 * (2 * 8192 + NG * 8192) + 1024 + 256;
  static bool done = false;
  if (!done) {
    QFX_CUDA(cudaFuncSetAttribute(wgrad_kernel<NG, kPartial, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    done = true;
  }
  wgrad_kernel<NG, kPartial, RB><<<grid, 384, SMEM, st>>>(P);
  QFX_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace qfx

using namespace qfx;

/* A [M, Na] (lda), B [M, Rp*G] (ldb), both bf16 row-major, Rp = 64 * ceil(r / 64).  mode 0: for every group g < G and j < r:
 *   Gp[g][i*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*Rp + j]                                  (i < Na)
 * mode 1 (Na = G*Dg): Gp[g][(i - g*Dg)*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*Rp + j]   for g = i / Dg.        */
extern "C" int qfx_lora_wgrad_tc(const void* A, int64_t lda, int Na, const void* B, int64_t ldb, int G, int M, int mode, int Dg,
                                 float* const* Gp, int64_t gs_i, int64_t gs_j, int r, void* stream) {
  QFX_CHECK_ARG(G >= 1 && G <= WG_MAXG && r >= 1 && r <= 64 * WG_MAXRB && M > 0 && Na % 128 == 0, "qfx_lora_wgrad_tc: bad shape");
  QFX_CHECK_ARG(mode == 0 || (mode == 1 && Dg % 128 == 0 && Na == G * Dg), "qfx_lora_wgrad_tc: bad mode/Dg");
  QFX_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "qfx_lora_wgrad_tc: leading dims must be multiples of 8");
  WgradParams P;
  memset(&P, 0, sizeof(P));
  {
    uint64_t dims[2] = {(uint64_t)Na, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lda * 2};
    uint32_t box[2] = {64, 64};
    int rc = make_tmap_bf16(&P.tmA, A, 2, dims, str, box);
    if (rc) return rc;
    uint64_t dimsb[2] = {(uint64_t)(64 * ((r + 63) / 64) * G), (uint64_t)M};
    uint64_t strb[1] = {(uint64_t)ldb * 2};
    rc = make_tmap_bf16(&P.tmB, B, 2, dimsb, strb, box);
    if (rc) return rc;
  }
  for (int g = 0; g < G; ++g) P.G[g] = Gp[g];
  P.gs_i = gs_i; P.gs_j = gs_j; P.M = M; P.Na = Na; P.ng = G; P.mode = mode; P.Dg = Dg; P.r = r;
  const int rb = (r + 63) / 64, tiles = Na / 128;
  int splits = (2 * num_sms() + tiles * rb - 1) / (tiles * rb);
  const int max_splits = (M + 255) / 256;  // at least 4 k-blocks per CTA
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int rows = ((M + splits - 1) / splits + 63) / 64 * 64;
  P.rows_per_split = rows;
  dim3 grid(tiles, (M + rows - 1) / rows, rb);
  const int ng = mode == 1 ? 1 : G;
  cudaStream_t st = (cudaStream_t)stream;
  switch (ng + 3 * (rb - 1)) {
    case 1: return launch_wgrad<1>(P, grid, st);
    case 2: return launch_wgrad<2>(P, grid, st);
    case 3: return launch_wgrad<3>(P, grid, st);
    case 4: return launch_wgrad<1, false, 2>(P, grid, st);
    case 5: return launch_wgrad<2, false, 2>(P, grid, st);
    default: return launch_wgrad<3, false, 2>(P, grid, st);
  }
}

/* Deterministic variant: the same operation and row split, but every CTA stores its [128 x NG*min(r - 64c, 64)] part of the
 * [128 x NG*r] partial of its split into `scratch` and one fixed-order pass adds the partials into Gp.  The split count depends on the shapes only (not on the GPU):
 *   splits = max(1, min(ceil(M / 256), ceil(QFX_DET_WGRAD_CTAS / (Na / 128)))),  rows = ceil(ceil(M / splits) / 64) * 64,
 *   scratch_floats >= ceil(M / rows) * Na * NG * r,  NG = (mode == 1 ? 1 : G). */
extern "C" int qfx_lora_wgrad_tc_det(const void* A, int64_t lda, int Na, const void* B, int64_t ldb, int G, int M, int mode, int Dg,
                                     float* const* Gp, int64_t gs_i, int64_t gs_j, int r, float* scratch, int64_t scratch_floats,
                                     void* stream) {
  QFX_CHECK_ARG(G >= 1 && G <= WG_MAXG && r >= 1 && r <= 64 * WG_MAXRB && M > 0 && Na % 128 == 0 && Na > 0,
                "qfx_lora_wgrad_tc_det: bad shape");
  QFX_CHECK_ARG(mode == 0 || (mode == 1 && Dg % 128 == 0 && Na == G * Dg), "qfx_lora_wgrad_tc_det: bad mode/Dg");
  QFX_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "qfx_lora_wgrad_tc_det: leading dims must be multiples of 8");
  const int tiles = Na / 128, ng = mode == 1 ? 1 : G, rb = (r + 63) / 64;
  int splits = (QFX_DET_WGRAD_CTAS + tiles - 1) / tiles;  // not scaled by rb: one scratch rule for every r
  const int max_splits = (M + 255) / 256;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  const int rows = ((M + splits - 1) / splits + 63) / 64 * 64;
  splits = (M + rows - 1) / rows;
  const int64_t need = (int64_t)splits * Na * ng * r;
  QFX_CHECK_ARG(scratch && scratch_floats >= need, "qfx_lora_wgrad_tc_det: scratch holds %lld floats, needs %lld",
                (long long)scratch_floats, (long long)need);
  WgradParams P;
  memset(&P, 0, sizeof(P));
  {
    uint64_t dims[2] = {(uint64_t)Na, (uint64_t)M};
    uint64_t str[1] = {(uint64_t)lda * 2};
    uint32_t box[2] = {64, 64};
    int rc = make_tmap_bf16(&P.tmA, A, 2, dims, str, box);
    if (rc) return rc;
    uint64_t dimsb[2] = {(uint64_t)(64 * ((r + 63) / 64) * G), (uint64_t)M};
    uint64_t strb[1] = {(uint64_t)ldb * 2};
    rc = make_tmap_bf16(&P.tmB, B, 2, dimsb, strb, box);
    if (rc) return rc;
  }
  for (int g = 0; g < G; ++g) P.G[g] = Gp[g];
  P.part = scratch;
  P.gs_i = gs_i; P.gs_j = gs_j; P.M = M; P.Na = Na; P.ng = G; P.mode = mode; P.Dg = Dg; P.r = r;
  P.rows_per_split = rows;
  const dim3 grid(tiles, splits, rb);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  switch (ng + 3 * (rb - 1)) {
    case 1: rc = launch_wgrad<1, true>(P, grid, st); break;
    case 2: rc = launch_wgrad<2, true>(P, grid, st); break;
    case 3: rc = launch_wgrad<3, true>(P, grid, st); break;
    case 4: rc = launch_wgrad<1, true, 2>(P, grid, st); break;
    case 5: rc = launch_wgrad<2, true, 2>(P, grid, st); break;
    default: rc = launch_wgrad<3, true, 2>(P, grid, st); break;
  }
  if (rc) return rc;
  SplitSum S;
  memset(&S, 0, sizeof(S));
  S.part = scratch; S.split_stride = (int64_t)Na * ng * r; S.splits = splits; S.rows = Na; S.cols = ng * r;
  for (int g = 0; g < G; ++g) S.dst[g] = Gp[g];
  S.rows_per_dst = mode == 1 ? Dg : Na;  // mode 1: A-column group g -> Gp[g];  mode 0: column group g -> Gp[g]
  S.cols_per_dst = r;
  S.ld_row = gs_i; S.ld_col = gs_j; S.accumulate = 1;
  return launch_split_sum(S, st);
}
