/* qfx.h — C ABI of libqfx_b200.so: the H100 (sm_90a) replacement for the reference's per-step hot path
 *
 *     noise-predict forward (MMDiT) -> flow-matching MSE -> backward -> LoRA gradients
 *
 * The reference (tsiendragon/qwen-image-finetune, package `qflux`) is pure Python and has NO FFI of its own
 * (SURVEY.md §8b): its plug point is the `trainer.dit` nn.Module called from `BaseTrainer._compute_loss`
 * (/root/reference/src/qflux/trainer/base_trainer.py:473-476, qwen_image_edit_trainer.py:827-836).  Each entry
 * point below therefore cites the reference *Python* call it replaces.  All pointers are raw device pointers
 * (bf16 unless stated), all calls are asynchronous on `stream` (a cudaStream_t passed as void*), nothing here
 * synchronises with the host, nothing falls back to the CPU.  Return value: 0 on success, otherwise a
 * cudaError_t / negative argument-error code; `qfx_last_error()` returns a static message.
 *
 * INTEGRATION.md shows the ctypes binding the reference side would add.
 */
#ifndef QFX_H_
#define QFX_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* qfx_last_error(void);
int qfx_version(void);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused LoRA projection GEMM (wgmma + TMA).  Replaces one `peft.tuners.lora.Linear.forward` call
 * (injected at base_trainer.py:929-941; y = base(x) + lora_B(lora_A(x)) * alpha/r) or its autograd backward, for
 * up to QFX_MAX_PROBLEMS row-groups that share N, K (e.g. the image and text streams of one MMDiT block:
 * transformer_qwenimage.py:286-293; or the three q|k|v slices of both streams of a LoRA backward, six small problems in one launch).
 *
 *   trans_b = 0 :  out[M,N] = epi( alpha * ( A[M,K] . B[N,K]^T  +  A2[M,64*kb2] . B2[N,64*kb2]^T ) + bias )
 *   trans_b = 1 :  out[M,N] = epi( alpha * ( A[M,K] . B[K,N]    +  A2[M,64*kb2] . B2[64*kb2,N]   ) )      (dgrad)
 *
 * The LoRA factor pair (A2,B2) is appended to the K loop of the SAME tensor-core contraction (rank padded to a
 * multiple of 64 with zeros by the caller: kb2 = 1 for r <= 64, 2 for r <= 128, n times that for an n-slot dgrad), so one register
 * accumulator receives base + low-rank update.
 * alpha scales the accumulator for the BIAS, ADD, DGELU and ATTN_DO epilogues only; GELU and RESID_GATE refuse alpha != 1.
 * out, out2, bias, resid, gate and aux are accessed as 16-byte vectors: their bases must be 16-byte aligned and their leading
 * dimensions multiples of 8 elements.
 */
#define QFX_MAX_PROBLEMS 6

enum qfx_epilogue {
  QFX_EPI_BIAS = 0,       /* out = alpha*acc + bias                                                  (nn.Linear)            */
  QFX_EPI_GELU = 1,       /* out2 = u = acc + bias ; out = gelu_tanh(u)        (FeedForward "gelu-approximate" net.0)       */
  QFX_EPI_RESID_GATE = 2, /* out = resid + gate[row / rows_per_batch, :] * (acc + bias)   (transformer_qwenimage.py:473,480);
                             out2 (optional) = acc + bias, the un-gated branch output (needed for d gate)                  */
  QFX_EPI_DGELU = 3,      /* out = acc * gelu_tanh'(aux)                                   (autograd of net.0's GELU)        */
  QFX_EPI_ADD = 4,        /* out = resid + alpha*acc   (trans_b=1: sum of two dgrads, FLUX single block qkv + proj_mlp)      */
  QFX_EPI_ATTN_DO = 5     /* trans_b=1, N = H*128: g = bf16(alpha*acc) is the gradient wrt the attention output of token
                             (b, s) = (row / rows_per_batch, s_offset + row % rows_per_batch).  Written HEAD-major into
                             out = dO_joint [B, H, S, 128] (ldo unused) — the layout qfx_attn_bwd reads — and, if out2 != NULL,
                             token-major to out2; delta[(b*H + h)*S + s] = sum_d g[h*128 + d] * aux[row, h*128 + d] with aux = the
                             attention output O (token-major).  Replaces qfx_attn_delta after the out-projection dgrad
                             (autograd of transformer_qwenimage.py:348-352 feeding SDPA's backward).                            */
};

typedef struct {
  const void* A;   int64_t lda;  /* [M, K] row-major, lda in elements */
  const void* B;   int64_t ldb;  /* trans_b=0: [N, K];  trans_b=1: [K, N] */
  int M;
  const void* A2;  int64_t lda2; /* LoRA left factor  [M, >= a2_col0 + 64*kb2]  (NULL/kb2=0: none) */
  const void* B2;  int64_t ldb2; /* LoRA right factor trans_b=0: [N, 64*kb2];  trans_b=1: [64*kb2, N] */
  int kb2;                       /* number of appended 64-wide k-blocks */
  int a2_col0;                   /* first column of A2 to use */
  const void* bias;              /* [N] or NULL */
  void* out;       int64_t ldo;  /* [M, N] */
  void* out2;      int64_t ldo2; /* QFX_EPI_GELU: pre-activation u;  QFX_EPI_RESID_GATE: optional un-gated branch output */
  const void* resid; int64_t ldr;/* QFX_EPI_RESID_GATE */
  const void* gate;  int64_t ldg; int rows_per_batch;
  const void* aux;   int64_t ldaux; /* QFX_EPI_DGELU: u */
  /* Ragged row groups (pad-to-max multi-resolution batches, transformer_qwen_custom.py:444-553): when row_tiles != NULL only the
   * n_row_tiles 256-row bands starting at rows row_tiles[i] (device int32, disjoint, ascending) are computed; the other rows of
   * `out`/`out2` are NOT written (the caller zero-fills them, qfx_zero_rows).  NULL: all M rows. */
  const int* row_tiles; int n_row_tiles;
  float* delta; int attn_S, attn_H, s_offset; /* QFX_EPI_ATTN_DO */
} qfx_gemm_problem;

/* lora_group_n > 0 (trans_b = 0 only): output columns [g*lora_group_n, (g+1)*lora_group_n) use A2 columns
 * a2_col0 + g*64*kb2 .. (fused q|k|v projection with one LoRA pair per third).  block_n: 0 = auto, else 64/128/192/256
 * (1000 + 128/256, a request for 256-row CTA-pair tiles, runs as 128/256). */
int qfx_gemm_bf16(const qfx_gemm_problem* probs, int nprob, int N, int K, int trans_b, int epilogue, float alpha,
                  int lora_group_n, int block_n, void* stream);
/* out[rows lo..hi) [:, 0:ncols) = 0 for the n_ranges {lo, hi} pairs in `ranges` (device int32): the padding rows a ragged GEMM skips. */
int qfx_zero_rows(void* out, int64_t ld, int ncols, const int* ranges, int n_ranges, void* stream);


/* ------------------------------------------------------------------------------------------------------------------
 * Joint text+image attention (head_dim 128), wgmma.  Q/K/V/dO/dK/dV: [B, H, S, 128] bf16 head-major, text positions
 * first.  Replaces dispatch_attention_fn -> F.scaled_dot_product_attention on the concatenated sequence and its autograd
 * backward (transformer_qwenimage.py:322-345; transformer_flux.py:149-156).  Pad-to-max multi-resolution batches
 * (transformer_qwen_custom.py:444-553, transformer_flux_custom.py:607-616): kv_len (int32 [B], may be NULL) masks keys
 * >= kv_len[b]; txt_len (int32 [B], may be NULL) additionally masks the text padding, keys in [txt_len[b], split).
 * Forward writes O token-major into two row groups: rows with joint position s < split of sample b go to
 * out0[(b*rows0 + s)*ld0 + h*128 ..], the others to out1[(b*rows1 + s - split)*ld1 + h*128 ..]; lse is the log2-domain
 * log-sum-exp [B,H,S].  Backward: dQ_accum is fp32 [B,H,S,128], zeroed by the caller (every key tile adds into it), 16-byte
 * aligned for qfx_attn_bwd (it is reduced into through a tensor map), 8-byte for qfx_attn_bwd_det; delta = rowsum(dO * O) [B,H,S].  txt_len needs 0 < split <= S.  Forward: rows0 >= split, rows1 >= S - split, out0 / out1
 * 16-byte aligned with ld0 / ld1 >= H*128 and multiples of 8.  A query tile of only padding rows (every position >= kv_len[b]
 * and >= split) gets O = 0 and lse = 0. */
int qfx_attn_fwd(const void* Q, const void* K, const void* V, void* out0, int64_t ld0, int rows0, void* out1, int64_t ld1,
                 int rows1, int split, float* lse, const int* kv_len, const int* txt_len, int B, int H, int S,
                 float softmax_scale, void* stream);
int qfx_attn_bwd(const void* Q, const void* K, const void* V, const void* dO, const float* lse, const float* delta,
                 float* dQ_accum, void* dK, void* dV, const int* kv_len, const int* txt_len, int split, int B, int H, int S,
                 float softmax_scale, void* stream);
/* delta[b,h,s] = sum_d O*dO from token-major rows (tokens_per_sample rows per sample at joint offset s_offset);
 * optionally scatters dO into the head-major layout the backward kernel loads with TMA. */
int qfx_attn_delta(const void* O, int64_t ldo, const void* dO, int64_t lddo, float* delta, void* dO_joint, int tokens,
                   int tokens_per_sample, int s_offset, int S, int H, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * HBM-bound glue (one warp per row, 16-byte accesses, fp32 math, bf16 rounding at the reference's eager rounding points).
 * Row -> sample: b = row / rows_per_batch; per-sample vectors (shift/scale/gate) have row stride ldmod / ldg. */
/* y = LN(x; no affine, eps) * (1 + scale[b]) + shift[b]   (transformer_qwenimage.py:420-423,443-448; AdaLayerNormContinuous) */
int qfx_ln_modulate_fwd(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale, int64_t ldmod,
                        int rows_per_batch, float* mean, float* rstd, int M, int D, float eps, void* stream);
/* dx = dres + LN_bwd(dy * (1 + scale[b])) ; optional dx_gated = dx * gate[b] (input of the next dgrad GEMM) */
int qfx_ln_modulate_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean, const float* rstd,
                        const void* scale, int64_t ldmod, int rows_per_batch, const void* dres, int64_t lddres, void* dx,
                        int64_t lddx, const void* gate, int64_t ldgate, void* dx_gated, int64_t lddxg, int M, int D, void* stream);
/* Gradients of the AdaLN modulation vectors (autograd of transformer_qwenimage.py:420-423,443-448,473,480 when the modulation
 * Linear carries LoRA):  per sample b (rows b*rows_per_batch ..) and column d, ACCUMULATED (+=) into fp32 [B, D] buffers:
 *   sum_out[b,d]  += sum_t g[t,d]                       (d shift; NULL to skip)
 *   prod_out[b,d] += sum_t g[t,d] * m[t,d]              (d scale with m = bf16(LN(x)) when mean/rstd are given (m = x),
 *                                                        d gate with m = the un-gated branch output when mean == NULL)
 * Refused before any CUDA call: M <= 0, D <= 0, D, ldg or ldm not a multiple of 8, M not a multiple of rows_per_batch > 0, and g or
 * m not 16-byte aligned (both are read in 16-byte vectors).  qfx_mod_grad_det refuses the same. */
int qfx_mod_grad(const void* g, int64_t ldg, const void* m, int64_t ldm, const float* mean, const float* rstd, int rows_per_batch,
                 float* sum_out, float* prod_out, int64_t ldo, int M, int D, void* stream);
/* out = bf16(a * gate[b]).  a, gate and out are accessed in 16-byte vectors: D, lda, ldg and ldo must be multiples of 8 and the three
 * bases 16-byte aligned, or the call is refused. */
int qfx_gate_mul(const void* a, int64_t lda, const void* gate, int64_t ldg, int rows_per_batch, void* out, int64_t ldo, int M,
                 int D, void* stream);
/* out = bf16(a + b), n elements (sums of the [B, D] conditioning embeddings, transformer_flux.py time_text_embed) */
int qfx_add_bf16(const void* a, const void* b, void* out, int64_t n, void* stream);
/* diffusers RMSNorm over rows (txt_norm, transformer_qwenimage.py:549,625) */
int qfx_rmsnorm_rows(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int M, int D, float eps, void* stream);
/* per-head RMSNorm(q,k) + RoPE + token-major [tok, q|k|v, H, 128] -> head-major Q/K/V[B,H,S,128] at joint position
 * s_offset + tok % tokens_per_sample (transformer_qwenimage.py:296-326).  rope: fp32 (cos,sin) pairs [S,64,2] when
 * rope_bstride = 0, else per sample [B,S,64,2] with rope_bstride = S.  round_mid = 1 reproduces diffusers' RMSNorm
 * (cast before the weight multiply), 0 = torch.nn.RMSNorm (FLUX).  The backward takes dQ as the fp32 accumulator. */
int qfx_qk_norm_rope_fwd(const void* qkv, int64_t ldqkv, const void* wq, const void* wk, const float* rope, int64_t rope_bstride,
                         void* Q, void* K, void* V, int tokens, int tokens_per_sample, int s_offset, int S, int H, float eps,
                         int round_mid, void* stream);
int qfx_qk_norm_rope_bwd(const void* dQ, const void* dK, const void* dV, const void* qkv, int64_t ldqkv, const void* wq,
                         const void* wk, const float* rope, int64_t rope_bstride, void* dqkv, int64_t lddqkv, int tokens,
                         int tokens_per_sample, int s_offset, int S, int H, float eps, int round_mid, void* stream);
/* Stream-pair variants of the glue above: ONE launch over a stream-major activation buffer whose rows [0, split) (text stream) and
 * [split, M) (image stream) carry different per-stream operands — modulation vectors / q-k norm weights / sample length / joint
 * offset — exactly as the reference applies img_mod vs txt_mod, norm_q vs norm_added_q (transformer_qwenimage.py:437-448, 305-312).
 * Arguments without suffix describe the first group, `...1` the second; split >= M degenerates to the single-group call. */
int qfx_ln_modulate_fwd_pair(const void* x, int64_t ldx, void* y, int64_t ldy, const void* shift, const void* scale, int64_t ldmod,
                             int rows_per_batch, float* mean, float* rstd, int M, int D, float eps, int split, const void* shift1,
                             const void* scale1, int rows_per_batch1, void* stream);
int qfx_ln_modulate_bwd_pair(const void* dy, int64_t lddy, const void* x, int64_t ldx, const float* mean, const float* rstd,
                             const void* scale, int64_t ldmod, int rows_per_batch, const void* dres, int64_t lddres, void* dx,
                             int64_t lddx, const void* gate, int64_t ldgate, void* dx_gated, int64_t lddxg, int M, int D, int split,
                             const void* scale1, const void* gate1, int rows_per_batch1, void* stream);
int qfx_qk_norm_rope_fwd_pair(const void* qkv, int64_t ldqkv, const void* wq, const void* wk, const float* rope,
                              int64_t rope_bstride, void* Q, void* K, void* V, int tokens, int tokens_per_sample, int s_offset, int S,
                              int H, float eps, int round_mid, int split, const void* wq1, const void* wk1, int tokens_per_sample1,
                              int s_offset1, void* stream);
/* clear_dq != 0: every dQ element is set to 0 after it has been read, so the fp32 accumulator is ready for the next attention backward
 * without a separate 118 MB fill (the two row groups together must cover all S positions of every sample). */
int qfx_qk_norm_rope_bwd_pair(void* dQ, const void* dK, const void* dV, const void* qkv, int64_t ldqkv, const void* wq,
                              const void* wk, const float* rope, int64_t rope_bstride, void* dqkv, int64_t lddqkv, int tokens,
                              int tokens_per_sample, int s_offset, int S, int H, float eps, int round_mid, int split, const void* wq1,
                              const void* wk1, int tokens_per_sample1, int s_offset1, int clear_dq, void* stream);
int qfx_attn_delta_pair(const void* O, int64_t ldo, const void* dO, int64_t lddo, float* delta, void* dO_joint, int tokens,
                        int tokens_per_sample, int s_offset, int S, int H, int split, int tokens_per_sample1, int s_offset1,
                        void* stream);
/* y[b,:] = act(x[b,:]) . W^T + bias, b < 8; act 0 none / 1 SiLU  (timestep MLP, img_mod/txt_mod, norm_out.linear) */
int qfx_gemv_act(const void* x, int64_t ldx, const void* W, int64_t ldw, const void* bias, void* y, int64_t ldy, int B, int N,
                 int K, int act, void* stream);
/* diffusers Timesteps(dim, flip_sin_to_cos=True, shift 0, scale): out[b] = [cos(scale*t*f) | sin(scale*t*f)] */
int qfx_timestep_sinusoid(const float* t, float scale, void* out, int B, int dim, void* stream);
/* packed[b] = [ (1-sigma_b) x0 + sigma_b noise | control ]   (qwen_image_edit_trainer.py:811-812) */
int qfx_flow_noisy_input(const void* x0, const void* noise, const void* control, const float* sigma, void* packed, int B, int L,
                         int Lc, int C, void* stream);
/* multi-resolution variant: sample b = [ noisy target (Lt[b] tokens) | control (Lc[b] tokens) | zero padding ], Ltot tokens
 * (per-sample concatenation of flux_kontext_trainer.py:660-700 / tools.py:319-396 pad_latents_for_multi_res) */
int qfx_flow_noisy_input_var(const void* x0, const void* noise, const void* control, const float* sigma, const int* Lt,
                             const int* Lc, void* packed, int B, int Ltmax, int Lcmax, int Ltot, int C, void* stream);
/* loss = norm * sum_{b,t<L,c} w[b,t] (pred - (noise - x0))^2 ; dpred = d loss / d pred * grad_scale (zeros for t >= L)
 * — covers MseLoss / MaskEditLoss / AttentionMaskMseLoss (losses/*.py) through (w, norm).  loss is overwritten.  Refused unless
 * loss != NULL, B, L, C > 0 and Ltot >= L (as qfx_flow_loss_det). */
int qfx_flow_loss(const void* pred, const void* x0, const void* noise, const float* w, float norm, float grad_scale, float* loss,
                  void* dpred, int B, int L, int Ltot, int C, void* stream);
/* G[i*gs_i + j*gs_j] += sum_m P[m,i] Q[m,j], j < r  (LoRA dB = dY^T (sXA^T), dA = (s dY B)^T X); fp32 atomics.
 * Refused unless r is 4, 8, 16, 32 or 64, G != NULL, M > 0 and Dp > 0 (as qfx_lora_wgrad_det). */
int qfx_lora_wgrad(const void* P, int64_t ldp, const void* Q, int64_t ldq, float* G, int64_t gs_i, int64_t gs_j, int M, int Dp,
                   int r, void* stream);
/* The same LoRA weight gradients on the tensor cores (wgmma, both operands MN-major straight from HBM, rows split over CTAs,
 * fp32 atomics), 1 <= r <= 128.  A [M, Na] (lda), B [M, Rp*G] (ldb), both bf16 row-major, with Rp = 64 * ceil(r / 64) (64 or 128:
 * each group's columns are the LoRA rank padded to whole 64-wide k-blocks); Gp: G device pointers to fp32 gradients.
 *   mode 0: for every group g < G and j < r:  Gp[g][i*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*Rp + j]            (dA, or 1-group dB)
 *   mode 1 (Na = G*Dg): Gp[g][(i - g*Dg)*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*Rp + j]  for g = i / Dg   (dB of a fused q|k|v site)
 * Na % 128 == 0.  Each 64-wide rank chunk of the groups is its own CTA column (grid z), so A is read once per chunk. */
int qfx_lora_wgrad_tc(const void* A, int64_t lda, int Na, const void* B, int64_t ldb, int G, int M, int mode, int Dg,
                      float* const* Gp, int64_t gs_i, int64_t gs_j, int r, void* stream);
/* out = bf16(g * pre_scale * min(1, max_norm / (||g * pre_scale|| + 1e-6)))  (clip_grad_norm_, base_trainer.py:449-455);
 * sumsq receives ||g*pre_scale||^2.  max_norm <= 0 disables clipping. */
int qfx_grad_finalize(const float* g, int64_t n, float pre_scale, float max_norm, float* sumsq, void* out_bf16, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused clip + AdamW over the flat fp32 LoRA gradient buffer (replaces clip_gradients + optimizer.step(),
 * base_trainer.py:449-455,528-533 with the default torch.optim.AdamW of :884-916).  `tensors` (device) describes every bf16
 * parameter: row-major [numel / cols, cols] with row stride ld elements, its gradient / moments at grad_offset in the flat
 * buffers.  `chunks` (device, int pairs {tensor index, first element}) tiles each tensor in pieces of <= QFX_ADAMW_CHUNK.
 * grad has been summed over ranks; pre_scale = 1/world; max_norm <= 0 disables clipping; sumsq receives ||grad*pre_scale||^2;
 * step >= 1 is the Adam step count (bias correction).  Moments are fp32.  All on `stream`, no host synchronisation. */
#define QFX_ADAMW_CHUNK 4096
typedef struct {
  void* param;
  int64_t grad_offset;
  int numel, cols;
  int64_t ld;
} qfx_adamw_tensor;
int qfx_fused_adamw(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const float* grad, int64_t n_grad,
                    float* exp_avg, float* exp_avg_sq, float* sumsq, float pre_scale, float max_norm, float lr, float beta1,
                    float beta2, float eps, float weight_decay, int step, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Deterministic variants (selected by the host when torch.use_deterministic_algorithms(True) is in effect).  Each computes what
 * the entry point it is named after computes, with the same arguments and accumulate / overwrite contract, but without
 * floating-point atomics: every cross-CTA sum is formed in a fixed order, so two calls on the same inputs give the same bits on
 * the same GPU.  Reductions store per-CTA partials with plain stores into caller-owned fp32 `scratch` (nothing is allocated
 * inside a call) and a second launch adds them up in split order.  Split counts depend on the shapes only, never on the SM count;
 * each function refuses a scratch smaller than its rule below, before any CUDA call.
 *
 * qfx_attn_bwd_det: dQ, dK, dV of qfx_attn_bwd.  dK / dV come from qfx_attn_bwd's key-major kernel without its dQ phase; dQ from a
 *   query-major kernel (one CTA per 128-query tile, looping over the 64-key tiles in ascending order) that adds every element of
 *   dQ_accum once.  Rows >= kv_len[b] of dQ_accum are left untouched.  No scratch. */
int qfx_attn_bwd_det(const void* Q, const void* K, const void* V, const void* dO, const float* lse, const float* delta,
                     float* dQ_accum, void* dK, void* dV, const int* kv_len, const int* txt_len, int split, int B, int H, int S,
                     float softmax_scale, void* stream);
/* qfx_lora_wgrad_tc_det: qfx_lora_wgrad_tc (1 <= r <= 128).  With NG = (mode == 1 ? 1 : G) and tiles = Na / 128:
 *   splits = max(1, min(ceil(M / 256), ceil(QFX_DET_WGRAD_CTAS / tiles))),  rows = 64 * ceil(ceil(M / splits) / 64),
 *   scratch_floats >= ceil(M / rows) * Na * NG * r            (at most ~QFX_DET_WGRAD_CTAS partial tiles of 128 x NG*r).
 * The split count does not depend on r: for r > 64 each split's two rank chunks store disjoint columns of the same partial tile. */
#define QFX_DET_WGRAD_CTAS 264
int qfx_lora_wgrad_tc_det(const void* A, int64_t lda, int Na, const void* B, int64_t ldb, int G, int M, int mode, int Dg,
                          float* const* Gp, int64_t gs_i, int64_t gs_j, int r, float* scratch, int64_t scratch_floats, void* stream);
/* qfx_lora_wgrad_det: qfx_lora_wgrad (r in 4/8/16/32/64).  rows = 64 * ceil(ceil(M / ceil(M / 512)) / 64),
 *   scratch_floats >= ceil(M / rows) * Dp * r. */
int qfx_lora_wgrad_det(const void* P, int64_t ldp, const void* Q, int64_t ldq, float* G, int64_t gs_i, int64_t gs_j, int M, int Dp,
                       int r, float* scratch, int64_t scratch_floats, void* stream);
/* qfx_mod_grad_det: qfx_mod_grad.  With B = M / rows_per_batch and cb = ceil(D / 256):
 *   splits = max(1, min(ceil(rows_per_batch / 32), ceil(QFX_DET_MODGRAD_CTAS / (cb * B)))),  scratch_floats >= splits * 2 * B * D. */
#define QFX_DET_MODGRAD_CTAS 528
int qfx_mod_grad_det(const void* g, int64_t ldg, const void* m, int64_t ldm, const float* mean, const float* rstd, int rows_per_batch,
                     float* sum_out, float* prod_out, int64_t ldo, int M, int D, float* scratch, int64_t scratch_floats, void* stream);
/* qfx_flow_loss_det: qfx_flow_loss (loss is overwritten).  scratch_floats >= QFX_DET_LOSS_PARTIALS. */
#define QFX_DET_LOSS_PARTIALS 296
int qfx_flow_loss_det(const void* pred, const void* x0, const void* noise, const float* w, float norm, float grad_scale, float* loss,
                      void* dpred, int B, int L, int Ltot, int C, float* scratch, int64_t scratch_floats, void* stream);
/* qfx_grad_finalize_det / qfx_fused_adamw_det: the gradient norm behind the clip of qfx_grad_finalize / qfx_fused_adamw.
 *   scratch_floats >= QFX_DET_NORM_PARTIALS. */
#define QFX_DET_NORM_PARTIALS 592
int qfx_grad_finalize_det(const float* g, int64_t n, float pre_scale, float max_norm, float* sumsq, void* out_bf16, float* scratch,
                          int64_t scratch_floats, void* stream);
int qfx_fused_adamw_det(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const float* grad, int64_t n_grad,
                        float* exp_avg, float* exp_avg_sq, float* sumsq, float pre_scale, float max_norm, float lr, float beta1,
                        float beta2, float eps, float weight_decay, int step, float* scratch, int64_t scratch_floats, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused clip + Prodigy over the flat fp32 LoRA gradient buffer: prodigyopt's Prodigy.step (slice_p = 1, no FSDP) after the clip of
 * qfx_fused_adamw, on the same `tensors` / `chunks` tables.  With g = grad * pre_scale * min(1, max_norm / (||grad*pre_scale|| + 1e-6))
 * (max_norm <= 0: no clip), plus weight_decay * p when decouple == 0, and with the OLD d and dlr = d * lr * bc(k),
 * bc(k) = use_bias_correction ? sqrt(1 - beta2^(k+1)) / (1 - beta1^(k+1)) : 1:
 *   pass A   m = beta1 m + d (1 - beta1) g  (beta1 == 0: m = g) ;  v = beta2 v + d^2 (1 - beta2) g^2 ;  s = beta3 s + (d / d0) (safeguard_warmup ? d : dlr) g
 *            dot += g (p0 - p) ;  den += |s|                              (per-CTA partials in scratch, no atomics)
 *   scalar   d_num = beta3 d_num + (d / d0) dlr dot  (fp64, partials added in a fixed order).  den == 0: SKIPPED = 1 and nothing
 *            else changes.  Else d_hat = d_coef d_num / den ; d = max(d, d_hat) if d == d0 ; d_max = max(d_max, d_hat) ;
 *            d = min(d_max, d growth_rate) ; k += 1
 *   pass B   unless skipped:  p = bf16(p - dlr (decouple ? weight_decay p : 0) - dlr m' / (sqrt(v) + d_new eps)),
 *            m' = m, or d_new m when beta1 == 0
 * m, v, s fp32 and p0 bf16 ([n_grad] each, grad's layout); `scalars` holds QFX_PRODIGY_SCALARS doubles indexed below (initially
 * d = d_max = d0, the rest 0) and is read and written on the device only.  sumsq receives ||grad*pre_scale||^2.  lr > 0: a step
 * with lr == 0 changes nothing in prodigyopt, so the caller launches nothing.  Five launches on `stream`, no host
 * synchronisation; the same inputs give the same bits.  scratch: fp32, 8-byte aligned, scratch_floats >= QFX_PRODIGY_SCRATCH(n_chunks). */
#define QFX_PRODIGY_SCALARS 8
#define QFX_PRODIGY_D 0
#define QFX_PRODIGY_D_MAX 1
#define QFX_PRODIGY_D_NUM 2
#define QFX_PRODIGY_K 3
#define QFX_PRODIGY_DLR 4     /* dlr of the last step */
#define QFX_PRODIGY_SKIPPED 5 /* 1 when the last step found den == 0 */
#define QFX_PRODIGY_D_DEN 6
#define QFX_PRODIGY_D_HAT 7
#define QFX_PRODIGY_SCRATCH(n_chunks) (QFX_DET_NORM_PARTIALS + 4 * (int64_t)(n_chunks))
int qfx_fused_prodigy(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const float* grad, int64_t n_grad, float* exp_avg,
                      float* exp_avg_sq, float* s, const void* p0, double* scalars, float* sumsq, float* scratch, int64_t scratch_floats,
                      float pre_scale, float max_norm, double lr, double beta1, double beta2, double beta3, double eps,
                      double weight_decay, int decouple, int use_bias_correction, int safeguard_warmup, double d0, double d_coef,
                      double growth_rate, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fused clip + 8-bit Adam over the flat fp32 LoRA gradient buffer: bitsandbytes' `optim.Adam8bit` (Optimizer2State "adam", block-wise,
 * percentile_clipping 100, no amsgrad; csrc/kernels.cu kOptimizerStatic8bit2StateBlockwise and kOptimizer32bit2State) after the clip of
 * qfx_fused_adamw, on the same `tensors` / `chunks` tables.  With g = grad * pre_scale * min(1, max_norm / (||grad*pre_scale|| + 1e-6))
 * (max_norm <= 0: no clip), per element in the fp32 arithmetic of those kernels, with step t >= 1:
 *   c1 = 1 - beta1^t,  c2 = sqrt(1 - beta2^t),  step_size = -lr c2 / c1                   (host, fp32)
 *   s1 = s1 beta1 + (1 - beta1) g ;  s2 = s2 beta2 + (1 - beta2) g g
 *   p = bf16(p + step_size s1 / (sqrt(s2) + c2 eps)) ;  p = bf16(p (1 - lr weight_decay))    (the second only when weight_decay > 0)
 * A non-finite g leaves its parameter alone and sets both states to 0, as bitsandbytes does.  lr == 0 still updates the states.
 * Tensor i (chunks' first member) keeps its states
 *   - numel < min_8bit_size: fp32 s1 = s1_32[state_offsets[i] + e], s2 = s2_32[...]  (bitsandbytes' 32-bit path);
 *   - otherwise 8-bit, block-wise: uint8 codes state1 / state2 at grad_offset + e (n_grad bytes each, like grad) and one fp32 absmax1 /
 *     absmax2 per QFX_ADAM8BIT_BLOCK elements of the tensor at state_offsets[i] + e / QFX_ADAM8BIT_BLOCK (the last block may be partial).
 *     Per block: the old states are qmap[code] * absmax_old; the new absmax is the block's max |s| over its elements; the parameter
 *     takes the unquantized new states; the new code is the nearest entry of the sorted 256-entry map to s / absmax (a tie takes the
 *     lower code).  state1 then follows bitsandbytes' sign rule: when qmap1[code] and s1 differ in sign bit, the code steps one
 *     toward s1.  A block whose new absmax is 0 stores QFX_ADAM8BIT_CODE1_ZERO / QFX_ADAM8BIT_CODE2_ZERO (the maps' 0 entries).
 *   qmap1 / qmap2: bitsandbytes' create_dynamic_map(signed=True) / (signed=False), 256 sorted fp32 values each (0 at index 127 / 0).
 * Codes of fp32-path tensors are not touched.  sumsq receives ||grad*pre_scale||^2; the norm's QFX_DET_NORM_PARTIALS partials go
 * to fp32 `scratch` (scratch_floats >= QFX_DET_NORM_PARTIALS) and are added in a fixed order.  Three launches on `stream`, no host
 * synchronisation, no floating-point atomics: the same inputs give the same bits.
 * QFX_ADAM8BIT_BLOCK follows bitsandbytes 0.45 and later, whose block-wise 8-bit optimizers use 256 (older releases used 2048);
 * it divides QFX_ADAMW_CHUNK, so no block crosses a chunk. */
#define QFX_ADAM8BIT_BLOCK 256
#define QFX_ADAM8BIT_CODE1_ZERO 127
#define QFX_ADAM8BIT_CODE2_ZERO 0
int qfx_fused_adam8bit(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const int64_t* state_offsets, const float* grad,
                       int64_t n_grad, unsigned char* state1, unsigned char* state2, float* absmax1, float* absmax2, float* s1_32,
                       float* s2_32, const float* qmap1, const float* qmap2, float* sumsq, float* scratch, int64_t scratch_floats,
                       float pre_scale, float max_norm, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                       int min_8bit_size, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Sharded optimizer state (qflux_b200/optim.py shard_state=True; replaces, per data-parallel rank, optimizer.step() of
 * base_trainer.py:528-533).  A rank owns the contiguous range [state_base, state_base + n_state) of the flat gradient: whole chunks of
 * the tables above (`chunks` / n_chunks is the rank's sub-list; n_chunks == 0 launches nothing).  Its state arrays hold that range
 * only, element fi at index fi - state_base; every chunk's gradient range must lie inside it.  `sumsq` is given, not computed: the
 * caller sums ||grad * pre_scale||^2 over the ranks' slices.  Per element each computes what its replicated form computes with that
 * sumsq; the replicated kernels run unchanged.  No host synchronisation; the same inputs give the same bits.
 *
 * qfx_sumsq_det: out[0] = ||x * pre_scale||^2 over n >= 0 floats, QFX_DET_NORM_PARTIALS grid-stride partials in scratch
 *   (scratch_floats >= QFX_DET_NORM_PARTIALS) added in a fixed order.  Two launches.
 * qfx_fused_adamw_slice: qfx_fused_adamw / _det on the slice.  One launch.
 * qfx_fused_adam8bit_slice: qfx_fused_adam8bit on the slice.  state1 / state2 are n_state bytes; state_offsets is the slice's own
 *   table (tensor i's absmax / fp32 states at state_offsets[i] + e / QFX_ADAM8BIT_BLOCK / + e in the slice's absmax* / s*_32 arrays,
 *   e the element of the tensor; entries may be negative).  One launch.
 * qfx_prodigy_slice_partials: pass A of qfx_fused_prodigy on the slice.  The chunks are entries [chunk0, chunk0 + n_chunks) of the
 *   full table of n_parts chunks; their (sum g (p0 - p), sum |s|) go to part[2 (chunk0 + i)], part[2 (chunk0 + i) + 1] (fp64).
 *   One launch.
 * qfx_prodigy_slice_update: once `part` holds all n_parts chunks' partials (the ranks' slices gathered), the scalar update of
 *   qfx_fused_prodigy over them in chunk order (the same bits as the replicated optimizer from the same partials), then pass B on
 *   the slice.  Two launches (one when n_chunks == 0). */
int qfx_sumsq_det(const float* x, int64_t n, float pre_scale, float* out, float* scratch, int64_t scratch_floats, void* stream);
int qfx_fused_adamw_slice(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const float* grad, int64_t n_grad,
                          int64_t state_base, int64_t n_state, float* exp_avg, float* exp_avg_sq, const float* sumsq, float pre_scale,
                          float max_norm, float lr, float beta1, float beta2, float eps, float weight_decay, int step, void* stream);
int qfx_fused_adam8bit_slice(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, const int64_t* state_offsets,
                             const float* grad, int64_t n_grad, int64_t state_base, int64_t n_state, unsigned char* state1,
                             unsigned char* state2, float* absmax1, float* absmax2, float* s1_32, float* s2_32, const float* qmap1,
                             const float* qmap2, const float* sumsq, float pre_scale, float max_norm, float lr, float beta1, float beta2,
                             float eps, float weight_decay, int step, int min_8bit_size, void* stream);
int qfx_prodigy_slice_partials(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, int chunk0, const float* grad,
                               int64_t n_grad, int64_t state_base, int64_t n_state, float* exp_avg, float* exp_avg_sq, float* s,
                               const void* p0, const double* scalars, const float* sumsq, double* part, int n_parts, float pre_scale,
                               float max_norm, double lr, double beta1, double beta2, double beta3, double weight_decay, int decouple,
                               int use_bias_correction, int safeguard_warmup, double d0, void* stream);
int qfx_prodigy_slice_update(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, int64_t n_grad, int64_t state_base,
                             int64_t n_state, const float* exp_avg, const float* exp_avg_sq, double* scalars, const double* part,
                             int n_parts, double lr, double beta1, double beta2, double beta3, double eps, double weight_decay,
                             int decouple, int use_bias_correction, double d0, double d_coef, double growth_rate, void* stream);
/* qfx_lora_pack / qfx_lora_unpack: the weight all-gather's staging.  For every element of the listed chunks whose gradient offset fi
 * lies in [g_lo, g_hi):  flat[fi - g_lo] = param element (pack),  param element = flat[fi - g_lo] (unpack);  flat is bf16, 2-byte
 * aligned; nothing else is read or written.  Runs of 8 elements within one row move as 16-byte vectors where both sides are 16-byte
 * aligned.  No atomics; one launch (none when n_chunks == 0 or g_hi == g_lo). */
int qfx_lora_pack(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, int64_t g_lo, int64_t g_hi, void* flat,
                  void* stream);
int qfx_lora_unpack(const qfx_adamw_tensor* tensors, const int* chunks, int n_chunks, int64_t g_lo, int64_t g_hi, const void* flat,
                    void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * NF4 frozen weights (4-bit base checkpoints: bitsandbytes `Linear4bit`, whose forward dequantizes the weight to bf16 and runs a
 * plain matmul, bitsandbytes/functional.py dequantize_4bit).  One launch dequantizes up to QFX_NF4_MAX_SEGMENTS tensors (the NF4
 * matrices of one block) into bf16:  out[i] = bf16_rn(NF4[nibble_i] * absmax[i / blocksize])  with the product in fp32,
 * element 2k = high nibble of codes[k], NF4 = bitsandbytes' built-in code book.  absmax is fp32, one value per `blocksize` elements
 * (nested absmax is folded by the caller).  n % 32 == 0, blocksize % 32 == 0 and divides n; codes and out 16-byte aligned.
 * The segment table is read on the host and passed by value: no device table, no host synchronisation. */
#define QFX_NF4_MAX_SEGMENTS 8
typedef struct {
  const void* codes;    /* n / 2 bytes */
  const float* absmax;  /* n / blocksize */
  void* out;            /* n bf16 */
  int64_t n;
  int blocksize;
} qfx_nf4_segment;
int qfx_nf4_dequant(const qfx_nf4_segment* segs, int nseg, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * FP8 frozen weights (float8-e4m3fn base checkpoints without scales, e.g. `*_fp8_e4m3fn` diffusers exports).  One launch expands
 * up to QFX_FP8_MAX_SEGMENTS tensors (the FP8 matrices of one block) into bf16:  out[i] = bf16(e4m3fn codes[i]), exact for every
 * finite code (subnormals down to 2^-9 included; -0 gives 0x8000).  n % 16 == 0; codes and out 16-byte aligned.  The segment
 * table is read on the host and passed by value: no device table, no host synchronisation. */
#define QFX_FP8_MAX_SEGMENTS 8
typedef struct {
  const void* codes;  /* n bytes, one e4m3fn code per element */
  void* out;          /* n bf16 */
  int64_t n;
} qfx_fp8_segment;
int qfx_fp8_expand(const qfx_fp8_segment* segs, int nseg, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Peer memory for sharded frozen weights (replaces FSDP's per-module all-gather, base_trainer.py:333-382, for the frozen block
 * weights).  A rank's weight shard lives in an allocation made by qfx_peer_alloc; its 64-byte handle is sent to the other ranks
 * of the node (any host transport), which map it with qfx_peer_open.  qfx_peer_copy_async then pulls bytes from a mapped peer
 * pointer into local memory with the copy engines over NVLink (cudaMemcpyAsync on `stream`, no SM work, no collective). */
#define QFX_PEER_HANDLE_BYTES 64
int qfx_peer_alloc(int64_t bytes, void** ptr, unsigned char* handle /* [QFX_PEER_HANDLE_BYTES] */);
int qfx_peer_free(void* ptr);
int qfx_peer_open(const unsigned char* handle, void** ptr);
int qfx_peer_close(void* ptr);
int qfx_peer_copy_async(void* dst, const void* src, int64_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Fixed-order sum of the ranks' flat fp32 LoRA gradients for bit-reproducible data-parallel steps on one node (replaces the
 * all-reduce(sum) of the gradient under torch.use_deterministic_algorithms(True); qflux_b200/sharding.py GradExchange):
 *   dst[i] = ((((+0) + src[0][i]) + src[1][i]) + ...) + src[nsrc-1][i]
 * in source order, each add an IEEE fp32 round-to-nearest add with denormals kept and no fused multiply-add; the grid never changes
 * the result.  A NaN result is some NaN (its payload is not specified).  `src` is a host array of nsrc <= QFX_MAX_RANKS device
 * pointers: local allocations or peer mappings from qfx_peer_open.  dst may be one of the sources (the same pointer) but may not
 * otherwise overlap one.  Every pointer 4-byte aligned; any n >= 0 (n == 0 launches nothing).  When all pointers share dst's
 * offset modulo 16 bytes the bulk moves in 16-byte vectors.  One launch on `stream`, no host synchronisation. */
#define QFX_MAX_RANKS 8
int qfx_dp_reduce_det(const float* const* src, int nsrc, float* dst, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QFX_H_ */
