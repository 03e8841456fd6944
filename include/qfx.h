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
 * multiple of 64 with zeros by the caller), so one register accumulator receives base + low-rank update.
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
 * log-sum-exp [B,H,S].  Backward: dQ_accum is fp32 [B,H,S,128], zeroed by the caller (every key tile adds into it);
 * delta = rowsum(dO * O) [B,H,S].  txt_len needs 0 < split <= S.  Forward: rows0 >= split, rows1 >= S - split, out0 / out1
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
 *                                                        d gate with m = the un-gated branch output when mean == NULL) */
int qfx_mod_grad(const void* g, int64_t ldg, const void* m, int64_t ldm, const float* mean, const float* rstd, int rows_per_batch,
                 float* sum_out, float* prod_out, int64_t ldo, int M, int D, void* stream);
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
 * — covers MseLoss / MaskEditLoss / AttentionMaskMseLoss (losses/*.py) through (w, norm). */
int qfx_flow_loss(const void* pred, const void* x0, const void* noise, const float* w, float norm, float grad_scale, float* loss,
                  void* dpred, int B, int L, int Ltot, int C, void* stream);
/* G[i*gs_i + j*gs_j] += sum_m P[m,i] Q[m,j], j < r  (LoRA dB = dY^T (sXA^T), dA = (s dY B)^T X); fp32 atomics */
int qfx_lora_wgrad(const void* P, int64_t ldp, const void* Q, int64_t ldq, float* G, int64_t gs_i, int64_t gs_j, int M, int Dp,
                   int r, void* stream);
/* The same LoRA weight gradients on the tensor cores (wgmma, both operands MN-major straight from HBM, rows split over CTAs,
 * fp32 atomics).  A [M, Na] (lda), B [M, 64*G] (ldb), both bf16 row-major; Gp: G device pointers to fp32 gradients.
 *   mode 0: for every group g < G and j < r:  Gp[g][i*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*64 + j]            (dA, or 1-group dB)
 *   mode 1 (Na = G*Dg): Gp[g][(i - g*Dg)*gs_i + j*gs_j] += sum_m A[m,i] * B[m, g*64 + j]  for g = i / Dg   (dB of a fused q|k|v site)
 * Na % 128 == 0. */
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

#ifdef __cplusplus
}
#endif
#endif /* QFX_H_ */
