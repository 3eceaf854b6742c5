/*
 * liboasr_b200 -- C ABI of the H100 (sm_90a) kernels behind olmoasr_b200.
 *
 * The reference (allenai/OLMoASR) has no FFI layer: its hot path is plain PyTorch library calls
 * made from olmoasr/model.py, olmoasr/inf_model.py and (third-party) whisper/audio.py.  Each entry
 * point below names the reference call it replaces (file:line under /root/reference).  The host side
 * (olmoasr_b200/*.py) binds these with ctypes; INTEGRATION.md shows the binding a reference
 * maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on it;
 *   - no allocation, no synchronisation, no global state besides a cached device-property query;
 *   - return 0 on success, a negative OASR_ERR_* otherwise; oasr_last_error() gives the message;
 *   - bf16 tensors are row-major, 16-byte aligned, row strides multiples of 8 elements unless noted.
 */
#ifndef OASR_B200_H_
#define OASR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define OASR_API __attribute__((visibility("default")))
#else
#define OASR_API
#endif

#define OASR_OK 0
#define OASR_ERR_INVALID (-1) /* bad argument (shape, alignment, enum)      */
#define OASR_ERR_CUDA (-2)    /* a CUDA runtime / driver call failed        */
#define OASR_ERR_UNSUPPORTED (-3)

/* ---- library ------------------------------------------------------------------------------ */
OASR_API const char* oasr_last_error(void); /* thread-local, valid until the next failing call          */
OASR_API int oasr_abi_version(void);
OASR_API int oasr_device_sm_count(void);
/* SMs the persistent GEMM may occupy (0 = all).  A persistent grid that does not fit next to a concurrent kernel
 * (NCCL's all-reduce CTAs under DDP, train_timestamps.py:2330) runs its displaced CTAs as a second wave; leaving
 * those SMs free avoids it.  Process-wide; returns the previous value. */
OASR_API int oasr_gemm_set_sm_budget(int n_sms);

/* ---- dense GEMM on wgmma -------------------------------------------------------------------------
 * Replaces F.linear in Linear.forward (olmoasr/model.py:97-101), its autograd dgrad / wgrad, the tied
 * logits matmul (model.py:768-770) and the two Conv1d calls (model.py:592-593) after im2col.
 *
 *   D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )        bf16 x bf16 -> fp32 accumulate
 *
 * Operand storage (the reduction index is k):
 *   OASR_K_MAJOR  : A stored [M][K] (lda = row stride), B stored [N][K]   -- k contiguous
 *   OASR_MN_MAJOR : A stored [K][M] (lda = row stride), B stored [K][N]   -- m / n contiguous
 * so forward y = x W^T is (K,K); dgrad dx = dy W is (K,MN); wgrad dW = dy^T x is (MN,MN).
 */
#define OASR_K_MAJOR 0
#define OASR_MN_MAJOR 1

#define OASR_EPI_BF16 0          /* C = bf16(acc + bf16(bias))                                  */
#define OASR_EPI_BF16_GELU 1     /* C = bf16(acc + bias) ; C2 = bf16(gelu_erf(C))               */
#define OASR_EPI_BF16_RESIDUAL 2 /* C = bf16(aux + bf16(acc + bias))                            */
#define OASR_EPI_BF16_GELU_BWD 3 /* C = bf16(bf16(acc) * gelu_erf'(aux))   aux = pre-activation  */
#define OASR_EPI_F32 4           /* C(f32) = acc + bias                                         */
#define OASR_EPI_F32_ATOMIC_ADD 5 /* C(f32) += acc   (split_k >= 1, C pre-initialised; one add per element; no bias) */

OASR_API int oasr_gemm_bf16(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb, int b_layout,
                   void* C, int64_t ldc, void* C2, const float* bias, const void* aux, int64_t ldaux,
                   int64_t M, int64_t N, int64_t K, int epilogue, int split_k, int block_n,
                   void* stream);

/* ---- log-mel front end ----------------------------------------------------------------------------
 * Replaces whisper.audio.log_mel_spectrogram as called per sample on CPU DataLoader workers by
 * AudioTextDataset.preprocess_audio (scripts/training/train_timestamps.py:196-214), eval.py:157-162 and
 * olmoasr/transcribe.py:148.  wave: (batch, n_samples) f32 or int16 (int16 is scaled by 1/32768 like
 * train_timestamps.py:196); out: (batch, n_mels, n_samples/160) f32; clip_max: (batch,) f32 scratch.
 * window/cos_tab/sin_tab: 400 f32 each (Hann window, cos/sin(2 pi i/400)); filters: (n_mels, 201) f32 with
 * non-zero column range [klo[m], khi[m]) per band.  The dynamic-range floor is per clip.
 * n_samples is the row length (a multiple of 640); n_valid <= n_samples (0 = n_samples) the true sample count of every
 * clip: the end reflection of torch.stft(center=True) happens at n_valid and frames >= n_valid/160 are padding (-inf
 * before, floor after the final pass), so recordings of any length give upstream's n // 160 frames exactly. */
OASR_API int oasr_logmel(const void* wave, int in_is_int16, const float* window, const float* cos_tab,
                         const float* sin_tab, const float* filters, const int* klo, const int* khi, float* out,
                         float* clip_max, int64_t batch, int64_t n_samples, int64_t n_mels, int64_t n_valid, void* stream);

/* ---- LayerNorm (olmoasr/model.py:25-39: F.layer_norm(x.float()).type(x.dtype)) -------------------
 * x, y, dy, dx, dresidual: (rows, d) bf16; weight/bias/dweight/dbias: (d,) f32; mean/rstd: (rows,) f32
 * (nullable in the forward).  Backward: dx = bf16(dresidual + bf16(dx_ln)) when dresidual != NULL;
 * dweight/dbias are ACCUMULATED (+=) with atomics: zero them first. */
OASR_API int oasr_layernorm_fwd(const void* x, const float* weight, const float* bias, void* y, float* mean,
                                float* rstd, int64_t rows, int64_t d, float eps, void* stream);
OASR_API int oasr_layernorm_bwd(const void* dy, const void* x, const float* weight, const float* mean,
                                const float* rstd, const void* dresidual, void* dx, float* dweight, float* dbias,
                                int64_t rows, int64_t d, void* stream);

/* ---- attention (head_dim 64) ----------------------------------------------------------------------
 * Replaces F.scaled_dot_product_attention in MultiHeadAttention.forward (olmoasr/model.py:331-340) and its
 * autograd.  q: (B*Tq, ldq) bf16 with head h at columns [64h, 64h+64); k, v: (B*Tkv, ld*) likewise; o like q.
 * causal != 0 applies key <= query; kv_len (B,) int32 (nullable) hides keys >= kv_len[b] -- together they are
 * the reference's `padding_mask + causal mask` (model.py:740-743, train_timestamps.py:314-315).  kv_len[b] is clamped
 * to [1, Tkv]: a sample with kv_len[b] <= 0 sees key 0 alone (no softmax row is ever empty), one with kv_len[b] > Tkv
 * sees every key.
 * lse: (B,H,Tq) f32, log2 domain: log2(sum_k 2^(s_k * scale * log2 e)).
 * Backward: delta (B,H,Tq) f32 is scratch. */
OASR_API int oasr_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream);
OASR_API int oasr_attention_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse,
                                float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                int64_t head_dim, int causal, const int32_t* kv_len, float scale, void* stream);

/* ---- token cross-entropy over bf16 logits ---------------------------------------------------------
 * Replaces F.cross_entropy(logits.view(-1,V), y.view(-1), ignore_index) (train_timestamps.py:1444-1448).
 * logits: (rows, ld) bf16, first V columns valid.  Forward writes lse (rows,) f32 (natural log) and ADDS
 * [sum of row losses, number of non-ignored rows, number of targets outside [0, V) that are not ignore_index] into
 * loss_sum_count[0..2] (4 floats, zero them first); ce_finalize writes the mean loss to loss[0].  Backward
 * overwrites logits in place with bf16(grad_out / count * (softmax - onehot)); ignored rows become zero. */
OASR_API int oasr_ce_fwd(const void* logits, const int64_t* targets, float* lse, float* loss_sum_count,
                         int64_t rows, int64_t V, int64_t ld, int64_t ignore_index, void* stream);
OASR_API int oasr_ce_finalize(const float* loss_sum_count, float* loss, void* stream);
OASR_API int oasr_ce_bwd(void* logits, const int64_t* targets, const float* lse, const float* loss_sum_count,
                         const float* grad_out, int64_t rows, int64_t V, int64_t ld, int64_t ignore_index,
                         void* stream);
/* `.float()` of model.py:770 for callers that ask for logits: (rows, ld) bf16 -> (rows, V) f32 */
OASR_API int oasr_logits_to_f32(const void* src, float* dst, int64_t rows, int64_t V, int64_t ld, void* stream);

/* ---- embedding (model.py:728-732) and its autograd (nn.Embedding padding_idx, model.py:665-667) ----
 * out[b,s,:] = bf16(emb[ids[b,s]] + pos[pos_offset + s]);  backward ACCUMULATES into demb / dpos. */
OASR_API int oasr_embed_fwd(const int64_t* ids, const float* emb, const float* pos, void* out, int64_t batch,
                            int64_t S, int64_t d, int64_t pos_offset, int64_t n_rows_emb, void* stream);
OASR_API int oasr_embed_bwd(const int64_t* ids, const void* dx, float* demb, float* dpos, int64_t batch, int64_t S,
                            int64_t d, int64_t padding_idx, int64_t n_rows_emb, void* stream);

/* ---- casts / conv-stem data movement / small reductions --------------------------------------------
 * cast_f32_to_bf16: the per-call `weight.to(x.dtype)` of Linear.forward (model.py:97-101), hoisted.
 * cast_conv_weight: Conv1d weight (C_out, C_in, 3) f32 -> (C_out, 3, C_in) bf16 (model.py:193-195) so that
 *   conv = im2col + GEMM; unpermute_conv_wgrad is the inverse for the fp32 weight gradient.
 * im2col_conv1: mel (B, C, T) f32 -> (B*T, kpad) bf16, A[b,t][k*C+c] = mel[b][c][t+k-1]        (model.py:592)
 * im2col_conv2: h (B, T_in, d) bf16 -> (B*T_out, 3d) bf16, rows 2t-1, 2t, 2t+1 (stride 2, pad 1) (model.py:593)
 * col2im_conv2_gelu_bwd: gradient w.r.t. conv2's input gathered back and multiplied by gelu'(pre1)
 * add_pos: (x + positional_embedding).to(x.dtype)                                              (model.py:602)
 * gelu_bwd: dy * gelu_erf'(pre);  colsum_bf16: db[n] += sum_m dy[m,n] (bias gradients, ACCUMULATES).
 * unpermute_conv_wgrad: accumulate != 0 adds into dst (a gradient-slab view) instead of overwriting it.
 * mask_to_kvlen: the decoder's dense additive padding mask (B, S, S) f32 (train_timestamps.py:314-315, model.py:740-743)
 *   -> kv_len[b] = number of un-masked key columns; err[0] |= 1 when some row is not [0]*len + [-inf]*(S-len). */
OASR_API int oasr_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
OASR_API int oasr_cast_conv_weight(const float* src, void* dst, int64_t c_out, int64_t c_in, void* stream);
OASR_API int oasr_unpermute_conv_wgrad(const float* src, float* dst, int64_t c_out, int64_t c_in, int accumulate,
                                       void* stream);
OASR_API int oasr_im2col_conv1(const float* mel, void* A, int64_t batch, int64_t C, int64_t T, int64_t kpad, void* stream);
OASR_API int oasr_im2col_conv2(const void* h, void* A, int64_t batch, int64_t T_in, int64_t T_out, int64_t d, void* stream);
OASR_API int oasr_col2im_conv2_gelu_bwd(const void* dA, const void* pre1, void* dpre1, int64_t batch, int64_t T_in,
                                        int64_t T_out, int64_t d, void* stream);
OASR_API int oasr_add_pos(const void* x, const float* pos, void* out, int64_t rows, int64_t T, int64_t d, void* stream);
OASR_API int oasr_gelu_bwd(const void* dy, const void* pre, void* out, int64_t n, void* stream);
OASR_API int oasr_colsum_bf16(const void* dy, float* db, int64_t M, int64_t N, int64_t ld, void* stream);
OASR_API int oasr_mask_to_kvlen(const float* mask, int32_t* kv_len, int32_t* err, int64_t batch, int64_t S, void* stream);

/* ---- fused optimizer step ("next" row: scripts/training/train_timestamps.py:1508-1522) -----------------
 * Replaces scaler.unscale_ -> clip_grad_norm_(max_norm) -> scaler.step(AdamW) (:1509-1521; AdamW defaults :2110-2113).
 * Three launches for the whole model: (1) sum of squares of the UNSCALED gradients (inv_scale is applied before
 * squaring) into out[0]; (2) optim_prepare, one thread: state[0] step (advanced only when the norm is finite: skipped
 * steps are not counted, like GradScaler + AdamW), state[1] unscale x clip coefficient, state[2] 1 - beta1^t,
 * state[3] sqrt(1 - beta2^t), state[4] skip flag, state[5] gradient norm; found_inf[0] = 1 on a non-finite norm;
 * (3) the AdamW update, which also refreshes an optional bf16 shadow of every parameter (the per-forward
 * `weight.to(x.dtype)` of model.py:97-101 never runs).  `state` is 8 floats on the device, zero-initialised.
 * Table form: recs = device table of {float* p, const float* g, float* m, float* v, int64 numel, bf16* shadow|NULL}
 * per tensor; chunks = device int2 {tensor index, chunk index}, oasr_optim_chunk_elems() elements per chunk.
 * Flat form: parameters, gradients, moments and shadow each live in ONE contiguous slab (olmoasr_b200/slab.py). */
OASR_API int oasr_optim_chunk_elems(void);
OASR_API int oasr_grad_sqnorm(const void* recs, const void* chunks, int64_t n_chunks, float inv_scale, float* out,
                              void* stream);
OASR_API int oasr_grad_sqnorm_flat(const float* g, int64_t numel, float inv_scale, float* out, void* stream);
OASR_API int oasr_optim_prepare(const float* norm_sq, float* found_inf, float* state, float inv_scale, float max_norm,
                                float beta1, float beta2, void* stream);
OASR_API int oasr_adamw_step(const void* recs, const void* chunks, int64_t n_chunks, const float* state, float lr,
                             float beta1, float beta2, float eps, float weight_decay, void* stream);
OASR_API int oasr_adamw_flat(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t numel,
                             const float* state, float lr, float beta1, float beta2, float eps, float weight_decay,
                             void* stream);

/* ---- greedy kv-cache decode step (BASELINE.json config 5) -------------------------------------------------
 * The per-step kernels behind `model.decode(mel, DecodingOptions(language="en", without_timestamps=True))`
 * (scripts/eval/eval.py:1846-1847 -> third-party whisper.decoding -> olmoasr/inf_model.py:320-362 TextDecoder.forward,
 * :150-196 MultiHeadAttention, :422-453 kv-cache hooks).  Activation dtype T = fp16 (upstream default fp16=True) or
 * bf16; every rounding point of inf_model.py:172-196 is reproduced (see csrc/decode.cu).  All per-step state (position,
 * tokens, finished flags) is in device memory so that one CUDA graph of these launches is replayed for every step.
 * Argument blocks are plain host structs passed by pointer (read during the call only). */
#define OASR_DTYPE_BF16 0
#define OASR_DTYPE_F16 1
#define OASR_DTYPE_F32 2

/* x = T(token_embedding[tokens[n, *pos]] + positional_embedding[*pos])   (inf_model.py:334-338) */
OASR_API int oasr_dec_embed(const int32_t* tokens, int64_t ld_tokens, const int32_t* pos_ptr, const float* emb,
                            const float* pos_emb, void* x, int64_t n_seq, int64_t d, int64_t n_vocab, int dtype,
                            void* stream);

/* Skinny Linear for <= 64 sequences: out = epilogue(prologue(x) W^T + bias), W (N, K) in dtype T streamed once.
 *   x_mode 0: x (M, K) T;  1: LayerNorm(x; gamma, beta, eps) fused (inf_model.py LayerNorm: fp32, one rounding);
 *          2: x = round_T(sum of n_partials fp32 slabs (each partial_stride elements apart))  -- dec_attention's output
 *   epi    0: T(acc + bias_T)   1: T(gelu_erf(T(acc + bias_T)))   2: T(res + T(acc + bias_T))
 *          3: float(T(acc)) into fp32 `out` (tied logits, inf_model.py:357-360)
 *          4: N = 3d fused [q | k | v]: q -> out, k / v -> row *pos of the static caches (n_seq, cache_len, d)
 *             (replaces the torch.cat of the kv-cache hook, inf_model.py:439-445) */
typedef struct oasr_dec_linear_args {
  const void* x; int64_t ldx; int32_t x_mode; int32_t n_partials; int64_t partial_stride;
  const float* ln_gamma; const float* ln_beta; float ln_eps; int32_t epi;
  const void* W; const float* bias;
  void* out; int64_t ldo; const void* res; int64_t ldres;
  void* k_cache; void* v_cache; int64_t cache_len; const int32_t* pos_ptr;
  int32_t M; int32_t N; int32_t K; int32_t dtype;
} oasr_dec_linear_args;
OASR_API int oasr_dec_linear(const oasr_dec_linear_args* args, void* stream);

/* Single-query attention over a static cache (inf_model.py:172-196 with n_ctx == 1): keys [0, *pos] (self) or
 * [0, n_keys) (cross); k / v element (n, j, h*64 + c) at n * kv_seq_stride + j * kv_row_stride + h*64 + c.
 * scores: (n_seq, n_head, scores_ld) f32 scratch; out_partial: (n_splits, n_seq, ld_out) f32, summed and rounded by
 * the consumer (oasr_dec_linear x_mode 2).  Head dim 64. */
typedef struct oasr_dec_attn_args {
  const void* q; int64_t ldq;
  const void* k; const void* v; int64_t kv_seq_stride; int64_t kv_row_stride;
  float* scores; int64_t scores_ld;
  float* out_partial; int64_t ld_out;
  const int32_t* pos_ptr; int32_t n_keys;
  int32_t n_seq; int32_t n_head; int32_t n_splits; float scale; int32_t dtype;
} oasr_dec_attn_args;
OASR_API int oasr_dec_attention(const oasr_dec_attn_args* args, void* stream);
/* Same as oasr_dec_attention, but sequence n reads K / V entry n / kv_group (beams of one clip share its cross K / V).
 * oasr_dec_attention is the kv_group = 1 case: the same launches and the same bits. */
OASR_API int oasr_dec_attention_grouped(const oasr_dec_attn_args* args, int kv_group, void* stream);

/* FP8 decoding (`DecodingOptions(fp8=True)`): the block projection weights and the cross-attention K / V are stored as
 * e4m3 codes Q with fp32 scales s, quantised by oasr_quantize_fp8_rows (s = amax / 448, q = e4m3(x * 448 / amax)).
 * Activations stay in T (fp16 or bf16); every other rounding point is the one stated above.  Sums are fp32.
 *
 * oasr_dec_linear_fp8w: as oasr_dec_linear, with W (N, K) e4m3 codes (one byte each, 16-byte aligned base) and w_scale
 *   (N,) fp32, one scale per output row.  With x~ the staged input (plain, LayerNorm or partial sum, rounded to T):
 *     y[m, n] = epi( round_T( s_n * sum_k x~[m, k] Q[n, k] + round_T(b_n) ) )
 *   and the GELU, residual, QKV-scatter and store epilogues unchanged.
 *
 * oasr_dec_attention_fp8kv: as oasr_dec_attention_grouped, with k / v e4m3 codes (strides in elements = bytes) and one
 *   scale per (key, head): element (n, j, h) of k_scale / v_scale at (n / kv_group) * scale_seq_stride
 *   + j * scale_row_stride + h.  With q~_c = round_T(q_c hd^-1/4):
 *     score_j = round_T( sK_j hd^-1/4 * sum_c q~_c QK_jc ),  p_j = round_T(softmax_j(score)),
 *     partial_c = sum_j (p_j sV_j) QV_jc  (fp32; summed over the splits in order and rounded once by the consumer).
 *   The engine's cross K / V buffer (L, N * 1500, 2d) has scales (L, N * 1500, 2H): one per (key, head, K|V) group of
 *   64 elements, i.e. oasr_quantize_fp8_rows of the projection viewed as rows of 64. */
OASR_API int oasr_dec_linear_fp8w(const oasr_dec_linear_args* args, const float* w_scale, void* stream);
OASR_API int oasr_dec_attention_fp8kv(const oasr_dec_attn_args* args, const float* k_scale, const float* v_scale,
                                      int64_t scale_seq_stride, int64_t scale_row_stride, int kv_group, void* stream);

/* Logit filters + greedy choice + bookkeeping (whisper/decoding.py SuppressBlank, SuppressTokens, GreedyDecoder.update,
 * the no-speech probability and the stop test of DecodingTask._main_loop), then *pos += 1.
 * tokens: (n_seq, ld_tokens) int32, position *pos holds the token just fed; the choice is written to *pos + 1 once
 * *pos >= sample_begin - 1.  done_flag[0] = 1 when every sequence's newest token is eot.
 * Each row is scanned by n_slices blocks (1..64); scratch: (n_seq, n_slices, 8) f32; counters: (n_seq,) int32, zero on
 * entry and left zero (the block that arrives last merges the slices in slice order). */
typedef struct oasr_dec_sample_args {
  const float* logits; int64_t ld_logits; int32_t* tokens; int64_t ld_tokens; int32_t* pos_ptr;
  const uint8_t* suppress; float* sum_logprobs; float* no_speech_prob; int32_t* n_unfinished; int32_t* done_flag;
  float* scratch; int32_t* counters;
  int32_t n_seq; int32_t n_vocab; int32_t sample_begin; int32_t sot_index; int32_t suppress_blank; int32_t blank;
  int32_t eot; int32_t no_speech; int32_t n_slices; int32_t reserved;
} oasr_dec_sample_args;
OASR_API int oasr_dec_sample(const oasr_dec_sample_args* args, void* stream);

/* The same step with ApplyTimestampRules and temperature sampling (whisper/decoding.py GreedyDecoder.update at any
 * temperature with SuppressBlank, SuppressTokens and, when `timestamps`, ApplyTimestampRules; replaces the hook loop's
 * per-row Python rules and `Categorical(logits=logits / temperature).sample()`), then *pos += 1.
 * temperature: NULL for greedy (argmax), else a device scalar; at > 0 the next token is the Gumbel-max draw
 * argmax_v logits_v / T + g_v over the allowed ids, with g_v from Philox4x32-10 keyed on row_keys[n] (device, one
 * uint64 per row) and counted with (v / 4, *pos): a sample of softmax(filtered logits / T) that depends on (row key,
 * position) only.  sum_logprobs collects log_softmax(filtered logits)[next] at temperature 1.  Temperature and keys are
 * read on the device at every launch, so one captured graph serves every temperature and seed.
 * scratch: (n_seq, n_slices, 48) f32; counters as for oasr_dec_sample.  max_initial_timestamp < 0: no initial limit.
 * n_seq <= 64. */
typedef struct oasr_dec_sample_rules_args {
  const float* logits; int64_t ld_logits; int32_t* tokens; int64_t ld_tokens; int32_t* pos_ptr;
  const uint8_t* suppress; float* sum_logprobs; float* no_speech_prob; int32_t* n_unfinished; int32_t* done_flag;
  float* scratch; int32_t* counters; const float* temperature; const uint64_t* row_keys;
  int32_t n_seq; int32_t n_vocab; int32_t sample_begin; int32_t sot_index; int32_t suppress_blank; int32_t blank;
  int32_t eot; int32_t no_speech; int32_t n_slices;
  int32_t timestamps; int32_t timestamp_begin; int32_t no_timestamps; int32_t max_initial_timestamp; int32_t reserved;
} oasr_dec_sample_rules_args;
OASR_API int oasr_dec_sample_rules(const oasr_dec_sample_rules_args* args, void* stream);

/* Beam search step (whisper/decoding.py BeamSearchDecoder.update with SuppressBlank, SuppressTokens and, when
 * `timestamps`, ApplyTimestampRules) over n_clips x beam rows (row = clip * beam + j), after the logits head.
 *   oasr_dec_beam_candidates: per row the top beam + 1 log-probs after every filter -> scratch
 *                              (n_clips * beam, n_slices, 48) f32; also the raw statistics for the no-speech probability.
 *   oasr_dec_beam_select:     one CTA per clip ranks the candidates, rewrites the clip's token rows (source prefix + new
 *                              token at *pos + 1), sum_logprobs and src_rows, appends eot candidates to the finished list
 *                              (fin_tokens (n_clips, max_candidates, ld_fin) int32 of length fin_len, fin_scores,
 *                              fin_count) while it has room, writes seq_len = *pos + 2; then *pos += 1 and
 *                              done_flag = every clip's list is full.  With done_flag already set nothing changes.
 *   oasr_dec_beam_reorder:    self-attention K / V rows [0, *pos) of every layer: row r <- row src_rows[r] (in place;
 *                              rows whose source is themselves are skipped).  Caches (n_layers, rows, cache_len, d).
 * max_initial_timestamp < 0: no initial-timestamp limit.  1 <= beam <= 8, max_candidates <= 32. */
typedef struct oasr_dec_beam_args {
  const float* logits; int64_t ld_logits; int32_t* tokens; int64_t ld_tokens; int32_t* pos_ptr;
  const uint8_t* suppress; float* sum_logprobs; float* no_speech_prob; int32_t* n_unfinished; int32_t* done_flag;
  float* scratch; int32_t* src_rows;
  int32_t* fin_tokens; int64_t ld_fin; float* fin_scores; int32_t* fin_len; int32_t* fin_count; int32_t* seq_len;
  int32_t n_clips; int32_t beam; int32_t max_candidates; int32_t n_vocab; int32_t n_slices; int32_t n_ctx;
  int32_t sample_begin; int32_t sot_index; int32_t suppress_blank; int32_t blank; int32_t eot; int32_t no_speech;
  int32_t timestamps; int32_t timestamp_begin; int32_t no_timestamps; int32_t max_initial_timestamp;
} oasr_dec_beam_args;
OASR_API int oasr_dec_beam_candidates(const oasr_dec_beam_args* args, void* stream);
OASR_API int oasr_dec_beam_select(const oasr_dec_beam_args* args, void* stream);
OASR_API int oasr_dec_beam_reorder(void* k_cache, void* v_cache, int64_t layer_stride, int64_t row_stride, int64_t n_layers,
                                   const int32_t* src_rows, const int32_t* pos_ptr, int32_t n_clips, int32_t beam, int32_t d,
                                   int32_t n_pos_blocks, int dtype, void* stream);

/* ---- word-level timestamps (whisper/timing.py find_alignment + dtw; the reference's transcribe.py:410-485) --------
 * oasr_align_cost: the DTW input of one window from the alignment heads' captured 16-bit query rows and cross keys.
 *   heads: DEVICE table of n_heads entries; q -> element (0, h * 64) of the layer's cross-attention query projection
 *   (n_tok rows, stride ldq), k -> element (0, h * 64) of that layer's cross key (>= n_frames rows, stride ldk), both of
 *   type `dtype` (OASR_DTYPE_BF16 / OASR_DTYPE_F16).  Per head, in fp32:
 *     QK = (q . k) / 8 (= (q hd^-1/4)(k hd^-1/4), qk_scale 1) over frames [0, n_frames);  W = softmax over frames;
 *     W = (W - mean) / std per frame over all n_tok rows (unbiased=False);  median filter of medfilt_width along frames
 *     with reflect padding (none when n_frames <= medfilt_width / 2);
 *   then the mean over heads (added in table order) of rows [1, n_tok - 1) is negated:
 *     cost (n_tok - 2, n_frames) fp32, row stride ld_cost.
 *   row_stats: (n_heads, n_tok, 2) fp32 workspace.  head_dim == 64, 3 <= n_tok <= 448, 1 <= n_frames <= 1500,
 *   medfilt_width odd and <= 7.  Two launches; bit-identical from run to run.
 * oasr_dtw: dynamic time warping of x (rows, cols) fp32 (row stride ldx), whisper's tie order: with
 *   c0 = cost[i-1][j-1], c1 = cost[i-1][j], c2 = cost[i][j-1]: t = 0 if c0 < c1 and c0 < c2, else 1 if c1 < c0 and
 *   c1 < c2, else 2; cost[i][j] = x[i-1][j-1] + c rounded to float32.  trace: (rows + 1) x (cols + 1) byte workspace.
 *   Writes the path (text_idx, time_idx) (int32, room for rows + cols entries) in path order and its length to
 *   *path_len.  One CTA; rows <= 17065.
 * oasr_align_cost_batched / oasr_dtw_batched: the same computations for n_windows windows of any sizes in one call each
 *   (the windows of one transcribe_batch() round).  `windows` is a DEVICE table of one descriptor per window; the kernels
 *   trust its entries, so the caller keeps every n_tok <= max_tok, n_frames <= max_frames and rows <= max_rows (the host
 *   sizes the grid and the shared memory from these maxima).  Each window's arithmetic is exactly that of the
 *   single-window entry point (which is the one-window case of the same kernels): the results are bit-identical.
 *   oasr_align_window: heads -> a device table of n_heads oasr_align_head entries; row_stats -> offset in floats of the
 *   window's (n_heads, n_tok, 2) workspace inside `row_stats`; cost (n_tok - 2, n_frames) with row stride ld_cost.
 *   oasr_dtw_window: x (rows, cols) with row stride ldx, a (rows + 1) x (cols + 1) byte trace, the path slots. */
typedef struct oasr_align_head {
  const void* q; const void* k; int64_t ldq; int64_t ldk;
} oasr_align_head;
typedef struct oasr_align_window {
  const oasr_align_head* heads; float* cost; int64_t ld_cost; int64_t row_stats; int32_t n_tok; int32_t n_frames;
} oasr_align_window;
typedef struct oasr_dtw_window {
  const float* x; int64_t ldx; uint8_t* trace; int32_t* text_idx; int32_t* time_idx; int32_t* path_len;
  int32_t rows; int32_t cols;
} oasr_dtw_window;
OASR_API int oasr_align_cost(const oasr_align_head* heads, int32_t n_heads, int32_t head_dim, int32_t n_tok,
                             int32_t n_frames, int32_t medfilt_width, float* row_stats, float* cost, int64_t ld_cost,
                             int dtype, void* stream);
OASR_API int oasr_dtw(const float* x, int64_t ldx, int32_t rows, int32_t cols, uint8_t* trace, int32_t* text_idx,
                      int32_t* time_idx, int32_t* path_len, void* stream);
OASR_API int oasr_align_cost_batched(const oasr_align_window* windows, int32_t n_windows, int32_t n_heads,
                                     int32_t head_dim, int32_t max_tok, int32_t max_frames, int32_t medfilt_width,
                                     float* row_stats, int dtype, void* stream);
OASR_API int oasr_dtw_batched(const oasr_dtw_window* windows, int32_t n_windows, int32_t max_rows, void* stream);

/* elementwise dtype conversion (weights fp32 -> T once per engine; bf16 encoder output / cross K,V -> fp16) */
OASR_API int oasr_convert(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n, void* stream);

/* ---- training kernels with a selectable 16-bit activation type -------------------------------------------------
 * The same kernels as the bf16 entry points above, for the reference's step under torch.autocast(dtype=float16)
 * (train_timestamps.py:1414, precision="float16" at :2128): `dtype` is OASR_DTYPE_BF16 (then each call is exactly its
 * bf16 twin: oasr_gemm16 = oasr_gemm_bf16, oasr_colsum16 = oasr_colsum_bf16, ...) or OASR_DTYPE_F16, which reads
 * and writes every 16-bit operand, activation and gradient as IEEE fp16 with the bf16 path's rounding points (the
 * wgmma GEMMs and attention MMAs run .f16 with fp32 accumulators; statistics, lse, delta, biases and weight gradients
 * stay fp32).  fp16 results outside +-65504 become +-inf, like torch's fp16 ops, so GradScaler sees an overflow.
 * oasr_im2col_conv2 is a copy and serves both types; the fp32 -> fp16 weight cast is oasr_convert. */
OASR_API int oasr_gemm16(const void* A, int64_t lda, int a_layout, const void* B, int64_t ldb, int b_layout, void* C,
                         int64_t ldc, void* C2, const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N,
                         int64_t K, int epilogue, int split_k, int block_n, int dtype, void* stream);
/* Low-rank adapters (LoRA).  oasr_gemm_lowrank16: oasr_gemm16 with a low-rank tail in the same fp32 accumulator,
 *   D[M,N] = epilogue( sum_k A[m,k] B[n,k] + sum_j A2[m,j] B2[n,j] )
 * A and A2 (M, K2) K-major, B2 stored like B ((N, K2) for b_layout K-major, (K2, N) for MN-major), K2 a multiple of 8
 * up to 192.  Forward (B K-major): OASR_EPI_BF16, _GELU, _RESIDUAL; dgrad (B MN-major): OASR_EPI_BF16, _RESIDUAL,
 * _GELU_BWD; no split-K.  A Linear y = x W^T + b + s (x A^T) B^T runs as A2 = T(s x A^T), B2 = B, and its dgrad
 * dx = dy W + s (dy B) A as A2 = T(s dy B), B2 = A.
 * oasr_cast_scaled16: dst[r * ld_dst + c] = T(scale * src[r * cols + c]) for an fp32 (rows, cols) src.
 * oasr_lora_merge_f32: out = W + scale * B A for fp32 W / out (N, K), B (N, r), A (r, K); out may be W; deterministic. */
OASR_API int oasr_gemm_lowrank16(const void* A, int64_t lda, const void* B, int64_t ldb, int b_layout, const void* A2,
                                 int64_t lda2, const void* B2, int64_t ldb2, void* C, int64_t ldc, void* C2,
                                 const float* bias, const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K,
                                 int64_t K2, int epilogue, int block_n, int dtype, void* stream);
OASR_API int oasr_cast_scaled16(const float* src, int64_t rows, int64_t cols, float scale, void* dst, int64_t ld_dst,
                                int dtype, void* stream);
OASR_API int oasr_lora_merge_f32(const float* W, const float* B, const float* A, float scale, float* out, int64_t N,
                                 int64_t K, int64_t r, void* stream);
/* FP8 training GEMMs (per-row dynamic scaling).  Formats: */
#define OASR_FP8_E4M3 0   /* max 448   */
#define OASR_FP8_E5M2 1   /* max 57344 */
/* oasr_gemm_fp8: D[M,N] = epilogue( (a_scale[m] * b_scale[n]) * sum_k A[m,k] B[n,k] ) with bf16 C / C2 / aux and the
 *   epilogues of oasr_gemm_bf16, the scaling applied to the fp32 accumulator as (acc * a_scale[m]) * b_scale[n] before
 *   the bias.  A (M, K) and B (N, K) are K-major fp8 (one byte per element) with 16-byte aligned bases, lda / ldb and K
 *   multiples of 16; a_scale (M,) and b_scale (N,) fp32.  Format pairs (a_fmt x b_fmt): e4m3 x e4m3 with OASR_EPI_BF16,
 *   _GELU or _RESIDUAL (a Linear's forward, B = W), and e5m2 x e4m3 with OASR_EPI_BF16, _RESIDUAL or _GELU_BWD (its
 *   dgrad, A = dy, B = W^T); anything else is OASR_ERR_INVALID / OASR_ERR_UNSUPPORTED.  The fp8 products of each
 *   128-deep k-block are summed in a separate accumulator and added to the fp32 one with IEEE adds.  block_n: 64, 128,
 *   or 0 (pick).  No split-K.
 * oasr_quantize_fp8_rows: per-row dynamic quantisation of a 16-bit (rows, cols) matrix x (type `dtype`, row stride ldx):
 *   amax = max |x[r, :]|, inv = fmax / amax, q[r, c] = fp8(x[r, c] * inv) (round to nearest even, saturating to
 *   +-fmax), scale[r] = amax / fmax, in fp32 with IEEE division; a zero row gives inv = scale = 1.  With transpose = 1
 *   the rows of x^T are quantised instead: q is (cols, rows) with row stride ldq and scale has cols entries.  cols (rows
 *   for transpose) a multiple of 8, x 16-byte aligned with ldx a multiple of 8, q 8-byte aligned with ldq a multiple
 *   of 8. */
OASR_API int oasr_gemm_fp8(const void* A, int64_t lda, int a_fmt, const float* a_scale, const void* B, int64_t ldb,
                           int b_fmt, const float* b_scale, void* C, int64_t ldc, void* C2, const float* bias,
                           const void* aux, int64_t ldaux, int64_t M, int64_t N, int64_t K, int epilogue, int block_n,
                           void* stream);
OASR_API int oasr_quantize_fp8_rows(const void* x, int64_t ldx, int64_t rows, int64_t cols, int dtype, int fmt,
                                    int transpose, void* q, int64_t ldq, float* scale, void* stream);
OASR_API int oasr_layernorm_fwd16(const void* x, const float* weight, const float* bias, void* y, float* mean,
                                  float* rstd, int64_t rows, int64_t d, float eps, int dtype, void* stream);
OASR_API int oasr_layernorm_bwd16(const void* dy, const void* x, const float* weight, const float* mean,
                                  const float* rstd, const void* dresidual, void* dx, float* dweight, float* dbias,
                                  int64_t rows, int64_t d, int dtype, void* stream);
OASR_API int oasr_attention_fwd16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, int dtype, void* stream);
OASR_API int oasr_attention_bwd16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                  const void* o, int64_t ldo, const void* dout, int64_t lddo, const float* lse,
                                  float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                  void* dv, int64_t lddv, int64_t B, int64_t H, int64_t Tq, int64_t Tkv,
                                  int64_t head_dim, int causal, const int32_t* kv_len, float scale, int dtype, void* stream);
OASR_API int oasr_ce_fwd16(const void* logits, const int64_t* targets, float* lse, float* loss_sum_count,
                           int64_t rows, int64_t V, int64_t ld, int64_t ignore_index, int dtype, void* stream);
OASR_API int oasr_ce_bwd16(void* logits, const int64_t* targets, const float* lse, const float* loss_sum_count,
                           const float* grad_out, int64_t rows, int64_t V, int64_t ld, int64_t ignore_index, int dtype,
                           void* stream);
OASR_API int oasr_logits_to_f32_16(const void* src, float* dst, int64_t rows, int64_t V, int64_t ld, int dtype,
                                   void* stream);
OASR_API int oasr_embed_fwd16(const int64_t* ids, const float* emb, const float* pos, void* out, int64_t batch,
                              int64_t S, int64_t d, int64_t pos_offset, int64_t n_rows_emb, int dtype, void* stream);
OASR_API int oasr_embed_bwd16(const int64_t* ids, const void* dx, float* demb, float* dpos, int64_t batch, int64_t S,
                              int64_t d, int64_t padding_idx, int64_t n_rows_emb, int dtype, void* stream);
OASR_API int oasr_cast_conv_weight16(const float* src, void* dst, int64_t c_out, int64_t c_in, int dtype, void* stream);
OASR_API int oasr_im2col_conv1_16(const float* mel, void* A, int64_t batch, int64_t C, int64_t T, int64_t kpad, int dtype,
                                  void* stream);
OASR_API int oasr_col2im_conv2_gelu_bwd16(const void* dA, const void* pre1, void* dpre1, int64_t batch, int64_t T_in,
                                          int64_t T_out, int64_t d, int dtype, void* stream);
OASR_API int oasr_add_pos16(const void* x, const float* pos, void* out, int64_t rows, int64_t T, int64_t d, int dtype,
                            void* stream);
OASR_API int oasr_gelu_bwd16(const void* dy, const void* pre, void* out, int64_t n, int dtype, void* stream);
OASR_API int oasr_colsum16(const void* dy, float* db, int64_t M, int64_t N, int64_t ld, int dtype, void* stream);
/* ---- packed (variable-length) decoder batches ----------------------------------------------------------------
 * A training batch whose sample b holds its first len_b tokens (the reference loader pads every transcript to n_text_ctx
 * with 51864 and masks the rest, train_timestamps.py:314-329) runs the decoder on its N = sum len_b real rows only:
 * sample b owns packed rows [cu_seqlens[b], cu_seqlens[b+1]) (int32, B+1 entries, cu_seqlens[0] = 0).
 *
 * oasr_attention_*_varlen16: the attention kernels above over packed query rows q / o / dq (N rows; lse and delta are
 * (H, N) f32).  tiles lists n_tiles (b, j) int32 pairs, one per 128-row query tile j of sample b that holds a row: only
 * those tiles are launched.  Two forms:
 *   kv_cu_seqlens == cu_seqlens: causal self-attention; k / v / dk / dv are packed like q and sample b sees its own
 *                                len_b keys (the reference's causal + padding mask); Tkv is ignored.
 *   kv_cu_seqlens == NULL:       cross-attention; k / v / dk / dv are dense (B*Tkv rows, sample b at row b*Tkv).
 * For each sample the results are bit-for-bit those of oasr_attention_fwd16 / _bwd16 on that sample alone (B = 1,
 * Tq = len_b).  No row of another sample is written.
 *
 * oasr_embed_fwd_packed16: out (N, d) = T(emb[ids[src_rows[r]]] + pos[src_rows[r] % S]), src_rows (N,) int32 holding
 * b*S + t of each packed row of ids (B, S).  oasr_embed_bwd_packed16 ACCUMULATES the packed gradient dx (N, d) into
 * demb / dpos with oasr_embed_bwd16's summation order (padded rows, whose gradient is zero, left out). */
OASR_API int oasr_attention_fwd_varlen16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                         int64_t ldv, void* o, int64_t ldo, float* lse, int64_t B, int64_t H, int64_t N,
                                         int64_t Tkv, int64_t head_dim, const int32_t* cu_seqlens,
                                         const int32_t* kv_cu_seqlens, const int32_t* tiles, int64_t n_tiles, float scale,
                                         int dtype, void* stream);
OASR_API int oasr_attention_bwd_varlen16(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                         int64_t ldv, const void* o, int64_t ldo, const void* dout, int64_t lddo,
                                         const float* lse, float* delta, void* dq, int64_t lddq, void* dk, int64_t lddk,
                                         void* dv, int64_t lddv, int64_t B, int64_t H, int64_t N, int64_t Tkv,
                                         int64_t head_dim, const int32_t* cu_seqlens, const int32_t* kv_cu_seqlens,
                                         const int32_t* tiles, int64_t n_tiles, float scale, int dtype, void* stream);
OASR_API int oasr_embed_fwd_packed16(const int64_t* ids, const float* emb, const float* pos, void* out,
                                     const int32_t* src_rows, int64_t N, int64_t S, int64_t d, int64_t n_rows_emb, int dtype,
                                     void* stream);
OASR_API int oasr_embed_bwd_packed16(const int64_t* ids, const void* dx, float* demb, float* dpos, const int32_t* src_rows,
                                     const int32_t* cu_seqlens, int64_t B, int64_t N, int64_t S, int64_t d,
                                     int64_t padding_idx, int64_t n_rows_emb, int dtype, void* stream);
/* The flat AdamW update refreshing a shadow slab of type `dtype` (bf16 or fp16; see oasr_adamw_flat). */
OASR_API int oasr_adamw_flat16(float* p, const float* g, float* m, float* v, void* shadow, int64_t numel,
                               const float* state, float lr, float beta1, float beta2, float eps, float weight_decay,
                               int dtype, void* stream);
/* oasr_optim_prepare for torch.amp.GradScaler (train_timestamps.py:2349, :1509-1521) without a host read: loss_scale
 * (nullable) is GradScaler's scale S on the device and ext_found_inf (nullable) its found-inf flag.  norm_sq is the
 * squared norm of g * inv_scale with the gradients still scaled by S; the step multiplies every gradient by
 * inv_scale / S, clips against sqrt(norm_sq) / S, and is skipped (not counted) when *ext_found_inf != 0 or that norm
 * is not finite. */
OASR_API int oasr_optim_prepare_amp(const float* norm_sq, float* found_inf, float* state, const float* loss_scale,
                                    const float* ext_found_inf, float inv_scale, float max_norm, float beta1, float beta2,
                                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OASR_B200_H_ */
