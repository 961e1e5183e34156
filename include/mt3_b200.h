/*
 * mt3_b200.h -- C ABI of the H100-native MT3 audio -> event-token hot path.
 *
 * The reference (magenta/mt3) is pure Python and has no FFI of its own; the seams
 * this library replaces are Python call signatures (SURVEY.md 8b).  Each entry
 * point names the reference interface it stands in for (file:line under
 * the reference project's mt3/).  INTEGRATION.md shows the ctypes stub a maintainer of
 * the reference would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer marked DEV is device memory
 *     owned by the caller (a torch tensor's data_ptr() is fine), HOST is host
 *     memory.  The library never allocates in the hot path: models and frontends
 *     allocate their tables once at *_create; all per-call scratch comes from the
 *     caller's workspace (mt3_workspace_bytes).
 *   - `stream` is a cudaStream_t passed as void*; all work is stream-ordered.
 *   - every function returns an int status (0 = MT3_OK); mt3_last_error() returns
 *     a thread-local description of the last failure.  These mirror the
 *     reference's fail-fast Python exceptions (rank asserts network.py:53,168,211,
 *     281; cache shape ValueError layers.py:266-270; bad token dtype layers.py:528).
 *   - handles are not thread-safe; one host thread per GPU/process.
 *   - inference only: dropout off.  The one random stream is the sampling picker's (mt3_generate_sampled):
 *     counter-based (Philox4x32-10), so a result depends on the key, the row's stream index and the position only.
 */
#ifndef MT3_B200_H_
#define MT3_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MT3_ABI_VERSION 2

enum {
  MT3_OK = 0,
  MT3_ERR_BAD_ARG = -1,      /* null pointer, non-positive size, bad flag          */
  MT3_ERR_SHAPE = -2,        /* shape the model/frontend was not created for        */
  MT3_ERR_UNSUPPORTED = -3,  /* valid request this build has no kernel for          */
  MT3_ERR_WORKSPACE = -4,    /* workspace too small / misaligned                    */
  MT3_ERR_CUDA = -5,         /* a CUDA runtime call failed (see mt3_last_error)     */
  MT3_ERR_STATE = -6         /* call order violated (e.g. decode before cross_kv)   */
};

int mt3_abi_version(void);
const char* mt3_last_error(void);
/* Number of kernels this library has launched in this process (bench.py's
 * gpu_launches claim is read from here).  Launches replayed through a CUDA graph
 * are counted per replay. */
uint64_t mt3_kernel_launch_count(void);

/* ------------------------------------------------------------------------- */
/* Frontend: spectrograms.compute_spectrogram (spectrograms.py:64-73) ->      */
/* spectral_ops.compute_logmel (spectral_ops.py:76-88) -> compute_mel (:57-73) */
/* -> compute_mag / stft (:35-54) -> safe_log (:29-32).                        */
/* ------------------------------------------------------------------------- */

typedef struct mt3_frontend mt3_frontend;

typedef struct {
  int32_t sample_rate;   /* spectrograms.py:23  (16000)                       */
  int32_t hop_width;     /* spectrograms.py:24  (128)                         */
  int32_t fft_size;      /* spectrograms.py:28  (2048; the only parity point) */
  int32_t num_mel_bins;  /* spectrograms.py:25  (512)                         */
  float log_eps;         /* spectral_ops.py:29  (1e-5, replace-not-add)       */
} mt3_frontend_config;

/* mel_matrix HOST float32 [fft_size/2+1, num_mel_bins] row-major: the matrix the
 * reference obtains from tf.signal.linear_to_mel_weight_matrix at
 * spectral_ops.py:69-70.  It is converted to a banded per-mel-bin form here. */
int mt3_frontend_create(const mt3_frontend_config* cfg, const float* mel_matrix, mt3_frontend** out);
int mt3_frontend_destroy(mt3_frontend* fe);

/* Number of frames for n samples: ceil(n / hop) (tf.signal.frame pad_end=True,
 * spectral_ops.py:47). */
int mt3_frontend_num_frames(const mt3_frontend* fe, int64_t n_samples);

/* audio DEV f32 [S, n_samples] (row stride = audio_stride elements), each row an
 * independent segment (preprocessors.py:613-618 runs per example).
 * n_valid_frames DEV i32 [S] or NULL: rows >= n_valid_frames[s] are written as
 * 0.0 -- the feature converter's padding of a short last segment (models.py:96).
 * out DEV f32 [S, T, num_mel_bins], T = ceil(n_samples / hop). */
int mt3_logmel_f32(const mt3_frontend* fe, const float* audio, int64_t audio_stride, int32_t num_segments,
                   int32_t n_samples, const int32_t* n_valid_frames, float* out, void* stream);

/* ------------------------------------------------------------------------- */
/* Model: network.Transformer (network.py:265-409) with network.T5Config      */
/* (network.py:25-41) as bound in gin/model.gin:47-59.                         */
/* ------------------------------------------------------------------------- */

typedef struct mt3_model mt3_model;

typedef struct {
  int32_t vocab_size;          /* vocabularies.num_embeddings (vocabularies.py:280) */
  int32_t emb_dim;             /* 512  */
  int32_t num_heads;           /* 6    */
  int32_t head_dim;            /* 64   */
  int32_t num_encoder_layers;  /* 8    */
  int32_t num_decoder_layers;  /* 8    */
  int32_t mlp_dim;             /* 1024 */
  int32_t input_depth;         /* spectrograms.input_depth = num_mel_bins (512)     */
  int32_t max_batch;           /* largest B any call will use                        */
  int32_t max_input_length;    /* largest T (256 mt3, 512 ismir2021)                 */
  int32_t max_decode_length;   /* decoder length L (1024)                            */
  int32_t gemm_mode;           /* MT3_GEMM_* below                                   */
  int32_t kv_cache_format;     /* MT3_KV_* below (ABI version 2)                     */
} mt3_model_config;

enum {
  MT3_GEMM_FP32_SIMT = 0,   /* exact fp32 FMA on CUDA cores (debug / parity anchor)  */
  MT3_GEMM_TF32X3 = 1,      /* wgmma tf32, 3-term split, fp32-faithful       */
  MT3_GEMM_TF32 = 2         /* wgmma tf32 single pass (10-bit mantissa)      */
};

/* Storage format of the decoder's K/V rows -- the self-attention cache (layers.py:249-289) and the hoisted
 * cross-attention K/V.  All arithmetic (projections, scores, softmax, P.V) stays float32; only the stored rows are
 * rounded, and the rounding of a stored row is amplified by every later softmax, the more the sharper the attention
 * (DESIGN.md section 4: error against the float64 oracle, diffuse / sharp attention / trained-checkpoint statistics of
 * tests/test_trained_statistics.py, where float32 arithmetic itself is at 9e-5):
 *   F32  the reference's values exactly                                   4e-6 / 2e-6 / 1.7e-4    100 % of the bytes
 *   P24  float32 cut to 16 mantissa bits, a u16 + u8 plane inside a row   5e-6 / 3e-5 / 1.9e-3     75 %   (default of InferenceModel)
 *   F16  IEEE half                                                        1.6e-4 / 1.2e-3 / 0.7    50 %   (bar: 5e-4)
 * At trained-checkpoint statistics only F32 rows stay inside the bar.                                                */
enum {
  MT3_KV_F32 = 0,
  MT3_KV_F16 = 1,
  MT3_KV_P24 = 2
};

/* Number of float32 elements in the flat weight blob and the offset of a named
 * parameter inside it.  The blob is the Flax parameter tree (SURVEY.md A.3) in
 * the order documented in INTEGRATION.md; names are the tree paths, e.g.
 * "encoder/layers_0/attention/query/kernel".  Returns -1 for an unknown name. */
int64_t mt3_model_num_params(const mt3_model_config* cfg);
int64_t mt3_model_param_offset(const mt3_model_config* cfg, const char* name, int64_t* numel);

/* weights DEV f32 [mt3_model_num_params]; copied/re-laid-out into library-owned
 * device memory (fused QKV, folded norm scales, K-major tiles), so the caller's
 * blob may be freed afterwards. */
int mt3_model_create(const mt3_model_config* cfg, const float* weights, mt3_model** out, void* stream);
int mt3_model_destroy(mt3_model* m);

/* Bytes of caller-provided DEV workspace for calls with this (B, T). 256-byte
 * aligned base required. */
int64_t mt3_workspace_bytes(const mt3_model* m, int32_t batch, int32_t input_length);
int mt3_model_set_workspace(mt3_model* m, void* workspace, int64_t bytes, int32_t batch, int32_t input_length);

/* Transformer.encode(encoder_input_tokens, enable_dropout=False) (network.py:275-301).
 * x DEV f32 [B, T, input_depth] -> encoded DEV f32 [B, T, emb_dim]. */
int mt3_encode(mt3_model* m, const float* x, float* encoded, void* stream);

/* Projects `encoded` to the cross-attention K/V of every decoder layer once per
 * batch (the reference re-projects on every step: network.py:129-135 passes no
 * decode flag) and resets the decode state: cache_index = 0,
 * position_embedder_index = 0 (layers.py:255-260, :589-596). */
int mt3_cross_kv(mt3_model* m, const float* encoded, void* stream);

/* One Transformer.decode(decode=True) step (network.py:303-361): embeds tok_in
 * DEV i32 [B] at the current position, appends self-attention K/V to the cache,
 * and writes logits DEV f32 [B, vocab] (may be NULL) and the greedy next token
 * tok_out DEV i32 [B] (may be NULL).  Position advances by one. */
int mt3_decode_step(mt3_model* m, const int32_t* tok_in, float* logits, int32_t* tok_out, void* stream);

enum {
  MT3_GEN_STOP_AT_EOS = 1,   /* end the loop once every sequence emitted EOS (id 1)   */
  MT3_GEN_USE_GRAPH = 2,     /* replay one captured CUDA graph per step                */
  MT3_GEN_BEAM1 = 4,         /* t5x decoding.beam_search bookkeeping at num_decodes = 1 (the reference's decode_fn,
                                models.py:127) instead of greedy-until-EOS: the live prefix continues with the best non-EOS
                                token, "prefix + EOS" hypotheses are ranked by log-prob / ((5 + length) / 6)^0.6, and the best
                                finished hypothesis is returned.  With MT3_GEN_STOP_AT_EOS the loop ends once every sequence's
                                finished score beats what its live prefix can still reach.                                */
  MT3_GEN_SAMPLE = 8         /* t5x decoding.temperature_sample's pick (mt3_generate_sampled only); not with MT3_GEN_BEAM1   */
};

/* predict_batch_with_aux stand-in (models.py:121-138 + t5x decode loop, greedy):
 * encode + cross_kv + up to num_steps greedy steps from BOS=0.  tokens_out DEV i32
 * [B, max_decode_length]: raw model ids, 0 after EOS and beyond num_steps.
 * x DEV f32 [B, T, input_depth].  steps_run HOST (may be NULL) receives the number
 * of steps executed.  Synchronises the stream before returning only when
 * MT3_GEN_STOP_AT_EOS is set (it has to poll the finished flag). */
int mt3_generate(mt3_model* m, const float* x, int32_t num_steps, int32_t flags, int32_t* tokens_out,
                 int32_t* steps_run, void* stream);

/* mt3_generate with the scores of T5X's predict_batch_with_aux: the same tokens, bit for bit, and
 *   token_scores_out DEV f32 [B, max_decode_length] (may be NULL): the log-probability in float32,
 *     logits[next] - logsumexp(logits row), of every emitted token, from the logits row that chose it.
 *     Greedy: every token up to and including the first EOS; 0 for the PAD after it and beyond the steps run.
 *     MT3_GEN_BEAM1: the returned hypothesis's -- its prefix, the EOS at position n - 1, 0 from n on (n = its
 *     length); the live prefix when nothing finished.
 *   scores_out DEV f32 [B] (may be NULL): greedy, the sum of the row's token scores in one fixed order;
 *     MT3_GEN_BEAM1, T5X beam_search's score: log-probability / ((5 + n) / 6)^0.6 of the best finished
 *     hypothesis, or the live log-probability when nothing finished.
 * A logits row with a NaN gives a NaN token score, and the NaN carries into the sequence score.  With both
 * outputs NULL this is mt3_generate; otherwise each step does one more reduction over its logits row (greedy)
 * or a few more stores (beam1), in CUDA graphs of their own. */
int mt3_generate_scored(mt3_model* m, const float* x, int32_t num_steps, int32_t flags, int32_t* tokens_out,
                        float* token_scores_out, float* scores_out, int32_t* steps_run, void* stream);

/* Transformer.decode(decode=False) / Transformer.__call__ (network.py:303-409 with decode=False, :196-262) and the token
 * scores of T5X's EncoderDecoderModel.score_batch (z_loss = 0): the teacher-forced decoder pass over all L positions at
 * once, from the caller's `encoded` DEV f32 [B, T, emb_dim] (the output of mt3_encode).
 *   decoder_input_tokens, decoder_target_tokens DEV i32 [B, L]; loss_weights DEV i32 [B, L] or NULL (= target > 0).
 *   Self-attention mask make_decoder_mask(decoder_target_tokens): query i sees key j iff j <= i and target[j] > 0;
 *   positions are arange(L); cross-attention sees all T encoder positions.
 *   logits DEV f32 [B, L, vocab] (16-byte aligned) or NULL; token_scores DEV f32 [B, L] or NULL:
 *   (logits[b, i, target] - logsumexp(logits[b, i, :])) * weight[b, i].  Not both NULL.
 *   Positions with target == 0 (padding) get the causal, key-masked result -- finite, 0 where no key is visible -- not the
 *   reference's all-masked row (DESIGN.md section 1), and score 0 under the default weights.
 * All K/V of the pass are float32 whatever kv_cache_format is, and live in `workspace` DEV (256-byte aligned,
 * mt3_teacher_forced_workspace_bytes); the decode state (workspace of mt3_model_set_workspace, K/V caches, position,
 * captured graphs) is not touched.  In the wgmma gemm modes the first call builds K-major copies of the decoder weights
 * (TF32X3 ~183 MB, TF32 ~92 MB at the mt3 shapes), owned by the model and freed by mt3_model_destroy.
 * Every argument is checked before any CUDA call: MT3_ERR_BAD_ARG (null handle / input, both outputs NULL),
 * MT3_ERR_SHAPE (batch, input_length or target_length outside (0, the model's limit]), MT3_ERR_WORKSPACE (short or
 * misaligned workspace). */
int64_t mt3_teacher_forced_workspace_bytes(const mt3_model* m, int32_t batch, int32_t input_length, int32_t target_length);
int mt3_decode_teacher_forced(mt3_model* m, const float* encoded, int32_t batch, int32_t input_length,
                              const int32_t* decoder_input_tokens, const int32_t* decoder_target_tokens,
                              const int32_t* loss_weights, int32_t target_length, float* logits, float* token_scores,
                              void* workspace, int64_t workspace_bytes, void* stream);

/* mt3_generate_scored with a forced decoder prefix per sequence: T5X predict_batch_with_aux(prompt_with_targets=True).
 *   prompt DEV i32 [B, prompt_len], 0 <= prompt_len <= num_steps: row b's prompt is its non-zero prefix, of length p_b.
 *   Prompt ids lie in [2, vocab); PAD 0 ends the prompt and every entry after it must be 0; EOS 1 is not allowed.  A
 *   violation returns MT3_ERR_BAD_ARG before any decode step runs (the check costs one kernel and an 8-byte copy back,
 *   and synchronises the stream).
 *   tokens_out[b, j] = prompt[b, j] for j < p_b; from p_b on the loop chooses (greedy, or MT3_GEN_BEAM1), conditioned on
 *   the prefix.  num_steps bounds the whole row, prompt included (T5X's max_decode_len), and *steps_run counts the
 *   prompt's positions too.
 *   Scores follow T5X's convention for forced prompts: forced tokens are not the model's choices.  token_scores_out is 0
 *   at forced positions; greedy's score sums the free positions; MT3_GEN_BEAM1 starts its live log-probability at 0 where
 *   the prompt ends, makes no "prefix + EOS" hypothesis at a forced position and keeps the brevity penalty of the full
 *   length.  A sequence cannot finish inside its prompt.
 *   The prefix all rows share, P = min p_b, is prefilled: one teacher-forced pass (mt3_decode_teacher_forced's kernels)
 *   writes the K/V rows of positions 0 .. P-1 into the decode cache and the loop starts at position P.  Positions from P to
 *   p_b are forced inside the loop.  In the wgmma gemm modes the first prefill builds the pass's decoder weights.
 *   workspace: the teacher-forced workspace, mt3_teacher_forced_workspace_bytes(m, B, T, prompt_len) bytes, 256-byte
 *   aligned (MT3_ERR_WORKSPACE otherwise); it may be NULL only when prompt_len == 0.
 * With prompt_len == 0, or every row empty, this is mt3_generate_scored: the same tokens and scores, bit for bit, no pass. */
int mt3_generate_prompted(mt3_model* m, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt, int32_t prompt_len,
                          int32_t* tokens_out, float* token_scores_out, float* scores_out, int32_t* steps_run, void* workspace,
                          int64_t workspace_bytes, void* stream);

/* Sampling parameters of mt3_generate_sampled.
 *   temperature: z = logits / temperature (float32 division), finite and >= 0.  At or below 1e-4 the greedy loop runs
 *     unchanged (T5X's MIN_TEMPERATURE): the tokens and scores of mt3_generate_prompted, bit for bit.
 *   topk: 0 = off; else keep every id whose z is >= the k-th largest z (ties kept); topk >= vocab keeps all.
 *   topp: 0 or 1 = off; else, after top-k, keep id i iff the softmax mass of the kept ids with z_j > z_i is below topp.
 *   top-k and top-p need vocab_size <= 4096 (MT3_ERR_UNSUPPORTED otherwise).
 *   key: the 64-bit Philox key (a JAX PRNGKey's two words as they are).  row0: row b draws from stream row0 + b.
 *   rescale_log_probs: != 0, token scores are log-probabilities under the distribution sampled from,
 *     z[next] - logsumexp(kept z) (T5X's default); 0, logits[next] - logsumexp(logits row), as greedy's. */
typedef struct mt3_sample_params {
  float temperature;
  int32_t topk;
  float topp;
  uint32_t key[2];
  uint32_t row0;
  int32_t rescale_log_probs;
} mt3_sample_params;

/* mt3_generate_prompted with flags | MT3_GEN_SAMPLE: each free position draws its token from the filtered softmax of
 * z by the Gumbel-max rule, next = argmax_i (z_i - log(-log(u_i))) over the kept ids (the first id wins a tie), with
 * u_i from Philox4x32-10 at counter (i / 4, position, row0 + b, 0), word i % 4, mapped to (2 (w >> 9) + 1) 2^-24.  The
 * numbers of a row depend only on (key, row0 + b, position): not on graphs, early stop, prefill or batch size.
 * EOS, PAD, NaN rows, forced prompt positions and scores_out (the sum of the token scores) are greedy's.
 * params HOST (required with MT3_GEN_SAMPLE, MT3_ERR_BAD_ARG otherwise, as are a temperature that is not finite and
 * >= 0, topk < 0, topp outside [0, 1] and MT3_GEN_SAMPLE | MT3_GEN_BEAM1).  Without MT3_GEN_SAMPLE this is
 * mt3_generate_prompted.  Synchronises the stream once to copy params. */
int mt3_generate_sampled(mt3_model* m, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt, int32_t prompt_len,
                         int32_t* tokens_out, float* token_scores_out, float* scores_out, int32_t* steps_run, void* workspace,
                         int64_t workspace_bytes, const mt3_sample_params* params, void* stream);

/* mt3_generate_sampled with an additive logit bias per sequence: which tokens the loop may emit (e.g. only some instruments).
 *   logit_bias DEV f32, row b at logit_bias + b * bias_ld; bias_ld = 0 gives every sequence the same row, otherwise
 *   bias_ld >= vocab_size.  Each entry is finite or -inf (-inf suppresses the id), and each row keeps at least one finite id.
 *   Every token picker (greedy, MT3_GEN_BEAM1, MT3_GEN_SAMPLE) behaves exactly as if the model had produced
 *     l'[b, i] = -inf where logit_bias[b, i] == -inf, else logits[b, i] + logit_bias[b, i] (one float32 add)
 *   instead of its logits: the choice of token, the NaN rule (a NaN at a suppressed id is never emitted), EOS, and every
 *   score.  Token scores are therefore log-probabilities under the constrained model -- greedy l'[next] - logsumexp(l');
 *   beam1's candidates, "prefix + EOS" hypotheses and length-normalised score; sampling z = l' / temperature, its top-k /
 *   top-p cuts and Gumbel-max over z, and l'[next] - logsumexp(l') with rescale_log_probs = 0.
 *   Forced prompt positions are the caller's tokens even where suppressed.  A sequence whose EOS is -inf cannot finish before
 *   num_steps.  With a bias of all zeros every output is bit-identical to an unbiased call.  mt3_decode_teacher_forced and
 *   mt3_decode_step stay unbiased.
 * The rows are copied into the model workspace and checked on the device before the encoder runs (one small kernel and an
 * 8-byte copy back, which synchronises the stream): a NaN or +inf entry, a row without a finite entry, or a bias_ld that is
 * neither 0 nor >= vocab_size returns MT3_ERR_BAD_ARG and leaves the model usable.  The biased pickers run in CUDA graphs of
 * their own, with no extra launch per step.  With logit_bias == NULL this is mt3_generate_sampled, bit for bit. */
int mt3_generate_biased(mt3_model* m, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt, int32_t prompt_len,
                        int32_t* tokens_out, float* token_scores_out, float* scores_out, int32_t* steps_run, void* workspace,
                        int64_t workspace_bytes, const mt3_sample_params* params, const float* logit_bias, int64_t bias_ld,
                        void* stream);

/* GenericTokenVocabulary._decode_tf (vocabularies.py:241-271): ids DEV i32 [B, L]
 * -> out DEV i32 [B, L] with id-3, EOS-and-after = -1, invalid = -2. */
int mt3_vocab_decode(const int32_t* ids, int32_t batch, int32_t length, int32_t num_regular_tokens, int32_t* out,
                     void* stream);

/* layers.dot_product_attention(query, key, value, bias=None) (layers.py:85-157) as a standalone op, float32, any head_dim:
 * softmax(q k^T + bias) v with no 1/sqrt(d) scaling.  q DEV f32 [batch, q_len, heads, head_dim]; k, v DEV f32
 * [batch, kv_len, heads, head_dim]; bias DEV f32 [batch, heads, q_len, kv_len] or NULL (the reference's combined mask /
 * relative-position bias, layers.py:143-146; broadcasting is the caller's job); out DEV f32 like q.  The model's own
 * attention kernels specialise this op for head_dim 64 and the two mask shapes MT3 uses (all-ones, causal-to-length). */
int mt3_dot_product_attention_f32(const float* q, const float* k, const float* v, const float* bias, int32_t batch,
                                  int32_t q_len, int32_t kv_len, int32_t num_heads, int32_t head_dim, float* out, void* stream);

/* Measurement hook for bench.py's roofline leg: launches one named hot kernel `iters` times at
 * the shapes of the bound workspace, cycling over the decoder/encoder layers so that successive
 * launches touch different memory.  kind: MT3_K_* below; `pos` = KV-cache length - 1 for the
 * self-attention kernel.  Results are scratch; call mt3_cross_kv again before decoding. */
enum {
  MT3_K_DEC_SELF_ATTN = 0,
  MT3_K_DEC_CROSS_ATTN = 1,
  MT3_K_DEC_QKV_GEMM = 2,
  MT3_K_ENC_QKV_GEMM = 3,
  MT3_K_ENC_ATTN = 4
};
int mt3_debug_launch(mt3_model* m, int32_t kind, int32_t pos, int32_t iters, void* stream);

/* Measurement hook: device timeline of ONE greedy decode step at cache position `pos` (>= 2), replayed as a
 * CUDA graph exactly like mt3_generate's step.  Every decode GEMM / attention node records into its slot of
 * `out` (host, [max_slots][16] u64): [0] earliest CTA start, [1] latest CTA end (ns, %globaltimer),
 * [2..6] SM-clock deltas of CTA (0,0) at its internal phase boundaries.  `names` receives the slot names,
 * newline separated.  Clobbers the decode state (position, tokens); call mt3_encode/mt3_cross_kv first. */
int mt3_debug_trace_step(mt3_model* m, int32_t pos, uint64_t* out, int32_t max_slots, char* names,
                         int32_t names_bytes, int32_t* n_slots, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MT3_B200_H_ */
