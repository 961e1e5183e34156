// Test-only shared library (libmt3kernels.so): thin extern "C" launchers for the hot-path kernels, one kernel per call,
// on caller-provided device pointers, on the legacy default stream.  Each calls the launcher the kernel's header defines
// and model.cu uses, so grid, block, shared memory and attributes are the model's own.  tests/test_kernel_parity.py and
// tests/test_decode_loop_kernels.py load it with ctypes and compare every kernel with a float64 (or exact) reference at
// ragged shapes.  The argument structs (TcGemmArgs, GemmArgs, DecGemmArgs) are passed by pointer exactly as the kernels
// take them, so every field is reachable from the tests; kh_sizeof() lets the caller check its mirror of their layout.  Every launcher returns an MT3_* status; kh_last_error()
// is the text behind a non-zero one.
//
// Built with hidden visibility: the kernel headers' inline launchers keep one-time state in function-local statics
// (e.g. "the shared-memory attribute is set"), and exported, these would be unified with libmt3b200.so's copies when
// both libraries are loaded into one process -- the model would then launch its own kernels without their attributes.
// Only the kh_* entry points are exported.
#include <stdarg.h>

#include "../attention_tc.cuh"
#include "../decode.cuh"
#include "../gemm_simt.cuh"
#include "../gemm_tc.cuh"
#include "../layers.cuh"

namespace mt3 {
std::string& last_error() { static thread_local std::string e; return e; }
int fail(int code, const char* fmt, ...) {
  char buf[1024]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  last_error() = buf; return code;
}
std::atomic<uint64_t> g_launch_count{0};
}  // namespace mt3

using namespace mt3;

namespace {

// x -> kv_store<N> (p24 format) -> p24_elt: the exact path a K/V element takes from a GEMM epilogue into the decode
// attention's FMAs.  code[i] = the 24 stored bits (hi16 << 8 | lo8).
template <int N>
__global__ void p24_roundtrip_kernel(const float* __restrict__ x, float* __restrict__ y, uint32_t* __restrict__ code, long long n) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one group of 8 elements = one p24 chunk
  if (g * 8 >= n) return;
  __align__(16) char row[192];            // a whole p24 row: u16 part at 0, u8 part at 128; this group is elements 0..7
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = x[g * 8 + e];
#pragma unroll
  for (int d = 0; d < 8; d += N) kv_store<N>(row, 2, d, v + d);
  const uint4 hi = *reinterpret_cast<const uint4*>(row);
  const uint2 lo = *reinterpret_cast<const uint2*>(row + 128);
  const unsigned short* h16 = reinterpret_cast<const unsigned short*>(row);
  const unsigned char* l8 = reinterpret_cast<const unsigned char*>(row + 128);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    y[g * 8 + e] = p24_elt(hi, lo, e);
    code[g * 8 + e] = ((uint32_t)h16[e] << 8) | l8[e];
  }
}

}  // namespace

#define KH_API __attribute__((visibility("default")))

extern "C" {

KH_API const char* kh_last_error(void) { return last_error().c_str(); }

// 0 TcGemmArgs, 1 GemmArgs, 2 DecGemmArgs
KH_API long long kh_sizeof(int which) {
  return which == 0 ? (long long)sizeof(TcGemmArgs) : which == 1 ? (long long)sizeof(GemmArgs) : which == 2 ? (long long)sizeof(DecGemmArgs) : -1;
}

// A [M, K] (row pitch lda), Wt = W^T [N, K] (row pitch ldw); *_lo null unless split3.  C and the epilogue from *a.
KH_API int kh_tc_gemm(const float* a_hi, const float* a_lo, int lda, const float* w_hi, const float* w_lo, int ldw, const TcGemmArgs* a,
               int split3) {
  TcOperand opA, opB;
  int r = make_operand(&opA, a_hi, a_lo, (uint64_t)a->M, (uint64_t)a->K, (uint64_t)lda);
  if (r != MT3_OK) return r;
  r = make_operand(&opB, w_hi, w_lo, (uint64_t)a->N, (uint64_t)a->K, (uint64_t)ldw);
  if (r != MT3_OK) return r;
  return launch_tc_gemm(opA, opB, *a, split3 != 0, 0);
}

KH_API int kh_sgemm(const GemmArgs* a) { return launch_sgemm(*a, 0); }

// The encoder's form of the attention kernels.  qkv [B*T, 3*H*64] (hi, lo), vt [B*H*64, T] (hi, lo; keys in vt_key_slot()
// order), out [B*T, H*64]
KH_API int kh_enc_attention_tc(const float* qkv_hi, const float* qkv_lo, const float* vt_hi, const float* vt_lo, int B, int T, int H,
                        float* out_hi, float* out_lo, int split3, float* scratch) {
  MT3_REQUIRE(attention_tc_supported(T, T, false), MT3_ERR_UNSUPPORTED, "tc attention: T=%d is not supported", T);
  const int Q = H * 64;
  TcOperand op, opv;
  int r = make_operand(&op, qkv_hi, qkv_lo, (uint64_t)B * T, (uint64_t)3 * Q, (uint64_t)3 * Q);
  if (r != MT3_OK) return r;
  r = make_operand(&opv, vt_hi, vt_lo, (uint64_t)B * H * 64, (uint64_t)T, (uint64_t)T, 64);
  if (r != MT3_OK) return r;
  return launch_attention_tc(op, 0, T, op, Q, T, opv, B, H, out_hi, out_lo, split3 != 0, false, false, nullptr, 0, 0, scratch);
}

KH_API long long kh_enc_attention_tc_scratch_floats(int B, int T, int H) { return (long long)attention_tc_scratch_floats(B, T, T, H, false); }
KH_API int kh_enc_attention_tc_supported(int T) { return attention_tc_supported(T, T, false) ? 1 : 0; }

KH_API int kh_enc_attention_fp32(const float* qkv, int B, int T, int H, float* out, float* out_lo) {
  const int Q = H * 64;
  return launch_attention_fp32(qkv, 3 * Q, 0, qkv, 3 * Q, Q, 2 * Q, T, T, H, B, out, out_lo, Q, nullptr, 0, 0);
}

// The teacher-forced decoder's attention forms.  q [B*Tq, ldq] (head h at columns q_col0 + 64 h), k [B*Tk, ldk] (k_col0),
// hi and lo; vt [B*H*64, Tk] (keys in vt_key_slot() order); out [B*Tq, H*64].  causal: Tq = Tk (a multiple of 128) and
// key_valid [B, n_valid]; otherwise every key is visible.  P . V is split in TF32X3, as the pass runs it.
KH_API int kh_attention_tc(const float* q_hi, const float* q_lo, int ldq, int q_col0, int Tq, const float* k_hi, const float* k_lo, int ldk,
                           int k_col0, int Tk, const float* vt_hi, const float* vt_lo, int B, int H, float* out_hi, float* out_lo, int split3,
                           int causal, const int* key_valid, int n_valid, float* scratch) {
  TcOperand oq, ok, ov;
  int r = make_operand(&oq, q_hi, q_lo, (uint64_t)B * Tq, (uint64_t)ldq, (uint64_t)ldq);
  if (r != MT3_OK) return r;
  r = make_operand(&ok, k_hi, k_lo, (uint64_t)B * Tk, (uint64_t)ldk, (uint64_t)ldk);
  if (r != MT3_OK) return r;
  r = make_operand(&ov, vt_hi, vt_lo, (uint64_t)B * H * 64, (uint64_t)Tk, (uint64_t)Tk, 64);
  if (r != MT3_OK) return r;
  return launch_attention_tc(oq, q_col0, Tq, ok, k_col0, Tk, ov, B, H, out_hi, out_lo, split3 != 0, true, causal != 0, key_valid, n_valid,
                             0, scratch);
}
KH_API long long kh_attention_tc_scratch_floats(int B, int Tq, int Tk, int H, int causal) {
  return (long long)attention_tc_scratch_floats(B, Tq, Tk, H, causal != 0);
}

// the exact-fp32 forms: q [B*Tq, ldq], kv [B*Tk, ldkv] (keys at k_col0, values at v_col0); causal iff key_valid != null
KH_API int kh_attention_fp32(const float* q, int ldq, int q_col0, const float* kv, int ldkv, int k_col0, int v_col0, int Tq, int Tk, int H,
                             int B, float* out, float* out_lo, const int* key_valid, int n_valid) {
  return launch_attention_fp32(q, ldq, q_col0, kv, ldkv, k_col0, v_col0, Tq, Tk, H, B, out, out_lo, H * 64, key_valid, n_valid, 0);
}

// token scores of logits rows row0 .. row0 + n_rows - 1 of [B * Lp] (logits [n_rows, V])
KH_API int kh_token_score(const float* logits, int V, int row0, int n_rows, int Lp, int L, const int* target, const int* weight,
                          float* scores, float* logits_out) {
  return launch_token_score(logits, V, row0, n_rows, Lp, L, target, weight, scores, logits_out, 0);
}

KH_API int kh_dec_gemm_cluster(const DecGemmArgs* a) { return launch_dec_gemm_cluster(*a, false, 0); }
KH_API int kh_dec_gemm(const DecGemmArgs* a) { return launch_dec_gemm(*a, 0); }
KH_API int kh_dec_gemm_out_q(const DecGemmArgs* a0, const DecGemmArgs* a1) { return launch_dec_gemm_out_q(*a0, *a1, false, 0); }
// the same launches with the 3xTF32 tensor-core multiply (the decoder's path in gemm modes TF32X3 and TF32)
KH_API int kh_dec_gemm_cluster_tc(const DecGemmArgs* a) { return launch_dec_gemm_cluster(*a, true, 0); }
KH_API int kh_dec_gemm_out_q_tc(const DecGemmArgs* a0, const DecGemmArgs* a1) { return launch_dec_gemm_out_q(*a0, *a1, true, 0); }

KH_API int kh_dec_attention(int fmt, const float* q, int ldq, int q_off, const void* kv, int H, int cap, const int* len_ptr, int len_add,
                     int max_len, float* out, int ldo, const float* q_ssq, int q_ssq_n, int q_ssq_ld, float q_dim, float q_eps,
                     int pf_tiles, int B) {
  return launch_dec_attention(fmt, q, ldq, q_off, kv, H, cap, len_ptr, len_add, max_len, out, ldo, q_ssq, q_ssq_n, q_ssq_ld, q_dim, q_eps,
                              nullptr, pf_tiles, B, false, 0);
}

// n a multiple of 8; N = 1, 2 or 4 elements per kv_store call
KH_API int kh_p24_roundtrip(const float* x, float* y, uint32_t* code, long long n, int N) {
  MT3_REQUIRE(n % 8 == 0 && (N == 1 || N == 2 || N == 4), MT3_ERR_BAD_ARG, "p24 roundtrip: n=%lld N=%d", n, N);
  const unsigned grid = (unsigned)((n / 8 + 255) / 256);
  if (N == 1) p24_roundtrip_kernel<1><<<grid, 256>>>(x, y, code, n);
  else if (N == 2) p24_roundtrip_kernel<2><<<grid, 256>>>(x, y, code, n);
  else p24_roundtrip_kernel<4><<<grid, 256>>>(x, y, code, n);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// The decode loop's token pickers, embedding and the encoder's RMSNorm.
// argmax_step_kernel: n_cta CTAs starting at sequence b0 (B spans the whole batch: the arrival counter advances the
// position once all B sequences of the step have arrived, over however many launches).
KH_API int kh_argmax_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, int out_ld, int* tok_user,
                          int* state, int advance, int b0, const float* emb, const float* pe, int pe_rows, int D, float* y_next,
                          int n_cta) {
  return launch_argmax_step(logits, V, B, tok_cur, finished, tokens_out, nullptr, out_ld, nullptr, tok_user, state, advance, b0, emb, pe,
                            pe_rows, D, y_next, n_cta, nullptr, 0);
}

KH_API int kh_beam1_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, int out_ld, int* state,
                         float* beam_f, int* beam_i, float alpha, int max_len, const float* emb, const float* pe, int pe_rows, int D,
                         float* y_next) {
  return launch_beam1_step(logits, V, B, tok_cur, finished, tokens_out, nullptr, out_ld, nullptr, state, beam_f, nullptr, beam_i, alpha,
                           max_len, emb, pe, pe_rows, D, y_next, nullptr, 0);
}

KH_API int kh_beam1_finalize(int* tokens, int B, int L, int steps, const int* beam_i) {
  return launch_beam1_finalize(tokens, B, L, steps, beam_i, nullptr, nullptr, nullptr, nullptr, 0);
}

// The same kernels with token scores (mt3_generate_scored): token_scores [B, out_ld] (row stride out_ld, like tokens_out),
// fin_lp_eos [B], scores [B]; beam_f [B][2] as above.
KH_API int kh_argmax_step_scored(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                 int out_ld, int* tok_user, int* state, int advance, int b0, const float* emb, const float* pe, int pe_rows,
                                 int D, float* y_next, int n_cta) {
  return launch_argmax_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, nullptr, tok_user, state, advance, b0, emb,
                            pe, pe_rows, D, y_next, n_cta, nullptr, 0);
}

KH_API int kh_beam1_step_scored(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                int out_ld, int* state, float* beam_f, float* fin_lp_eos, int* beam_i, float alpha, int max_len,
                                const float* emb, const float* pe, int pe_rows, int D, float* y_next) {
  return launch_beam1_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, nullptr, state, beam_f, fin_lp_eos, beam_i,
                           alpha, max_len, emb, pe, pe_rows, D, y_next, nullptr, 0);
}

// The forced forms (mt3_generate_prompted): plen [B] prompt lengths; at pos < plen[b] the kernels emit tokens_out[b, pos]
// (which the caller fills) with score 0 and no finish.  token_scores (and fin_lp_eos) may be NULL.
KH_API int kh_argmax_step_forced(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                 int out_ld, const int* plen, int* tok_user, int* state, int advance, int b0, const float* emb,
                                 const float* pe, int pe_rows, int D, float* y_next, int n_cta) {
  return launch_argmax_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, tok_user, state, advance, b0, emb, pe,
                            pe_rows, D, y_next, n_cta, nullptr, 0);
}

// sample_step_kernel (mt3_generate_sampled): B CTAs, sp DEV (mt3_sample_params); token_scores and plen may be NULL.
// Top-k / top-p at V > kSampleMaxSortV are refused here, as mt3_generate_sampled refuses them.
KH_API int kh_sample_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores, int out_ld,
                          const int* plen, int* state, const mt3_sample_params* sp, int topk, float topp, const float* emb, const float* pe,
                          int pe_rows, int D, float* y_next) {
  MT3_REQUIRE(V <= kSampleMaxSortV || !((topk > 0 && topk < V) || (topp > 0.f && topp < 1.f)), MT3_ERR_UNSUPPORTED,
              "kh_sample_step: top-k / top-p need V <= %d", kSampleMaxSortV);
  return launch_sample_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D, y_next,
                            nullptr, 0);
}

KH_API int kh_beam1_step_forced(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                int out_ld, const int* plen, int* state, float* beam_f, float* fin_lp_eos, int* beam_i, float alpha,
                                int max_len, const float* emb, const float* pe, int pe_rows, int D, float* y_next) {
  return launch_beam1_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i,
                           alpha, max_len, emb, pe, pe_rows, D, y_next, nullptr, 0);
}

// The biased pickers (mt3_generate_biased): the forced forms above with bias [B, V] (row stride V), which the picker reads
// through biased_logit.  token_scores, fin_lp_eos and plen may be NULL; bias may not (NULL launches the unbiased kernel).
KH_API int kh_argmax_step_biased(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                 int out_ld, const int* plen, int* tok_user, int* state, int advance, int b0, const float* emb,
                                 const float* pe, int pe_rows, int D, float* y_next, int n_cta, const float* bias) {
  MT3_REQUIRE(bias, MT3_ERR_BAD_ARG, "kh_argmax_step_biased: null bias");
  return launch_argmax_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, tok_user, state, advance, b0, emb, pe,
                            pe_rows, D, y_next, n_cta, bias, 0);
}

KH_API int kh_beam1_step_biased(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                int out_ld, const int* plen, int* state, float* beam_f, float* fin_lp_eos, int* beam_i, float alpha,
                                int max_len, const float* emb, const float* pe, int pe_rows, int D, float* y_next, const float* bias) {
  MT3_REQUIRE(bias, MT3_ERR_BAD_ARG, "kh_beam1_step_biased: null bias");
  return launch_beam1_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i,
                           alpha, max_len, emb, pe, pe_rows, D, y_next, bias, 0);
}

KH_API int kh_sample_step_biased(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                                 int out_ld, const int* plen, int* state, const mt3_sample_params* sp, int topk, float topp, const float* emb,
                                 const float* pe, int pe_rows, int D, float* y_next, const float* bias) {
  MT3_REQUIRE(bias, MT3_ERR_BAD_ARG, "kh_sample_step_biased: null bias");
  MT3_REQUIRE(V <= kSampleMaxSortV || !((topk > 0 && topk < V) || (topp > 0.f && topp < 1.f)), MT3_ERR_UNSUPPORTED,
              "kh_sample_step_biased: top-k / top-p need V <= %d", kSampleMaxSortV);
  return launch_sample_step(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D, y_next,
                            bias, 0);
}

KH_API int kh_beam1_finalize_scored(int* tokens, int B, int L, int steps, const int* beam_i, float* token_scores, const float* beam_f,
                                    const float* fin_lp_eos, float* scores) {
  return launch_beam1_finalize(tokens, B, L, steps, beam_i, token_scores, beam_f, fin_lp_eos, scores, 0);
}

KH_API int kh_seq_score(const float* token_scores, int B, int L, float* scores) {
  return launch_seq_score(token_scores, B, L, scores, 0);
}

// y [b0 + n, D] rows b0 .. b0 + n - 1
KH_API int kh_embed(const int* tok, const float* emb, int D, int V, const float* pe, const int* pos_ptr, float* y, int b0, int n) {
  return launch_embed(tok, emb, D, V, pe, pos_ptr, y, b0, n, 0);
}

KH_API int kh_row_rstd(const float* x, const float* x_lo, int ld, int M, int D, float eps, float* rstd) {
  return launch_row_rstd(x, x_lo, ld, M, D, eps, rstd, 0);
}

KH_API int kh_rmsnorm(const float* x, const float* x_lo, int ldx, int M, int D, float eps, const float* g, float* y, int ldy) {
  return launch_rmsnorm(x, x_lo, ldx, M, D, eps, g, y, ldy, 0);
}

}  // extern "C"
