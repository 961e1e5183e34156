// Host orchestration of the MT3 encoder / decoder on sm_90a behind the C ABI.
//
// Reference semantics: network.py:44-85 (EncoderLayer), :88-155 (DecoderLayer), :158-193
// (Encoder), :196-262 (Decoder), :275-361 (Transformer.encode/decode); layers.py for the ops.
// Data layout in HBM (all fp32, row-major):
//   hidden h        [B*T, D]
//   qkv             [B*T, 3Q]   columns [q | k | v], each (head, 64)
//   cross K/V       [Ld][B][K|V][H][T][64]  head-major, fp32 or fp16 (hoisted: computed once per batch)
//   self K/V cache  [Ld][B][K|V][H][L][64]  head-major, fp32 or fp16 (append = 12 rows of 64 per sequence per layer)
// The reference's [B,H,D,L] cache layout (layers.py:249-260) is a TPU scatter trick; the
// ABI exposes tokens and logits, not the cache, so the layout is ours.
#include <string.h>
#include <math.h>
#include <string>
#include <vector>
#include <map>
#include <tuple>

#include "common.cuh"
#include "gemm_simt.cuh"
#include "gemm_tc.cuh"
#include "attention_tc.cuh"
#include "decode.cuh"
#include "layers.cuh"

namespace mt3 {

struct ParamEntry { std::string name; int64_t rows, cols, offset; };

static std::vector<ParamEntry> param_table(const mt3_model_config& c) {
  std::vector<ParamEntry> t;
  int64_t off = 0;
  auto add = [&](const std::string& n, int64_t r, int64_t co) {
    t.push_back({n, r, co, off});
    off += r * co;
  };
  const int64_t D = c.emb_dim, Q = (int64_t)c.num_heads * c.head_dim, F = c.mlp_dim, V = c.vocab_size;
  add("encoder/continuous_inputs_projection/kernel", c.input_depth, D);
  for (int i = 0; i < c.num_encoder_layers; ++i) {
    const std::string p = "encoder/layers_" + std::to_string(i) + "/";
    add(p + "pre_attention_layer_norm/scale", 1, D);
    add(p + "attention/query/kernel", D, Q);
    add(p + "attention/key/kernel", D, Q);
    add(p + "attention/value/kernel", D, Q);
    add(p + "attention/out/kernel", Q, D);
    add(p + "pre_mlp_layer_norm/scale", 1, D);
    add(p + "mlp/wi_0/kernel", D, F);
    add(p + "mlp/wi_1/kernel", D, F);
    add(p + "mlp/wo/kernel", F, D);
  }
  add("encoder/encoder_norm/scale", 1, D);
  add("decoder/token_embedder/embedding", V, D);
  for (int i = 0; i < c.num_decoder_layers; ++i) {
    const std::string p = "decoder/layers_" + std::to_string(i) + "/";
    add(p + "pre_self_attention_layer_norm/scale", 1, D);
    add(p + "self_attention/query/kernel", D, Q);
    add(p + "self_attention/key/kernel", D, Q);
    add(p + "self_attention/value/kernel", D, Q);
    add(p + "self_attention/out/kernel", Q, D);
    add(p + "pre_cross_attention_layer_norm/scale", 1, D);
    add(p + "encoder_decoder_attention/query/kernel", D, Q);
    add(p + "encoder_decoder_attention/key/kernel", D, Q);
    add(p + "encoder_decoder_attention/value/kernel", D, Q);
    add(p + "encoder_decoder_attention/out/kernel", Q, D);
    add(p + "pre_mlp_layer_norm/scale", 1, D);
    add(p + "mlp/wi_0/kernel", D, F);
    add(p + "mlp/wi_1/kernel", D, F);
    add(p + "mlp/wo/kernel", F, D);
  }
  add("decoder/decoder_norm/scale", 1, D);
  add("decoder/logits_dense/kernel", D, V);
  return t;
}

// K-major ("transposed", [N,K]) copy of a prepared weight for the wgmma path, optionally tf32 hi/lo split.
struct TcW { float* hi = nullptr; float* lo = nullptr; TcOperand op; int K = 0, N = 0; };
// An activation buffer [rows, ld]; lo != null when it is carried as a tf32 hi/lo pair.
struct Act { float* hi = nullptr; float* lo = nullptr; TcOperand op; };

// A bump allocator over one device region, in steps of `align` bytes (256 in the workspaces, one float in the weight slabs).
// base == nullptr only measures: take() returns null and `used` grows all the same, so the one function that carves a
// region also states its size.  take(0) is null and takes nothing.
struct Carve {
  char* base = nullptr;
  int64_t align = 256;
  int64_t used = 0;
  template <class T = float> T* take(int64_t n) {
    if (n <= 0) return nullptr;
    T* r = base ? (T*)(base + used) : nullptr;
    used += align_up(n * (int64_t)sizeof(T), align);
    return r;
  }
};

// What the full-sequence layer steps (seq_*) work on, for B sequences of T rows: the residual stream h, its RMSNorm
// statistic, qkv, the attention output ao and the MLP hidden g (lo planes in TF32X3).  Where the self-attention runs on
// the wgmma kernel (tc_attn), qkv also has its lo plane, V^T [B*H*64, T] exists and so does the key-split scratch;
// elsewhere no kernel reads them.  The encoder carves one set in the model workspace, the teacher-forced pass one in its own.
struct SeqActs {
  int B = 0, T = 0;
  bool tc_attn = false;
  Act h, qkv, vt, ao, g;
  float* rstd = nullptr;
  float* scratch = nullptr;
};

struct EncLayer { float *wqkv, *wo, *wi, *wo2; TcW t_wqkv, t_wo, t_wi, t_wo2; };
struct DecLayer {
  float *wqkv, *wo, *wq_c, *wkv_c, *wo_c, *wi, *wo2; float* wc1 = nullptr; TcW t_wkv_c;   // wc1: [Q+D, Q] = [Wo.Wq ; Wq]
  TcW t_wqkv, t_wo, t_wq_c, t_wo_c, t_wi, t_wo2;   // teacher-forced pass only: built on its first call (ensure_tf_weights)
};

// The buffers of the caller's model workspace, carved by carve_workspace
struct WsBuffers {
  SeqActs ea;                     // the encoder's activations
  Act a_x, a_enc;                 // TF32X3 only: hi/lo splits of the caller's encoder input and of `encoded`
  float* encoded = nullptr;
  char *ckv = nullptr, *skv = nullptr;   // head-major K/V rows (kv_row bytes each)
  float *dy = nullptr, *dy2 = nullptr;   // the decode step's residual stream and its ping-pong partner (dec_layer_outq)
  float* dssq = nullptr;          // [B][D/32] sum-of-squares partials
  float *dq = nullptr, *dao = nullptr, *dg = nullptr, *dlogits = nullptr;
  int *tok_cur = nullptr, *finished = nullptr, *tokens = nullptr, *state = nullptr;
  float* beam_f = nullptr; int* beam_i = nullptr;   // beam-size-1 search state (MT3_GEN_BEAM1)
  float* fin_lp_eos = nullptr;    // [B] EOS log-probability of each best finished hypothesis (beam_f's third float per sequence)
  float *tok_scores = nullptr, *seq_scores = nullptr;   // [B, L] and [B] of mt3_generate_scored
  int* plen = nullptr;            // [B] forced prompt lengths of the token pickers (0 = free from position 0)
  int* prompt_info = nullptr;     // {P = shortest prompt, 1 + first invalid row or 0} of prompt_scan_kernel
  int* pf_tok = nullptr;          // [2][B, L] decoder inputs and key-validity targets of the prefill pass
  mt3_sample_params* sample = nullptr;   // the sampling picker's parameters (MT3_GEN_SAMPLE), written once per generate
  float* bias = nullptr;          // [B, V] the token pickers' logit bias (mt3_generate_biased), written once per biased generate
  float* dpartial = nullptr;      // split-K scratch of the non-cluster decode GEMM
  int* dcounters = nullptr;       // [dec_tiles()]
};

constexpr int kPeRows = 2048;     // rows of the sinusoid table (FixedEmbed.max_length, layers.py:565)

struct Model : WsBuffers {
  mt3_model_config cfg;
  int D, H, Q, F, V, Le, Ld, L;
  float* slab = nullptr;          // all prepared weights
  float* slab_tc = nullptr;       // K-major (and hi/lo) copies for the wgmma path
  bool tc = false, split3 = false;
  TcW t_w_in;
  bool pdl_attn = true;           // programmatic dependent launch of the decode attention kernels (K/V streamed under the
                                  // preceding GEMM); MT3_PDL=0 turns it off, the reference for the value-neutrality tests
  int pf_attn = 16;               // MT3_PF_ATTN=n: the decode-step attention kernels prefetch the n K/V tiles that follow their
                                  // shared-memory ring into L2 while they wait under the preceding GEMM (decode.cuh; value-neutral;
                                  // 0 = off)
  int pf_kv = 4;        // MT3_PF_KV=n: the GEMM node before each layer's QKV projection prefetches the first n tiles of every
                                  // K and V stream of that layer's self-attention into L2 (decode.cuh KvStage; value-neutral; 0 = off)
  bool pdl_gemm = true;           // programmatic edges between consecutive decode GEMM nodes (dec_chain()); MT3_PDL_GEMM=0 turns
                                  // them off, the reference for the value-neutrality tests
  int kv_fmt = 0;                 // cfg.kv_cache_format: storage format of the self and cross K/V rows (kv_dest())
  int kv_row = 256;               // bytes per K/V row of 64 elements
  // debug timeline (mt3_debug_trace_step): while `tracing` is set every decode GEMM / attention launch gets a slot
  unsigned long long* trace = nullptr;
  bool tracing = false;
  std::vector<std::string> trace_names;
  bool tc_attn_ok = true;         // MT3_TC_ATTENTION=0 in the environment forces the exact-fp32 attention kernel
  float* w_in = nullptr;
  std::vector<EncLayer> enc;
  float* enc_norm_g = nullptr;
  float* emb = nullptr;
  std::vector<DecLayer> dec;
  float* w_logits = nullptr;
  TcW t_w_logits;                 // teacher-forced pass only, like DecLayer::t_wqkv ...
  float* slab_tf = nullptr;       // K-major (and hi/lo) decoder weights of the teacher-forced pass; null until its first call
  float* pe = nullptr;            // [kPeRows, D] sinusoid table

  // workspace (caller-owned; its buffers are the WsBuffers)
  char* ws = nullptr;
  int B = 0, T = 0;
  bool have_cross = false;
  int host_pos = 0;               // host mirror of the device position (cache overflow guard)

  // CUDA graph of one greedy step
  cudaStream_t cap_stream = nullptr;
  cudaGraph_t graph = nullptr;              // the graph of the CURRENT (workspace, B, T) binding ...
  cudaGraphExec_t graph_exec = nullptr;
  uint64_t graph_kernels = 0;
  int graph_mode = 1;
  struct StepGraph { cudaGraph_t g; cudaGraphExec_t e; uint64_t kernels; };
  std::map<std::tuple<const void*, int, int, int>, StepGraph> graphs;   // ... kept per binding, so that a short tail batch does not
                                                                   // throw away the full batch's graph (and vice versa)
  int* h_flag = nullptr;          // pinned
};

// byte address of layer l's K/V block: [B][K|V][H][cap] rows of kv_row bytes
static char* kv_layer(const Model* m, char* base, int l, int cap) {
  return base + (int64_t)l * m->B * cap * 2 * m->H * m->kv_row;
}

// out [Q + D, Q]: rows [0, Q) = Wo [Q, D] . Wq [D, Q] accumulated in fp64 and rounded once; rows [Q, Q + D) = Wq.
// (q = rstd . (y + o.Wo) . Wq  =  rstd . ([o | y] . out): the out-projection folded into the query projection.)
__global__ void compose_out_q_kernel(const float* __restrict__ wo, const float* __restrict__ wq, int Q, int D, float* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= Q) return;
  if (i < Q) {
    double acc = 0.0;
    for (int k = 0; k < D; ++k) acc += (double)wo[(long long)i * D + k] * (double)wq[(long long)k * Q + j];
    out[(long long)i * Q + j] = (float)acc;
  } else {
    out[(long long)i * Q + j] = wq[(long long)(i - Q) * Q + j];
  }
}

static int prep_copy(cudaStream_t s, const float* src, int K, int N, const float* g, float* dst, int ldd, int col_off,
                     int col_stride) {
  const long long n = (long long)K * N;
  scale_copy_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(src, K, N, g, dst, ldd, col_off, col_stride);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// K-major copy (hi/lo in TF32X3) of w [K, N] for the wgmma path: carved from c and, unless c only measures, filled
static int prep_tc_weight(Model* m, cudaStream_t s, const float* w, int K, int N, Carve& c, TcW* out) {
  out->K = K; out->N = N;
  out->hi = c.take((int64_t)K * N);
  out->lo = c.take(m->split3 ? (int64_t)K * N : 0);
  if (!c.base) return MT3_OK;
  transpose_split_kernel<<<dim3(cdiv(N, 32), cdiv(K, 32)), dim3(32, 8), 0, s>>>(w, K, N, out->hi, out->lo);
  MT3_LAUNCH_CHECK();
  return make_operand(&out->op, out->hi, out->lo, N, K, K);
}

// A weight slab: fill(Carve&) runs once to measure it (launching nothing), then on the allocation, whose launches are
// waited for.  *out is set on success only.
template <class Fill>
static int make_slab(float** out, const char* what, cudaStream_t s, Fill fill) {
  Carve c{nullptr, sizeof(float)};
  MT3_TRY(fill(c));
  char* slab = nullptr;
  cudaError_t e = cudaMalloc((void**)&slab, (size_t)c.used);
  if (e != cudaSuccess) return fail(MT3_ERR_CUDA, "%s: cudaMalloc -> %s", what, cudaGetErrorString(e));
  c = Carve{slab, sizeof(float)};
  int rc = fill(c);
  if (rc == MT3_OK && (e = cudaStreamSynchronize(s)) != cudaSuccess) rc = fail(MT3_ERR_CUDA, "%s -> %s", what, cudaGetErrorString(e));
  if (rc != MT3_OK) {
    cudaFree(slab);
    return rc;
  }
  *out = (float*)slab;
  return MT3_OK;
}

// The epilogue of an encoder-side GEMM C[M, N] = A[M, K] . W[K, N], in the wgmma kernel's terms (enc_gemm() maps it onto
// the SIMT kernel's).
static TcGemmArgs gemm_epi(int M, int N, int K, float* C_hi, float* C_lo, int ldc) {
  TcGemmArgs a;
  memset(&a, 0, sizeof(a));
  a.M = M; a.N = N; a.K = K; a.C_hi = C_hi; a.C_lo = C_lo; a.ldc = ldc; a.n_split = N; a.epi = EPI_STORE;
  return a;
}

// One encoder-side GEMM on the back end gemm_mode picks: wgmma on the K-major copy tw, or the SIMT kernel on the row-major
// w.  A is dense (row pitch K), w has row pitch N.  Activations that feed a GEMM are carried as tf32 hi/lo pairs in TF32X3
// mode only, and the V^T store only feeds the wgmma attention, so the SIMT kernel never sees a lo plane or V^T.
static int enc_gemm(const Model* m, const Act& A, const float* w, const TcW& tw, const TcGemmArgs& e, cudaStream_t s) {
  if (m->tc) return launch_tc_gemm(A.op, tw.op, e, m->split3, s);
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.A = A.hi; a.lda = e.K; a.B = w; a.ldb = e.N; a.M = e.M; a.N = e.N; a.K = e.K;
  a.row_scale = e.row_scale; a.epi = e.epi; a.R = e.R_hi; a.ldr = e.ldr; a.pe = e.pe; a.pe_T = e.pe_T; a.pe_ld = e.pe_ld;
  a.C = e.C_hi; a.ldc = e.ldc;
  a.n_split = e.n_split; a.C1 = e.C1; a.kv_fmt = e.kv_fmt; a.hm_rows_per_b = e.hm_rows_per_b; a.hm_cap = e.hm_cap; a.hm_H = e.hm_H;
  a.hm_pos = e.hm_pos;
  return launch_sgemm(a, s);
}

// an activation [rows, cols] (lo null unless TF32X3); on the wgmma path also its TMA operand
static int make_act(const Model* m, float* hi, float* lo, int64_t rows, int cols, Act* a, uint32_t box_rows = 128) {
  a->hi = hi; a->lo = lo;
  return m->tc ? make_operand(&a->op, hi, lo, (uint64_t)rows, (uint64_t)cols, (uint64_t)cols, box_rows) : MT3_OK;
}
// make_act on an activation carved from c, with a lo plane when `lo`
static int carve_act(const Model* m, Carve& c, int64_t rows, int cols, bool lo, Act* a, uint32_t box_rows = 128) {
  float* hi = c.take(rows * cols);
  float* l = c.take(lo ? rows * cols : 0);
  return c.base ? make_act(m, hi, l, rows, cols, a, box_rows) : MT3_OK;
}

// x [M, K], owned by the caller, as the A operand of an encoder-side GEMM; in TF32X3 mode it is split into `pair` first.
static int enc_input(const Model* m, const float* x, int64_t M, int K, const Act& pair, Act* out, cudaStream_t s) {
  if (m->split3) {
    const long long n4 = M * K / 4;
    split_pair_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, s>>>(x, pair.hi, pair.lo, n4);
    MT3_LAUNCH_CHECK();
    *out = pair;
    return MT3_OK;
  }
  return make_act(m, const_cast<float*>(x), nullptr, M, K, out);
}

// Attention on the wgmma kernel: the mode asks for it and the kernel takes the shape.
static bool tc_attention(const Model* m, int Tq, int Tk, bool causal) {
  return m->tc && m->tc_attn_ok && attention_tc_supported(Tq, Tk, causal);
}

// The activations of B sequences of T rows; other_scratch: floats of attention scratch another attention of the same pass
// shares with the self-attention's
static int carve_seq(const Model* m, Carve& c, int B, int T, bool causal, int64_t other_scratch, SeqActs* a) {
  const int64_t M = (int64_t)B * T;
  const bool s3 = m->split3;
  a->B = B; a->T = T;
  a->tc_attn = tc_attention(m, T, T, causal);
  MT3_TRY(carve_act(m, c, M, m->D, s3, &a->h));
  a->rstd = c.take(M);
  MT3_TRY(carve_act(m, c, M, 3 * m->Q, s3 && a->tc_attn, &a->qkv));
  if (a->tc_attn) MT3_TRY(carve_act(m, c, (int64_t)B * m->H * 64, T, s3, &a->vt, 64));
  MT3_TRY(carve_act(m, c, M, m->Q, s3, &a->ao));
  MT3_TRY(carve_act(m, c, M, m->F, s3, &a->g));
  a->scratch = c.take(std::max(a->tc_attn ? attention_tc_scratch_floats(B, T, T, m->H, causal) : 0, other_scratch));
  return MT3_OK;
}

// The layer steps of a full sequence, shared by the encoder (network.py:44-85) and the teacher-forced decoder pass
// (:88-155), on the B * T rows of a.h.  RMSNorm statistic of h, applied as the next GEMM's row scale
static int seq_rstd(const Model* m, const SeqActs& a, cudaStream_t s) {
  return launch_row_rstd(a.h.hi, a.h.lo, m->D, a.B * a.T, m->D, 1e-6f, a.rstd, s);
}
// QKV projection into qkv [B*T, 3Q].  The wgmma self-attention needs qkv as a tf32 hi/lo pair (TF32X3) and the V third
// also transposed per head into vt: the K-major operand of P.V
static int seq_qkv(const Model* m, const SeqActs& a, const float* w, const TcW& tw, cudaStream_t s) {
  const int Q = m->Q;
  TcGemmArgs e = gemm_epi(a.B * a.T, 3 * Q, m->D, a.qkv.hi, a.qkv.lo, 3 * Q);
  e.row_scale = a.rstd;
  if (a.tc_attn) {
    e.VT_hi = a.vt.hi; e.VT_lo = a.vt.lo; e.vt_col0 = 2 * Q; e.vt_T = a.T; e.vt_H = m->H;
  }
  return enc_gemm(m, a.h, w, tw, e, s);
}
// Self-attention from qkv into ao: on the wgmma kernel where tc_attn, else exact fp32.  key_valid [B, n_valid]: causal
// with per-key validity (make_decoder_mask); null: every key visible.  split_p: P . V in 3xTF32 too (TF32X3; see
// attention_tc_kernel's PSPLIT).
static int seq_self_attention(const Model* m, const SeqActs& a, const int* key_valid, int n_valid, bool split_p, cudaStream_t s) {
  const int Q = m->Q;
  if (a.tc_attn)
    return launch_attention_tc(a.qkv.op, 0, a.T, a.qkv.op, Q, a.T, a.vt.op, a.B, m->H, a.ao.hi, a.ao.lo, m->split3, split_p,
                               key_valid != nullptr, key_valid, n_valid, s, a.scratch);
  return launch_attention_fp32(a.qkv.hi, 3 * Q, 0, a.qkv.hi, 3 * Q, Q, 2 * Q, a.T, a.T, m->H, a.B, a.ao.hi, a.ao.lo, Q, key_valid, n_valid,
                               s);
}
// h += A . W: the attention out-projections (A = attention output) and the MLP out-projection (A = g)
static int seq_residual(const Model* m, const SeqActs& a, const Act& A, int K, const float* w, const TcW& tw, cudaStream_t s) {
  const int D = m->D;
  TcGemmArgs e = gemm_epi(a.B * a.T, D, K, a.h.hi, a.h.lo, D);
  e.epi = EPI_RESIDUAL; e.R_hi = a.h.hi; e.R_lo = a.h.lo; e.ldr = D;
  return enc_gemm(m, A, w, tw, e, s);
}
// gated-GELU MLP-in into g [B*T, F]
static int seq_mlp_in(const Model* m, const SeqActs& a, const float* w, const TcW& tw, cudaStream_t s) {
  const int F = m->F;
  TcGemmArgs e = gemm_epi(a.B * a.T, 2 * F, m->D, a.g.hi, a.g.lo, F);
  e.row_scale = a.rstd; e.epi = EPI_GATED_GELU;
  return enc_gemm(m, a.h, w, tw, e, s);
}

// Encoder (network.py:158-193): input projection + PE, the layers, and the closing RMSNorm into `encoded`.
static int encode_impl(Model* m, const float* x, float* encoded, cudaStream_t s) {
  const SeqActs& a = m->ea;
  const int M = m->B * m->T, D = m->D, depth = m->cfg.input_depth;
  // the exact-fp32 attention kernel's limit, in every mode
  MT3_REQUIRE(attention_fp32_smem(m->T) <= kAttFp32MaxSmem, MT3_ERR_UNSUPPORTED, "encode: input_length %d too long for the attention kernel",
              m->T);
  Act ax;
  MT3_TRY(enc_input(m, x, M, depth, m->a_x, &ax, s));
  {
    TcGemmArgs e = gemm_epi(M, D, depth, a.h.hi, a.h.lo, D);
    e.epi = EPI_ADD_PE; e.pe = m->pe; e.pe_T = m->T; e.pe_ld = D;
    MT3_TRY(enc_gemm(m, ax, m->w_in, m->t_w_in, e, s));
  }
  for (int l = 0; l < m->Le; ++l) {
    const EncLayer& w = m->enc[l];
    MT3_TRY(seq_rstd(m, a, s));
    MT3_TRY(seq_qkv(m, a, w.wqkv, w.t_wqkv, s));
    MT3_TRY(seq_self_attention(m, a, nullptr, 0, false, s));
    MT3_TRY(seq_residual(m, a, a.ao, m->Q, w.wo, w.t_wo, s));
    MT3_TRY(seq_rstd(m, a, s));
    MT3_TRY(seq_mlp_in(m, a, w.wi, w.t_wi, s));
    MT3_TRY(seq_residual(m, a, a.g, m->F, w.wo2, w.t_wo2, s));
  }
  return launch_rmsnorm(a.h.hi, a.h.lo, D, M, D, 1e-6f, m->enc_norm_g, encoded, D, s);
}

// Output tiles of the widest decode GEMM (QKV, MLP-in or logits): the length of the decode GEMMs' tile counters
static int dec_tiles(const Model* m) { return cdiv(std::max(std::max(3 * m->Q, 2 * m->F), m->V), kDecBN); }

// The hoisted cross-attention K/V of every decoder layer, head-major, and the reset of the decode state.
static int cross_kv_impl(Model* m, const float* encoded, cudaStream_t s) {
  const int M = m->B * m->T, D = m->D, Q = m->Q;
  Act ae;
  MT3_TRY(enc_input(m, encoded, M, D, m->a_enc, &ae, s));
  for (int l = 0; l < m->Ld; ++l) {
    TcGemmArgs a = gemm_epi(M, 2 * Q, D, nullptr, nullptr, 2 * Q);
    a.n_split = 0; a.C1 = kv_layer(m, m->ckv, l, m->T); a.kv_fmt = m->kv_fmt; a.hm_rows_per_b = m->T; a.hm_cap = m->T; a.hm_H = m->H;
    MT3_TRY(enc_gemm(m, ae, m->dec[l].wkv_c, m->dec[l].t_wkv_c, a, s));
  }
  MT3_CUDA_CHECK(cudaMemsetAsync(m->state, 0, 4 * sizeof(int), s));
  MT3_CUDA_CHECK(cudaMemsetAsync(m->dcounters, 0, (size_t)dec_tiles(m) * sizeof(int), s));
  MT3_CUDA_CHECK(cudaMemsetAsync(m->finished, 0, (size_t)m->B * sizeof(int), s));
  MT3_CUDA_CHECK(cudaMemsetAsync(m->tok_cur, 0, (size_t)m->B * sizeof(int), s));
  m->have_cross = true;
  m->host_pos = 0;
  return MT3_OK;
}

constexpr int kTraceSlots = 256, kTraceWords = 16;   // words 8..15: %smid of the 8 CTAs of tile 0's cluster
static unsigned long long* trace_slot(Model* m, const char* name) {
  if (!m->tracing || (int)m->trace_names.size() >= kTraceSlots) return nullptr;
  m->trace_names.push_back(name);
  return m->trace + (size_t)(m->trace_names.size() - 1) * kTraceWords;
}

// Decode-step GEMM on M = B rows in blocks of 64: split-K cluster kernel with the RMSNorm statistic fused (decode.cuh);
// its multiply is exact fp32 in gemm_mode SIMT and 3xTF32 on the tensor cores in both tensor modes (single-pass TF32
// stays an encoder-only trade).  The non-cluster kernel (exact fp32) for K the cluster kernel does not tile.
// name: the node's trace name (mt3_debug_trace_step).
static int dec_gemm(Model* m, const char* name, const float* A, int lda, const float* W, int N, int K, int norm, int epi, float* C,
                    int ldc, int n_split, char* kv, const int* pos, cudaStream_t s, const KvStage& kst = KvStage{},
                    const DecChain& ch = DecChain{}) {
  for (int r0 = 0; r0 < m->B; r0 += kDecBM) {
    DecGemmArgs a;
    memset(&a, 0, sizeof(a));
    a.A = A + (int64_t)r0 * lda; a.lda = lda; a.W = W; a.ldw = N; a.M = std::min(kDecBM, m->B - r0);
    a.N = N; a.K = K;
    a.norm = norm; a.eps = 1e-6f; a.epi = epi;
    a.R = C + (int64_t)r0 * ldc; a.ldr = ldc;                  // residual is always added in place
    a.C = C + (int64_t)r0 * ldc; a.ldc = ldc; a.n_split = n_split;
    if (kv) {  // rows_per_b = 1: skip r0 sequences, each 2*H*cap rows
      a.C1 = kv + (int64_t)r0 * 2 * m->H * m->L * m->kv_row; a.kv_fmt = m->kv_fmt;
      a.hm_rows_per_b = 1; a.hm_cap = m->L; a.hm_H = m->H; a.hm_pos = pos;
    }
    a.partial = m->dpartial;
    a.counters = m->dcounters;
    a.trace = trace_slot(m, name);
    int rc = launch_dec_gemm_cluster(a, m->tc, s, r0 == 0 ? kst : KvStage{}, ch);
    if (rc == MT3_ERR_UNSUPPORTED) rc = launch_dec_gemm(a, s);
    MT3_TRY(rc);
  }
  return MT3_OK;
}

// prefetch: the launch is part of a decode step (the kernel starts under the preceding GEMM): L2 prefetch of m->pf_attn tiles
static int dec_attention(Model* m, const float* q, const char* kv, int cap, const int* len_ptr, int len_add, float* out, cudaStream_t s,
                         const float* q_ssq = nullptr, bool prefetch = false) {
  return launch_dec_attention(m->kv_fmt, q, m->Q, 0, kv, m->H, cap, len_ptr, len_add, std::max(m->L, m->T), out, m->Q, q_ssq, m->D / 32,
                              m->D / 32, (float)m->D, 1e-6f, trace_slot(m, len_ptr ? "attn_self" : "attn_cross"),
                              prefetch ? m->pf_attn : 0, m->B, m->pdl_attn, s);
}

// y_out = y_in + o.Wo  and  q_raw = [o | y_in].[Wo.Wq ; Wq]  in ONE launch; the RMSNorm factor of y_out is applied to
// q inside the cross-attention kernel from the per-tile sums of squares this launch leaves in m->dssq.
// MT3_ERR_UNSUPPORTED (nothing launched) unless B <= 64 and the mt3 widths Q = 384, D = 512.
static int dec_gemm_out_q(Model* m, const DecLayer& w, const float* y_in, float* y_out, cudaStream_t s) {
  const int D = m->D, Q = m->Q;
  if (m->B > kDecBM || Q != 384 || D != 512) return MT3_ERR_UNSUPPORTED;
  DecGemmArgs a0, a1;
  memset(&a0, 0, sizeof(a0));
  a0.A = m->dao; a0.lda = Q; a0.W = w.wo; a0.ldw = D; a0.M = m->B; a0.N = D; a0.K = Q;
  a0.eps = 1e-6f; a0.epi = EPI_RESIDUAL; a0.R = y_in; a0.ldr = D; a0.C = y_out; a0.ldc = D; a0.n_split = D;
  a0.ssq_out = m->dssq; a0.ssq_ld = D / 32;
  a0.trace = trace_slot(m, "gemm_out+cross_q");
  memset(&a1, 0, sizeof(a1));
  a1.A = m->dao; a1.lda = Q; a1.A2 = y_in; a1.lda2 = D; a1.K0 = Q;
  a1.W = w.wc1; a1.ldw = Q; a1.M = m->B; a1.N = Q; a1.K = Q + D;
  a1.eps = 1e-6f; a1.epi = EPI_STORE; a1.C = m->dq; a1.ldc = Q; a1.n_split = Q;
  a1.R = a1.C; a1.ldr = Q;
  a1.trace = a0.trace;
  return launch_dec_gemm_out_q(a0, a1, m->tc, s);
}

// The state one decode step carries from layer to layer: the current residual-stream buffer (ping-pongs between m->dy
// and m->dy2 across fused out+query launches), and whether the cross-attention query in m->dq is the fused launch's
// un-normalised q_raw.
struct DecBranch { float* y; bool q_raw; };

// decoder input of the first step: E[tok_in] + PE[pos] into m->dy
static int dec_embed(Model* m, const int* tok_in, cudaStream_t s) {
  return launch_embed(tok_in, m->emb, m->D, m->V, m->pe, m->state, m->dy, 0, m->B, s);
}
// What the GEMM node before layer l's QKV projection prefetches of that layer's self-attention K/V; len_add: cache rows
// written before that attention's step beyond *m->state at the time the GEMM runs (1 when the argmax kernel, which
// advances the position, lies in between).
static KvStage kv_stage_for(const Model* m, int l, int len_add) {
  KvStage k{};
  if (m->pf_kv <= 0) return k;
  k.base = kv_layer(m, m->skv, l, m->L);
  k.len_ptr = m->state; k.len_add = len_add;
  k.streams = 2 * m->B * m->H;
  k.max_rows = m->pf_kv * (m->kv_fmt == MT3_KV_F32 ? 32 : 64);
  k.row_bytes = m->kv_row;
  k.stream_bytes = (long long)m->L * m->kv_row;
  return k;
}

// The programmatic edges of a decode GEMM node (DecChain): after_gemm -- its predecessor is a decode GEMM, which then lets
// it launch early (the node loads its weights under it); late -- this node triggers its successor after the cluster
// exchange.  Per edge, measured (DESIGN.md §3): MLP-in -> MLP-out and MLP-out -> QKV / logits trigger late; the cross
// out-projection (1.2 MB of weights, 128 CTAs) triggers right after its wait, so that the MLP-in loads its weights under
// it.  A GEMM before an attention kernel also triggers right after its wait: the attention kernel streams K/V under the
// GEMM.  A GEMM after an attention kernel is launched plainly: started under the attention kernel it was slower (the
// GEMM CTAs that find room start long before their cluster peers).  The argmax kernel -> next step's layer-0 QKV edge is
// not taken: the first step of every graph has no kernel before its QKV, and at one edge per step it could save at most
// about 1 us of a 580 us step.
static DecChain dec_chain(const Model* m, bool after_gemm, bool late) {
  DecChain c;
  c.pdl = m->pdl_gemm && after_gemm;
  c.late_trigger = m->pdl_gemm && late;
  return c;
}

// fused RMSNorm + QKV projection + K/V cache append (layers.py:238-240, :272-289); layer l > 0 follows the MLP-out GEMM
static int dec_layer_qkv(Model* m, const DecBranch& b, int l, cudaStream_t s) {
  return dec_gemm(m, "gemm_qkv_append", b.y, m->D, m->dec[l].wqkv, 3 * m->Q, m->D, 1, EPI_STORE, m->dq, m->Q, m->Q,
                  kv_layer(m, m->skv, l, m->L), m->state, s, KvStage{}, dec_chain(m, l > 0, false));
}
static int dec_layer_self(Model* m, int l, cudaStream_t s) {
  return dec_attention(m, m->dq, kv_layer(m, m->skv, l, m->L), m->L, m->state, 1, m->dao, s, nullptr, true);
}
// self-attention out-projection + residual, cross-attention query projection (one launch where the fused kernel
// takes the shape)
static int dec_layer_outq(Model* m, DecBranch& b, int l, cudaStream_t s) {
  const DecLayer& w = m->dec[l];
  const int D = m->D, Q = m->Q;
  float* y_next = (b.y == m->dy) ? m->dy2 : m->dy;      // the fused launch reads y while other CTAs write y': ping-pong
  const int rc = dec_gemm_out_q(m, w, b.y, y_next, s);
  b.q_raw = rc == MT3_OK;
  if (rc == MT3_OK) {
    b.y = y_next;
    return MT3_OK;
  }
  if (rc != MT3_ERR_UNSUPPORTED) return rc;
  MT3_TRY(dec_gemm(m, "gemm_attn_out", m->dao, Q, w.wo, D, Q, 0, EPI_RESIDUAL, b.y, D, D, nullptr, nullptr, s));
  return dec_gemm(m, "gemm_cross_q", b.y, D, w.wq_c, Q, D, 1, EPI_STORE, m->dq, Q, Q, nullptr, nullptr, s);
}
static int dec_layer_cross(Model* m, const DecBranch& b, int l, cudaStream_t s) {
  return dec_attention(m, m->dq, kv_layer(m, m->ckv, l, m->T), m->T, nullptr, m->T, m->dao, s, b.q_raw ? m->dssq : nullptr, true);
}
static int dec_layer_mlp(Model* m, const DecBranch& b, int l, cudaStream_t s) {
  const DecLayer& w = m->dec[l];
  const int D = m->D, Q = m->Q, F = m->F;
  MT3_TRY(dec_gemm(m, "gemm_attn_out", m->dao, Q, w.wo_c, D, Q, 0, EPI_RESIDUAL, b.y, D, D, nullptr, nullptr, s, KvStage{},
                   dec_chain(m, false, false)));
  MT3_TRY(dec_gemm(m, "gemm_mlp_in", b.y, D, w.wi, 2 * F, D, 1, EPI_GATED_GELU, m->dg, F, 2 * F, nullptr, nullptr, s, KvStage{},
                   dec_chain(m, true, true)));
  // followed by the next layer's QKV projection or by the logits projection
  MT3_TRY(dec_gemm(m, "gemm_mlp_out", m->dg, F, w.wo2, D, F, 0, EPI_RESIDUAL, b.y, D, D, nullptr, nullptr, s,
                   l + 1 < m->Ld ? kv_stage_for(m, l + 1, 0) : KvStage{}, dec_chain(m, true, true)));
  return MT3_OK;
}

// One decode step (network.py:303-361 -> :196-262 -> :88-155) for the whole batch.  tok_in DEV [B]; logits
// DEV [B,V]; greedy != 0 runs the argmax/bookkeeping kernel (tok_user optional), else only the position advances.
// 7 launches per layer: [norm+QKV+KV-append] [self-attn] [out+residual | norm+q] [cross-attn] [out+residual]
// [norm+gated-GELU MLP in] [MLP out+residual].
// loop_step: a step of mt3_generate's loop -- the decoder input m->dy was already written (by dec_embed before the first
// step, by the previous step's argmax kernel afterwards), and this step's argmax kernel writes the next one.
// scored: the token picker also writes each emitted token's log-probability to m->tok_scores (mt3_generate_scored).
// biased: the loop's token picker reads its logits through the logit bias m->bias (mt3_generate_biased).
static int decode_step_impl(Model* m, const int* tok_in, float* logits, int greedy, int* tok_user, int use_finished,
                            int* tokens_ws, cudaStream_t s, bool loop_step = false, bool scored = false, bool biased = false) {
  if (!loop_step) MT3_TRY(dec_embed(m, tok_in, s));
  DecBranch b{m->dy, false};
  for (int l = 0; l < m->Ld; ++l) {
    MT3_TRY(dec_layer_qkv(m, b, l, s));
    MT3_TRY(dec_layer_self(m, l, s));
    MT3_TRY(dec_layer_outq(m, b, l, s));
    MT3_TRY(dec_layer_cross(m, b, l, s));
    MT3_TRY(dec_layer_mlp(m, b, l, s));
  }
  MT3_TRY(dec_gemm(m, "gemm_logits", b.y, m->D, m->w_logits, m->V, m->D, 1, EPI_STORE, logits, m->V, m->V, nullptr, nullptr, s,
                   kv_stage_for(m, 0, 1), dec_chain(m, true, false)));
  float* y_next = loop_step ? m->dy : nullptr;
  float* tok_scores = scored ? m->tok_scores : nullptr;
  const float* bias = loop_step && biased ? m->bias : nullptr;
  if (greedy == 2) {        // T5X beam_search bookkeeping at num_decodes = 1 (generate loop only)
    MT3_TRY(launch_beam1_step(logits, m->V, m->B, m->tok_cur, m->finished, tokens_ws, tok_scores, m->L, m->plen, m->state, m->beam_f,
                              m->fin_lp_eos, m->beam_i, 0.6f, m->L, m->emb, m->pe, kPeRows, m->D, y_next, bias, s));
  } else if (greedy == 3) { // T5X temperature_sample's pick (generate loop only), parameters in the workspace
    MT3_TRY(launch_sample_step(logits, m->V, m->B, m->tok_cur, m->finished, tokens_ws, tok_scores, m->L, m->plen, m->state, m->sample,
                               m->emb, m->pe, kPeRows, m->D, y_next, bias, s));
  } else if (greedy) {
    MT3_TRY(launch_argmax_step(logits, m->V, m->B, use_finished ? m->tok_cur : nullptr, use_finished ? m->finished : nullptr, tokens_ws,
                               tok_scores, m->L, loop_step ? m->plen : nullptr, tok_user, m->state, 1, 0, m->emb, m->pe, kPeRows, m->D,
                               y_next, m->B, bias, s));
  } else {
    MT3_CUDA_CHECK(launch_kernel(advance_pos_kernel, dim3(1), dim3(1), 0, s, false, m->state));
    MT3_LAUNCH_CHECK();
  }
  return MT3_OK;
}

static void drop_graphs(Model* m) {
  for (auto& kv : m->graphs) {
    if (kv.second.e) cudaGraphExecDestroy(kv.second.e);
    if (kv.second.g) cudaGraphDestroy(kv.second.g);
  }
  m->graphs.clear();
  m->graph_exec = nullptr;
  m->graph = nullptr;
}

// make the graph of the current (workspace, B, T, decode mode) binding current, if one has been captured
static void select_graph(Model* m, int mode = 1) {
  m->graph_mode = mode;
  const auto it = m->graphs.find(std::make_tuple((const void*)m->ws, m->B, m->T, mode));
  if (it == m->graphs.end()) {
    m->graph = nullptr; m->graph_exec = nullptr; m->graph_kernels = 0;
  } else {
    m->graph = it->second.g; m->graph_exec = it->second.e; m->graph_kernels = it->second.kernels;
  }
}

// mode: 1 greedy, 2 beam-size-1 search, 3 sampling; nsteps consecutive decode steps per graph (the position lives on the device, so a
// graph of 16 steps is the single-step graph 16 times over: one graph launch and its ~3 us of inter-launch latency per 16 steps);
// scored: the token pickers write token scores (a graph of its own, so that the unscored graphs do no extra work);
// biased: the token pickers read the logit bias (a graph of its own, so that the unbiased graphs keep their kernels)
static int ensure_graph(Model* m, int mode, int nsteps, bool scored, bool biased) {
  const int key = mode | (scored ? 4 : 0) | (biased ? 8 : 0) | (nsteps << 8);
  if (m->graph_mode != key) select_graph(m, key);
  if (m->graph_exec) return MT3_OK;
  if (!m->cap_stream) MT3_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
  const uint64_t before = g_launch_count.load();
  MT3_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
  int r = MT3_OK;
  for (int i = 0; i < nsteps && r == MT3_OK; ++i)
    r = decode_step_impl(m, m->tok_cur, m->dlogits, mode, nullptr, 1, m->tokens, m->cap_stream, true, scored, biased);
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(m->cap_stream, &g);
  if (r != MT3_OK) {
    if (g) cudaGraphDestroy(g);
    return r;
  }
  if (e != cudaSuccess) return fail(MT3_ERR_CUDA, "cudaStreamEndCapture -> %s", cudaGetErrorString(e));
  m->graph = g;
  m->graph_kernels = g_launch_count.load() - before;
  g_launch_count.fetch_sub(m->graph_kernels);   // capture does not execute
  MT3_CUDA_CHECK(cudaGraphInstantiate(&m->graph_exec, m->graph, 0));
  // bound the cache: forget the graphs of other (workspace, B, T) bindings.  The current binding's stay: it has at most 24
  // (3 modes x scored or not x biased or not x 1 or 16 steps), and a caller may still hold one of them (mt3_generate_scored
  // keeps the 16-step graph while it makes sure of the single-step one).
  if (m->graphs.size() >= 32) {
    for (auto it = m->graphs.begin(); it != m->graphs.end();) {
      if (std::get<0>(it->first) != (const void*)m->ws || std::get<1>(it->first) != m->B || std::get<2>(it->first) != m->T) {
        cudaGraphExecDestroy(it->second.e);
        cudaGraphDestroy(it->second.g);
        it = m->graphs.erase(it);
      } else {
        ++it;
      }
    }
  }
  m->graphs[std::make_tuple((const void*)m->ws, m->B, m->T, key)] = Model::StepGraph{m->graph, m->graph_exec, m->graph_kernels};
  return MT3_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// Teacher-forced decoder pass (network.py:196-262, :327-335 with decode=False): all L positions at once, M = B * Lp rows
// (Lp = L rounded up to the attention query tile; rows past L are zero inputs that causality keeps away from the real
// positions).  The encoder's GEMM epilogues and back ends; causal self-attention and cross-attention on the wgmma kernel
// (attention_tc.cuh) or exactly in fp32 (layers.cuh); K/V in float32 that live in the caller's workspace for the pass
// only.  Touches none of the decode state (model workspace, caches, position, graphs).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kTfLogitRows = 8192;   // logits rows per chunk of the logits GEMM + score kernel (50 MB at V = 1536)

static int tf_pad(int L) { return cdiv(L, kAtQ) * kAtQ; }

// The pass's workspace: the full-sequence activations of B sequences of Lp causal rows, and what the cross-attention and
// the logits add: the queries qc, `encoded` as a tf32 hi/lo pair (TF32X3), one layer's cross K | V [B*T, 2Q] (V also as
// V^T in cvt where the cross-attention runs on the wgmma kernel, tcc) and one chunk of logits rows.
struct TfActs {
  SeqActs seq;
  bool tcc = false;
  Act qc, enc_pair, ckv, cvt;
  float* logits = nullptr;
};
static int carve_tf(const Model* m, Carve& c, int B, int T, int L, TfActs* w) {
  const int Lp = tf_pad(L);
  const int64_t M = (int64_t)B * Lp, Me = (int64_t)B * T;
  const bool s3 = m->split3;
  w->tcc = tc_attention(m, Lp, T, false);
  MT3_TRY(carve_seq(m, c, B, Lp, true, w->tcc ? attention_tc_scratch_floats(B, Lp, T, m->H, false) : 0, &w->seq));
  MT3_TRY(carve_act(m, c, M, m->Q, s3 && w->tcc, &w->qc));
  if (s3) MT3_TRY(carve_act(m, c, Me, m->D, true, &w->enc_pair));
  MT3_TRY(carve_act(m, c, Me, 2 * m->Q, s3 && w->tcc, &w->ckv));
  if (w->tcc) MT3_TRY(carve_act(m, c, (int64_t)B * m->H * 64, T, s3, &w->cvt, 64));
  w->logits = c.take(std::min(M, (int64_t)kTfLogitRows) * m->V);
  return MT3_OK;
}

static int64_t tf_workspace_bytes(const Model* m, int B, int T, int L) {
  Carve c;
  TfActs w;
  carve_tf(m, c, B, T, L, &w);
  return c.used;
}

// The caller's workspace for the pass over B x L targets and T inputs: non-null, 256-byte aligned and large enough
static int check_tf_workspace(const Model* m, const char* name, const void* ws, int64_t bytes, int B, int T, int L) {
  MT3_REQUIRE(ws && ((uintptr_t)ws & 255) == 0, MT3_ERR_WORKSPACE, "%s: the teacher-forced workspace must be non-null and 256-byte aligned",
              name);
  const int64_t need = tf_workspace_bytes(m, B, T, L);
  MT3_REQUIRE(bytes >= need, MT3_ERR_WORKSPACE, "%s: workspace has %lld bytes, %lld needed", name, (long long)bytes, (long long)need);
  return MT3_OK;
}

// Whether the pass takes L targets over T inputs: the exact-fp32 attention kernel's limits wherever it runs
static bool tf_supported(const Model* m, int T, int L) {
  const int Lp = tf_pad(L);
  return (tc_attention(m, Lp, Lp, true) || attention_fp32_smem(Lp) <= kAttFp32MaxSmem) &&
         (tc_attention(m, Lp, T, false) || attention_fp32_smem(T) <= kAttFp32MaxSmem);
}

// K-major (hi/lo in TF32X3) copies of the decoder weights the pass multiplies on the wgmma path: made on its first call,
// so that a model that only transcribes keeps its footprint (TF32X3 ~183 MB, TF32 ~92 MB at the mt3 shapes).
static int ensure_tf_weights(Model* m, cudaStream_t s) {
  if (!m->tc || m->slab_tf) return MT3_OK;
  const int D = m->D, Q = m->Q, F = m->F;
  return make_slab(&m->slab_tf, "teacher-forced weight prep", s, [&](Carve& c) -> int {
    for (DecLayer& L : m->dec) {
      MT3_TRY(prep_tc_weight(m, s, L.wqkv, D, 3 * Q, c, &L.t_wqkv));
      MT3_TRY(prep_tc_weight(m, s, L.wo, Q, D, c, &L.t_wo));
      MT3_TRY(prep_tc_weight(m, s, L.wq_c, D, Q, c, &L.t_wq_c));
      MT3_TRY(prep_tc_weight(m, s, L.wo_c, Q, D, c, &L.t_wo_c));
      MT3_TRY(prep_tc_weight(m, s, L.wi, D, 2 * F, c, &L.t_wi));
      MT3_TRY(prep_tc_weight(m, s, L.wo2, F, D, c, &L.t_wo2));
    }
    return prep_tc_weight(m, s, m->w_logits, D, m->V, c, &m->t_w_logits);
  });
}

// Positions t < n of every sequence of the pass's self-attention K/V -> the decode cache: head-major rows [b][K|V][h][cap] at
// positions 0 .. n - 1, in kv_fmt, through kv_dest / kv_store (the row writer of the GEMM epilogues and the decode append).
// K from qkv [B*Lp, 3Q] (columns Q ..); V from qkv's columns 2Q .. or, where the wgmma attention runs, from its V^T
// [B*H*64, Lp] (keys in vt_key_slot() order).  hi + lo is the float32 value the pass attends with (split_tf32 is exact).
__global__ void prefill_kv_kernel(const float* __restrict__ qkv_hi, const float* __restrict__ qkv_lo, const float* __restrict__ vt_hi,
                                  const float* __restrict__ vt_lo, int Lp, int H, int kv_fmt, char* __restrict__ dst, int cap) {
  const int t = blockIdx.x, b = blockIdx.y, Q = H * 64;
  const long long m = (long long)b * Lp + t;
  for (int c = 4 * threadIdx.x; c < 2 * Q; c += 4 * blockDim.x) {
    float v[4];
    if (c < Q || !vt_hi) {
      const long long i = m * 3 * Q + Q + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = qkv_hi[i + j] + (qkv_lo ? qkv_lo[i + j] : 0.f);
    } else {
      const int h = (c - Q) >> 6, d = (c - Q) & 63;
      const long long i = (((long long)b * H + h) * 64 + d) * Lp + vt_key_slot(t);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = vt_hi[i + (long long)j * Lp] + (vt_lo ? vt_lo[i + (long long)j * Lp] : 0.f);
    }
    int d;
    char* row = dst + kv_dest(b, c, 1, cap, H, t, kv_fmt, d);
    kv_store<4>(row, kv_fmt, d, v);
  }
}

// kv_cache: the prefill form (mt3_generate_prompted).  Every layer's self-attention K/V of positions 0 .. L - 1 go to the
// decode cache (kv_layer(m, kv_cache, l, m->L)); nothing after the last layer's QKV projection runs, and logits and scores
// are not computed.
static int teacher_forced_impl(Model* m, const float* encoded, int B, int T, const int* tok_in, const int* tgt, const int* wts, int L,
                               float* logits, float* scores, char* ws, cudaStream_t s, char* kv_cache = nullptr) {
  TfActs w;
  Carve c{ws};
  MT3_TRY(carve_tf(m, c, B, T, L, &w));
  const SeqActs& y = w.seq;
  const int Lp = y.T, D = m->D, Q = m->Q, F = m->F, V = m->V, H = m->H;
  const int M = B * Lp, Me = B * T;
  Act enc;
  MT3_TRY(enc_input(m, encoded, Me, D, w.enc_pair, &enc, s));

  MT3_TRY(launch_embed_seq(tok_in, B, L, Lp, m->emb, D, V, m->pe, y.h.hi, y.h.lo, s));
  for (int l = 0; l < m->Ld; ++l) {
    const DecLayer& dl = m->dec[l];
    // self-attention: RMSNorm folded into the QKV projection's row scale; mask make_decoder_mask(targets)
    MT3_TRY(seq_rstd(m, y, s));
    MT3_TRY(seq_qkv(m, y, dl.wqkv, dl.t_wqkv, s));
    if (kv_cache) {
      prefill_kv_kernel<<<dim3(L, B), 128, 0, s>>>(y.qkv.hi, y.qkv.lo, y.vt.hi, y.vt.lo, Lp, H, m->kv_fmt, kv_layer(m, kv_cache, l, m->L),
                                                   m->L);
      MT3_LAUNCH_CHECK();
      if (l == m->Ld - 1) return MT3_OK;
    }
    MT3_TRY(seq_self_attention(m, y, tgt, L, true, s));
    MT3_TRY(seq_residual(m, y, y.ao, Q, dl.wo, dl.t_wo, s));
    // cross-attention over all T encoder positions; K/V projected from `encoded` for this layer
    MT3_TRY(seq_rstd(m, y, s));
    {
      TcGemmArgs a = gemm_epi(M, Q, D, w.qc.hi, w.qc.lo, Q);
      a.row_scale = y.rstd;
      MT3_TRY(enc_gemm(m, y.h, dl.wq_c, dl.t_wq_c, a, s));
    }
    {
      TcGemmArgs a = gemm_epi(Me, 2 * Q, D, w.ckv.hi, w.ckv.lo, 2 * Q);
      if (w.tcc) { a.VT_hi = w.cvt.hi; a.VT_lo = w.cvt.lo; a.vt_col0 = Q; a.vt_T = T; a.vt_H = H; }
      MT3_TRY(enc_gemm(m, enc, dl.wkv_c, dl.t_wkv_c, a, s));
    }
    if (w.tcc)
      MT3_TRY(launch_attention_tc(w.qc.op, 0, Lp, w.ckv.op, 0, T, w.cvt.op, B, H, y.ao.hi, y.ao.lo, m->split3, true, false, nullptr, 0, s,
                                  y.scratch));
    else MT3_TRY(launch_attention_fp32(w.qc.hi, Q, 0, w.ckv.hi, 2 * Q, 0, Q, Lp, T, H, B, y.ao.hi, y.ao.lo, Q, nullptr, 0, s));
    MT3_TRY(seq_residual(m, y, y.ao, Q, dl.wo_c, dl.t_wo_c, s));
    // gated-GELU MLP
    MT3_TRY(seq_rstd(m, y, s));
    MT3_TRY(seq_mlp_in(m, y, dl.wi, dl.t_wi, s));
    MT3_TRY(seq_residual(m, y, y.g, F, dl.wo2, dl.t_wo2, s));
  }
  // decoder_norm (folded into w_logits) + logits_dense, then the scores, in chunks of rows
  MT3_TRY(seq_rstd(m, y, s));
  float* chunk = w.logits;
  for (int64_t r0 = 0; r0 < M; r0 += kTfLogitRows) {
    const int n = (int)std::min((int64_t)kTfLogitRows, M - r0);
    Act ys;
    MT3_TRY(make_act(m, y.h.hi + r0 * D, y.h.lo ? y.h.lo + r0 * D : nullptr, n, D, &ys));
    TcGemmArgs a = gemm_epi(n, V, D, chunk, nullptr, V);
    a.row_scale = y.rstd + r0;
    MT3_TRY(enc_gemm(m, ys, m->w_logits, m->t_w_logits, a, s));
    MT3_TRY(launch_token_score(chunk, V, (int)r0, n, Lp, L, tgt, wts, scores, logits, s));
  }
  return MT3_OK;
}

}  // namespace mt3

using namespace mt3;

extern "C" int64_t mt3_model_num_params(const mt3_model_config* cfg) {
  if (!cfg) return -1;
  auto t = param_table(*cfg);
  return t.back().offset + t.back().rows * t.back().cols;
}

extern "C" int64_t mt3_model_param_offset(const mt3_model_config* cfg, const char* name, int64_t* numel) {
  if (!cfg || !name) return -1;
  for (const auto& e : param_table(*cfg))
    if (e.name == name) {
      if (numel) *numel = e.rows * e.cols;
      return e.offset;
    }
  return -1;
}

// The prepared weights: each buffer carved from c (float counts, no padding) and, unless c only measures, filled from the
// reference's tensors in `weights` (fused, scale-folded and precomposed as DESIGN.md §2 lists)
static int prep_weights(Model* m, const float* weights, Carve& c, cudaStream_t s) {
  const mt3_model_config* cfg = &m->cfg;
  const int D = m->D, Q = m->Q, F = m->F, V = m->V;
  const auto t = param_table(*cfg);
  auto W = [&](const std::string& n) -> const float* {
    for (const auto& en : t) if (en.name == n) return weights + en.offset;
    return nullptr;
  };
  int rc = MT3_OK;
#define PREP(...) do { if (rc == MT3_OK && c.base) rc = prep_copy(s, __VA_ARGS__); } while (0)
  m->w_in = c.take((int64_t)cfg->input_depth * D);
  PREP(W("encoder/continuous_inputs_projection/kernel"), cfg->input_depth, D, nullptr, m->w_in, D, 0, 1);
  m->enc.resize(m->Le);
  for (int i = 0; i < m->Le; ++i) {
    const std::string pre = "encoder/layers_" + std::to_string(i) + "/";
    EncLayer& L = m->enc[i];
    const float* g1 = W(pre + "pre_attention_layer_norm/scale");
    const float* g2 = W(pre + "pre_mlp_layer_norm/scale");
    L.wqkv = c.take((int64_t)D * 3 * Q);
    PREP(W(pre + "attention/query/kernel"), D, Q, g1, L.wqkv, 3 * Q, 0, 1);
    PREP(W(pre + "attention/key/kernel"), D, Q, g1, L.wqkv, 3 * Q, Q, 1);
    PREP(W(pre + "attention/value/kernel"), D, Q, g1, L.wqkv, 3 * Q, 2 * Q, 1);
    L.wo = c.take((int64_t)Q * D);
    PREP(W(pre + "attention/out/kernel"), Q, D, nullptr, L.wo, D, 0, 1);
    L.wi = c.take((int64_t)D * 2 * F);
    PREP(W(pre + "mlp/wi_0/kernel"), D, F, g2, L.wi, 2 * F, 0, 2);
    PREP(W(pre + "mlp/wi_1/kernel"), D, F, g2, L.wi, 2 * F, 1, 2);
    L.wo2 = c.take((int64_t)F * D);
    PREP(W(pre + "mlp/wo/kernel"), F, D, nullptr, L.wo2, D, 0, 1);
  }
  m->enc_norm_g = c.take(D);
  PREP(W("encoder/encoder_norm/scale"), 1, D, nullptr, m->enc_norm_g, D, 0, 1);
  m->emb = c.take((int64_t)V * D);
  PREP(W("decoder/token_embedder/embedding"), V, D, nullptr, m->emb, D, 0, 1);
  m->dec.resize(m->Ld);
  for (int i = 0; i < m->Ld; ++i) {
    const std::string pre = "decoder/layers_" + std::to_string(i) + "/";
    DecLayer& L = m->dec[i];
    const float* g1 = W(pre + "pre_self_attention_layer_norm/scale");
    const float* g2 = W(pre + "pre_cross_attention_layer_norm/scale");
    const float* g3 = W(pre + "pre_mlp_layer_norm/scale");
    L.wqkv = c.take((int64_t)D * 3 * Q);
    PREP(W(pre + "self_attention/query/kernel"), D, Q, g1, L.wqkv, 3 * Q, 0, 1);
    PREP(W(pre + "self_attention/key/kernel"), D, Q, g1, L.wqkv, 3 * Q, Q, 1);
    PREP(W(pre + "self_attention/value/kernel"), D, Q, g1, L.wqkv, 3 * Q, 2 * Q, 1);
    L.wo = c.take((int64_t)Q * D);
    PREP(W(pre + "self_attention/out/kernel"), Q, D, nullptr, L.wo, D, 0, 1);
    L.wq_c = c.take((int64_t)D * Q);
    PREP(W(pre + "encoder_decoder_attention/query/kernel"), D, Q, g2, L.wq_c, Q, 0, 1);
    L.wc1 = c.take((int64_t)(Q + D) * Q);
    if (rc == MT3_OK && c.base) {
      compose_out_q_kernel<<<dim3(cdiv(Q, 128), Q + D), 128, 0, s>>>(L.wo, L.wq_c, Q, D, L.wc1);
      if (cudaGetLastError() != cudaSuccess) rc = fail(MT3_ERR_CUDA, "mt3_model_create: compose_out_q launch failed");
    }
    L.wkv_c = c.take((int64_t)D * 2 * Q);   // applied to `encoded`, which is already normed: no fold
    PREP(W(pre + "encoder_decoder_attention/key/kernel"), D, Q, nullptr, L.wkv_c, 2 * Q, 0, 1);
    PREP(W(pre + "encoder_decoder_attention/value/kernel"), D, Q, nullptr, L.wkv_c, 2 * Q, Q, 1);
    L.wo_c = c.take((int64_t)Q * D);
    PREP(W(pre + "encoder_decoder_attention/out/kernel"), Q, D, nullptr, L.wo_c, D, 0, 1);
    L.wi = c.take((int64_t)D * 2 * F);
    PREP(W(pre + "mlp/wi_0/kernel"), D, F, g3, L.wi, 2 * F, 0, 2);
    PREP(W(pre + "mlp/wi_1/kernel"), D, F, g3, L.wi, 2 * F, 1, 2);
    L.wo2 = c.take((int64_t)F * D);
    PREP(W(pre + "mlp/wo/kernel"), F, D, nullptr, L.wo2, D, 0, 1);
  }
  m->w_logits = c.take((int64_t)D * V);
  PREP(W("decoder/logits_dense/kernel"), D, V, W("decoder/decoder_norm/scale"), m->w_logits, V, 0, 1);
#undef PREP
  m->pe = c.take((int64_t)kPeRows * D);
  return rc;
}

extern "C" int mt3_model_create(const mt3_model_config* cfg, const float* weights, mt3_model** out, void* stream) {
  MT3_REQUIRE(cfg && weights && out, MT3_ERR_BAD_ARG, "mt3_model_create: null argument");
  MT3_REQUIRE(cfg->head_dim == kHD, MT3_ERR_UNSUPPORTED, "mt3_model_create: head_dim %d (kernels are built for 64)", cfg->head_dim);
  MT3_REQUIRE(cfg->emb_dim % 64 == 0 && cfg->mlp_dim % 64 == 0 && cfg->input_depth % 16 == 0 && cfg->vocab_size % 4 == 0,
              MT3_ERR_UNSUPPORTED, "mt3_model_create: emb/mlp dims must be multiples of 64, input depth of 16, vocab of 4");
  MT3_REQUIRE(cfg->num_heads > 0 && cfg->num_encoder_layers >= 0 && cfg->num_decoder_layers > 0 && cfg->max_batch > 0 &&
                  cfg->max_input_length > 0 && cfg->max_decode_length > 0,
              MT3_ERR_BAD_ARG, "mt3_model_create: non-positive size");
  MT3_REQUIRE(cfg->max_decode_length <= kPeRows && cfg->max_input_length <= kPeRows, MT3_ERR_UNSUPPORTED,
              "mt3_model_create: lengths above FixedEmbed.max_length=2048 (layers.py:565)");
  MT3_REQUIRE(cfg->gemm_mode == MT3_GEMM_FP32_SIMT || cfg->gemm_mode == MT3_GEMM_TF32X3 || cfg->gemm_mode == MT3_GEMM_TF32,
              MT3_ERR_BAD_ARG, "mt3_model_create: unknown gemm_mode %d", cfg->gemm_mode);
  MT3_REQUIRE(cfg->kv_cache_format == MT3_KV_F32 || cfg->kv_cache_format == MT3_KV_F16 || cfg->kv_cache_format == MT3_KV_P24, MT3_ERR_BAD_ARG,
              "mt3_model_create: unknown kv_cache_format %d", cfg->kv_cache_format);
  if (cfg->gemm_mode != MT3_GEMM_FP32_SIMT)
    MT3_REQUIRE(cfg->emb_dim % 32 == 0 && cfg->mlp_dim % 32 == 0 && cfg->input_depth % 32 == 0, MT3_ERR_UNSUPPORTED,
                "mt3_model_create: the wgmma path needs emb/mlp/input dims that are multiples of 32");
  cudaStream_t s = (cudaStream_t)stream;
  Model* m = new Model();
  m->cfg = *cfg;
  m->D = cfg->emb_dim; m->H = cfg->num_heads; m->Q = cfg->num_heads * cfg->head_dim; m->F = cfg->mlp_dim;
  m->V = cfg->vocab_size; m->Le = cfg->num_encoder_layers; m->Ld = cfg->num_decoder_layers; m->L = cfg->max_decode_length;
  const int D = m->D, Q = m->Q, F = m->F, V = m->V;
  int rc = make_slab(&m->slab, "mt3_model_create: prepared weights", s,
                     [&](Carve& c) { return prep_weights(m, weights, c, s); });
  if (rc == MT3_OK) {
    // layers.py:51-82 (float64 on the host, rounded to float32 like the reference's numpy code)
    std::vector<float> pe((size_t)kPeRows * D, 0.f);
    const int half = D / 2;
    const double scale_factor = -log(10000.0 / 1.0) / (double)(half - 1);
    for (int pos = 0; pos < kPeRows; ++pos)
      for (int i = 0; i < half; ++i) {
        const double div = 1.0 * exp((double)i * scale_factor);
        pe[(size_t)pos * D + i] = (float)sin((double)pos * div);
        pe[(size_t)pos * D + half + i] = (float)cos((double)pos * div);
      }
    cudaError_t e = cudaMemcpyAsync(m->pe, pe.data(), pe.size() * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(MT3_ERR_CUDA, "mt3_model_create: PE upload -> %s", cudaGetErrorString(e));
  }
  {
    const char* e_pdl = getenv("MT3_PDL");
    m->pdl_attn = !(e_pdl && e_pdl[0] == '0');
    const char* e_attn = getenv("MT3_TC_ATTENTION");
    m->tc_attn_ok = !(e_attn && e_attn[0] == '0');
    const char* e_pfa = getenv("MT3_PF_ATTN");
    if (e_pfa) m->pf_attn = std::max(0, atoi(e_pfa));
    const char* e_pfk = getenv("MT3_PF_KV");
    if (e_pfk) m->pf_kv = std::max(0, atoi(e_pfk));
    const char* e_pg = getenv("MT3_PDL_GEMM");
    m->pdl_gemm = !(e_pg && e_pg[0] == '0');
  }
  m->kv_fmt = cfg->kv_cache_format;
  m->kv_row = kv_row_bytes(m->kv_fmt);
  m->tc = cfg->gemm_mode != MT3_GEMM_FP32_SIMT;
  m->split3 = cfg->gemm_mode == MT3_GEMM_TF32X3;
  if (rc == MT3_OK && m->tc)
    rc = make_slab(&m->slab_tc, "mt3_model_create: tc weight prep", s, [&](Carve& c) -> int {
      MT3_TRY(prep_tc_weight(m, s, m->w_in, cfg->input_depth, D, c, &m->t_w_in));
      for (EncLayer& L : m->enc) {
        MT3_TRY(prep_tc_weight(m, s, L.wqkv, D, 3 * Q, c, &L.t_wqkv));
        MT3_TRY(prep_tc_weight(m, s, L.wo, Q, D, c, &L.t_wo));
        MT3_TRY(prep_tc_weight(m, s, L.wi, D, 2 * F, c, &L.t_wi));
        MT3_TRY(prep_tc_weight(m, s, L.wo2, F, D, c, &L.t_wo2));
      }
      for (DecLayer& L : m->dec) MT3_TRY(prep_tc_weight(m, s, L.wkv_c, D, 2 * Q, c, &L.t_wkv_c));
      return MT3_OK;
    });
  if (rc == MT3_OK) {
    const cudaError_t e = cudaMallocHost((void**)&m->h_flag, 4 * sizeof(int));
    if (e != cudaSuccess) rc = fail(MT3_ERR_CUDA, "mt3_model_create: cudaMallocHost -> %s", cudaGetErrorString(e));
  }
  if (rc != MT3_OK) {
    cudaFree(m->slab);
    cudaFree(m->slab_tc);
    delete m;
    return rc;
  }
  *out = reinterpret_cast<mt3_model*>(m);
  return MT3_OK;
}

extern "C" int mt3_model_destroy(mt3_model* h) {
  if (!h) return MT3_OK;
  Model* m = reinterpret_cast<Model*>(h);
  drop_graphs(m);
  if (m->cap_stream) cudaStreamDestroy(m->cap_stream);
  if (m->h_flag) cudaFreeHost(m->h_flag);
  cudaFree(m->slab);
  cudaFree(m->slab_tc);
  cudaFree(m->slab_tf);
  delete m;
  return MT3_OK;
}

// The model workspace for B sequences of T inputs
static int carve_workspace(const Model* m, Carve& c, int B, int T, WsBuffers* w) {
  const int64_t M = (int64_t)B * T, D = m->D, Q = m->Q, F = m->F, L = m->L;
  MT3_TRY(carve_seq(m, c, B, T, false, 0, &w->ea));
  if (m->split3) {
    MT3_TRY(carve_act(m, c, M, m->cfg.input_depth, true, &w->a_x));
    MT3_TRY(carve_act(m, c, M, m->D, true, &w->a_enc));
  }
  w->encoded = c.take(M * D);
  w->ckv = c.take<char>((int64_t)m->Ld * M * 2 * m->H * m->kv_row);
  w->skv = c.take<char>((int64_t)m->Ld * B * L * 2 * m->H * m->kv_row);
  w->dy = c.take(B * D);
  w->dy2 = c.take(B * D);
  w->dssq = c.take(B * (D / 32));
  w->dq = c.take(B * Q);
  w->dao = c.take(B * Q);
  w->dg = c.take(B * F);
  w->dlogits = c.take((int64_t)B * m->V);
  w->tok_cur = c.take<int>(B);
  w->finished = c.take<int>(B);
  w->tokens = c.take<int>(B * L);
  w->state = c.take<int>(16);
  w->dpartial = c.take((int64_t)16 * dec_tiles(m) * kDecTileFloats);   // up to 16 K chunks
  w->dcounters = c.take<int>(dec_tiles(m));
  w->beam_f = c.take(3 * B);      // {live_lp, finished score} per sequence, then fin_lp_eos [B]
  w->fin_lp_eos = w->beam_f ? w->beam_f + 2 * B : nullptr;
  w->beam_i = c.take<int>(B);
  w->tok_scores = c.take(B * L);
  w->seq_scores = c.take(B);
  w->plen = c.take<int>(B);
  w->prompt_info = c.take<int>(2);
  w->pf_tok = c.take<int>(2 * B * L);
  w->sample = c.take<mt3_sample_params>(1);
  w->bias = c.take((int64_t)B * m->V);
  return MT3_OK;
}

extern "C" int64_t mt3_workspace_bytes(const mt3_model* h, int32_t batch, int32_t input_length) {
  if (!h || batch <= 0 || input_length <= 0) return -1;
  Carve c;
  WsBuffers w;
  carve_workspace(reinterpret_cast<const Model*>(h), c, batch, input_length, &w);
  return c.used;
}

extern "C" int mt3_model_set_workspace(mt3_model* h, void* workspace, int64_t bytes, int32_t batch, int32_t input_length) {
  MT3_REQUIRE(h && workspace, MT3_ERR_BAD_ARG, "mt3_model_set_workspace: null argument");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_REQUIRE(batch > 0 && batch <= m->cfg.max_batch, MT3_ERR_SHAPE, "batch %d outside (0, max_batch=%d]", batch, m->cfg.max_batch);
  MT3_REQUIRE(input_length > 0 && input_length <= m->cfg.max_input_length, MT3_ERR_SHAPE,
              "input_length %d outside (0, max_input_length=%d]", input_length, m->cfg.max_input_length);
  MT3_REQUIRE(((uintptr_t)workspace & 255) == 0, MT3_ERR_WORKSPACE, "workspace must be 256-byte aligned");
  Carve c{(char*)workspace};
  WsBuffers w;
  MT3_TRY(carve_workspace(m, c, batch, input_length, &w));
  MT3_REQUIRE(bytes >= c.used, MT3_ERR_WORKSPACE, "workspace has %lld bytes, %lld needed", (long long)bytes, (long long)c.used);
  static_cast<WsBuffers&>(*m) = w;
  m->ws = (char*)workspace; m->B = batch; m->T = input_length;
  m->have_cross = false;
  select_graph(m);
  return MT3_OK;
}

#define MT3_NEED_WS(m) MT3_REQUIRE((m)->ws, MT3_ERR_STATE, "no workspace set (call mt3_model_set_workspace first)")

extern "C" int mt3_encode(mt3_model* h, const float* x, float* encoded, void* stream) {
  MT3_REQUIRE(h && x && encoded, MT3_ERR_BAD_ARG, "mt3_encode: null argument");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  return encode_impl(m, x, encoded, (cudaStream_t)stream);
}

extern "C" int mt3_cross_kv(mt3_model* h, const float* encoded, void* stream) {
  MT3_REQUIRE(h && encoded, MT3_ERR_BAD_ARG, "mt3_cross_kv: null argument");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  return cross_kv_impl(m, encoded, (cudaStream_t)stream);
}

extern "C" int mt3_decode_step(mt3_model* h, const int32_t* tok_in, float* logits, int32_t* tok_out, void* stream) {
  MT3_REQUIRE(h && tok_in, MT3_ERR_BAD_ARG, "mt3_decode_step: null argument");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  MT3_REQUIRE(m->have_cross, MT3_ERR_STATE, "mt3_decode_step before mt3_cross_kv");
  MT3_REQUIRE(m->host_pos < m->L, MT3_ERR_STATE, "mt3_decode_step: cache full (%d steps = max_decode_length)", m->L);
  m->host_pos += 1;
  return decode_step_impl(m, tok_in, logits ? logits : m->dlogits, tok_out != nullptr, tok_out, 0, nullptr,
                          (cudaStream_t)stream);
}

// Prompt rows [B, prompt_len] (mt3_generate_prompted), one warp per row: p_b = the length of the non-zero prefix,
// which must hold ids in [2, V), with only 0 after it.  Writes plen[b] = p_b and the row into tokens[b, 0 .. prompt_len);
// info = {min p_b, 1 + the first invalid row (0 when every row is valid)}.
__global__ void __launch_bounds__(256) prompt_scan_kernel(const int* __restrict__ prompt, int B, int prompt_len, int V,
                                                          int* __restrict__ plen, int* __restrict__ tokens, int ld_tokens,
                                                          int* __restrict__ info) {
  __shared__ int s_min, s_bad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_min = prompt_len; s_bad = B; }
  __syncthreads();
  for (int b = warp; b < B; b += 8) {
    const int* row = prompt + (long long)b * prompt_len;
    int p = prompt_len;
    for (int j0 = 0; j0 < prompt_len; j0 += 32) {
      const int j = j0 + lane;
      const unsigned z = __ballot_sync(0xffffffffu, j < prompt_len && row[j] == 0);
      if (z) { p = j0 + __ffs(z) - 1; break; }
    }
    bool bad = false;
    for (int j = lane; j < prompt_len; j += 32) {
      const int v = row[j];
      bad |= j < p ? (v < 2 || v >= V) : v != 0;
      tokens[(long long)b * ld_tokens + j] = v;
    }
    if (lane == 0) plen[b] = p;
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicMin(&s_bad, b);
    if (lane == 0) atomicMin(&s_min, p);
  }
  __syncthreads();
  if (threadIdx.x == 0) { info[0] = s_min; info[1] = s_bad < B ? s_bad + 1 : 0; }
}

// Logit bias rows (mt3_generate_biased), one warp per row: dst[b, :] = bias[b * ld, ...] ([B, V]; ld = 0 repeats one row).
// A row is valid when every entry is finite or -inf and at least one is finite.  info[1] holds 0 or prompt_scan_kernel's
// code on entry; a 0 becomes -(1 + the first invalid row), so one 8-byte copy reports both checks.
__global__ void __launch_bounds__(1024) bias_load_kernel(const float* __restrict__ bias, long long ld, int B, int V,
                                                         float* __restrict__ dst, int* __restrict__ info) {
  __shared__ int s_bad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_bad = B;
  __syncthreads();
  for (int b = warp; b < B; b += 32) {
    const float* row = bias + b * ld;
    bool bad = false, finite = false;
    for (int j = lane; j < V; j += 32) {
      const float v = row[j];
      bad |= !(v < INFINITY);             // NaN or +inf
      finite |= v > -INFINITY && v < INFINITY;
      dst[(long long)b * V + j] = v;
    }
    const bool row_bad = __any_sync(0xffffffffu, bad) || !__any_sync(0xffffffffu, finite);
    if (row_bad && lane == 0) atomicMin(&s_bad, b);
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_bad < B && info[1] == 0) info[1] = -(s_bad + 1);
}

// The prefill pass's inputs over the shared prefix of P positions: decoder inputs BOS, prompt[:, 0 .. P-2] and targets
// prompt[:, 0 .. P-1] (all non-zero: every key < P is valid), both [B, P]; and the loop's state after it: position P, next
// decoder input prompt[:, P-1].
__global__ void prefill_inputs_kernel(const int* __restrict__ prompt, int prompt_len, int P, int* __restrict__ dec_in,
                                      int* __restrict__ tgt, int* __restrict__ tok_cur, int* __restrict__ state) {
  const int b = blockIdx.x;
  const int* row = prompt + (long long)b * prompt_len;
  for (int j = threadIdx.x; j < P; j += blockDim.x) {
    dec_in[(long long)b * P + j] = j ? row[j - 1] : 0;
    tgt[(long long)b * P + j] = row[j];
  }
  if (threadIdx.x == 0) {
    tok_cur[b] = row[P - 1];
    if (b == 0) state[0] = P;
  }
}

// Shortest shared prompt prefix worth one teacher-forced pass instead of stepping the loop through it.  Measured at bench's
// configuration (DESIGN.md §6): the pass over P <= 128 positions costs about as much as the loop's first 17 steps.
constexpr int kPrefillMinP = 20;

// Temperatures at or below this pick greedily (T5X's MIN_TEMPERATURE): MT3_GEN_SAMPLE then runs the greedy loop unchanged.
constexpr float kMinTemperature = 1e-4f;

// mt3_generate, mt3_generate_scored, mt3_generate_prompted, mt3_generate_sampled and mt3_generate_biased; `name` is the entry
// point the caller used, for its error messages.  prompt_len == 0: no prompt (prompt and workspace unused).  sp: HOST, read
// with MT3_GEN_SAMPLE only.  bias: DEV or null (no bias), rows bias_ld apart.
static int generate_impl(const char* name, mt3_model* h, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt,
                         int32_t prompt_len, int32_t* tokens_out, float* token_scores_out, float* scores_out, int32_t* steps_run,
                         void* workspace, int64_t workspace_bytes, const mt3_sample_params* sp, void* stream,
                         const float* bias = nullptr, int64_t bias_ld = 0) {
  MT3_REQUIRE(h && x && tokens_out, MT3_ERR_BAD_ARG, "%s: null argument", name);
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  MT3_REQUIRE(num_steps >= 0 && num_steps <= m->L, MT3_ERR_SHAPE, "%s: num_steps %d outside [0, max_decode_length=%d]", name, num_steps,
              m->L);
  MT3_REQUIRE((flags & ~(MT3_GEN_STOP_AT_EOS | MT3_GEN_USE_GRAPH | MT3_GEN_BEAM1 | MT3_GEN_SAMPLE)) == 0, MT3_ERR_BAD_ARG,
              "%s: unknown flag bits 0x%x", name, flags);
  const bool sample = (flags & MT3_GEN_SAMPLE) != 0;
  if (sample) {
    MT3_REQUIRE(!(flags & MT3_GEN_BEAM1), MT3_ERR_BAD_ARG, "%s: MT3_GEN_SAMPLE and MT3_GEN_BEAM1 exclude each other", name);
    MT3_REQUIRE(sp, MT3_ERR_BAD_ARG, "%s: MT3_GEN_SAMPLE without sampling parameters", name);
    MT3_REQUIRE(isfinite(sp->temperature) && sp->temperature >= 0.f, MT3_ERR_BAD_ARG, "%s: temperature %g is not finite and >= 0", name,
                (double)sp->temperature);
    MT3_REQUIRE(sp->topk >= 0, MT3_ERR_BAD_ARG, "%s: topk %d < 0", name, sp->topk);
    MT3_REQUIRE(sp->topp >= 0.f && sp->topp <= 1.f, MT3_ERR_BAD_ARG, "%s: topp %g outside [0, 1]", name, (double)sp->topp);
  }
  const bool filtered = sample && ((sp->topk > 0 && sp->topk < m->V) || (sp->topp > 0.f && sp->topp < 1.f));
  MT3_REQUIRE(!filtered || m->V <= kSampleMaxSortV, MT3_ERR_UNSUPPORTED, "%s: top-k / top-p need vocab_size <= %d (have %d)", name,
              kSampleMaxSortV, m->V);
  MT3_REQUIRE(prompt_len >= 0 && prompt_len <= num_steps, MT3_ERR_BAD_ARG, "%s: prompt_len %d outside [0, num_steps=%d]", name, prompt_len,
              num_steps);
  MT3_REQUIRE(prompt_len == 0 || prompt, MT3_ERR_BAD_ARG, "%s: prompt is NULL with prompt_len %d", name, prompt_len);
  if (prompt_len > 0) MT3_TRY(check_tf_workspace(m, name, workspace, workspace_bytes, m->B, m->T, prompt_len));
  const bool biased = bias != nullptr;
  MT3_REQUIRE(!biased || bias_ld == 0 || bias_ld >= m->V, MT3_ERR_BAD_ARG, "%s: bias_ld %lld is neither 0 nor >= vocab_size %d", name,
              (long long)bias_ld, m->V);
  cudaStream_t s = (cudaStream_t)stream;
  MT3_CUDA_CHECK(cudaMemsetAsync(m->tokens, 0, (size_t)m->B * m->L * sizeof(int), s));
  MT3_CUDA_CHECK(cudaMemsetAsync(m->plen, 0, (size_t)m->B * sizeof(int), s));
  if (sample && sp->temperature > kMinTemperature) {
    // one graph per (mode, scored, steps) serves every parameter set: the picker reads them from the workspace
    MT3_CUDA_CHECK(cudaMemcpyAsync(m->sample, sp, sizeof(mt3_sample_params), cudaMemcpyHostToDevice, s));
    MT3_CUDA_CHECK(cudaStreamSynchronize(s));        // `sp` is the caller's pageable memory
  }
  int P = 0;                                    // prompt prefix every row shares
  if (prompt_len > 0 || biased) {
    if (prompt_len > 0) {
      prompt_scan_kernel<<<1, 256, 0, s>>>(prompt, m->B, prompt_len, m->V, m->plen, m->tokens, m->L, m->prompt_info);
      MT3_LAUNCH_CHECK();
    } else {
      MT3_CUDA_CHECK(cudaMemsetAsync(m->prompt_info, 0, 2 * sizeof(int), s));
    }
    if (biased) {     // the picker reads the bias from the workspace, so one graph per (mode, scored, steps) serves every bias
      bias_load_kernel<<<1, 1024, 0, s>>>(bias, (long long)bias_ld, m->B, m->V, m->bias, m->prompt_info);
      MT3_LAUNCH_CHECK();
    }
    MT3_CUDA_CHECK(cudaMemcpyAsync(m->h_flag + 2, m->prompt_info, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
    MT3_CUDA_CHECK(cudaStreamSynchronize(s));
    if (m->h_flag[3]) {
      MT3_CUDA_CHECK(cudaMemsetAsync(m->plen, 0, (size_t)m->B * sizeof(int), s));
      if (m->h_flag[3] < 0)
        return fail(MT3_ERR_BAD_ARG, "%s: logit_bias row %d holds a NaN or +inf, or no finite entry", name, -m->h_flag[3] - 1);
      return fail(MT3_ERR_BAD_ARG, "%s: prompt row %d is not a prefix of ids in [2, %d) followed by zeros", name, m->h_flag[3] - 1, m->V);
    }
    P = m->h_flag[2];
  }
  MT3_TRY(encode_impl(m, x, m->encoded, s));
  MT3_TRY(cross_kv_impl(m, m->encoded, s));
  const bool scored = token_scores_out || scores_out;
  if (scored) MT3_CUDA_CHECK(cudaMemsetAsync(m->tok_scores, 0, (size_t)m->B * m->L * sizeof(float), s));
  const bool use_graph = (flags & MT3_GEN_USE_GRAPH) != 0;
  const bool stop = (flags & MT3_GEN_STOP_AT_EOS) != 0;
  const int mode = (flags & MT3_GEN_BEAM1) ? 2 : (sample && sp->temperature > kMinTemperature) ? 3 : 1;
  if (mode == 2) {      // live log-probability 0, finished score NEG_INF (t5x decoding.NEG_INF = -1e7), no finished hypothesis
    std::vector<float> init((size_t)2 * m->B);
    for (int i = 0; i < m->B; ++i) { init[2 * i] = 0.f; init[2 * i + 1] = -1.0e7f; }
    MT3_CUDA_CHECK(cudaMemcpyAsync(m->beam_f, init.data(), init.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    MT3_CUDA_CHECK(cudaStreamSynchronize(s));        // `init` is stack-owned pageable memory
    MT3_CUDA_CHECK(cudaMemsetAsync(m->beam_i, 0, (size_t)m->B * sizeof(int), s));
  }
  // the shared prefix: one teacher-forced pass writes its K/V rows into the cache, and the loop starts at position P.
  // The tokens there are forced (plen), so they score 0 and finish nothing, as the loop's forced steps do.
  int start = 0;
  if (P >= kPrefillMinP && tf_supported(m, m->T, P)) {
    MT3_TRY(check_tf_workspace(m, name, workspace, workspace_bytes, m->B, m->T, P));
    MT3_TRY(ensure_tf_weights(m, s));
    int* dec_in = m->pf_tok;
    int* tgt = m->pf_tok + (int64_t)m->B * P;
    prefill_inputs_kernel<<<m->B, 128, 0, s>>>(prompt, prompt_len, P, dec_in, tgt, m->tok_cur, m->state);
    MT3_LAUNCH_CHECK();
    MT3_TRY(teacher_forced_impl(m, m->encoded, m->B, m->T, dec_in, tgt, nullptr, P, nullptr, nullptr, (char*)workspace, s, m->skv));
    start = P;
    m->host_pos = P;
  }
  constexpr int kBlock = 16;                    // steps per graph launch (and between two polls of the all-finished flag)
  cudaGraphExec_t g1 = nullptr, gN = nullptr;
  uint64_t k1 = 0, kN = 0;
  if (use_graph) {
    if (num_steps - start >= kBlock) {
      MT3_TRY(ensure_graph(m, mode, kBlock, scored, biased));
      gN = m->graph_exec; kN = m->graph_kernels;
    }
    if ((num_steps - start) % kBlock != 0) {
      MT3_TRY(ensure_graph(m, mode, 1, scored, biased));
      g1 = m->graph_exec; k1 = m->graph_kernels;
    }
  }
  if (num_steps > start)   // decoder input of the first step: BOS (tok_cur was zeroed by cross_kv) at position 0, or the prompt's
    MT3_TRY(dec_embed(m, m->tok_cur, s));      // token P - 1 at position P; later ones come from the token picker
  int ran = start;
  for (int step = start; step < num_steps;) {
    int n = 1;
    if (use_graph && gN && num_steps - step >= kBlock) {
      MT3_CUDA_CHECK(cudaGraphLaunch(gN, s));
      count_launch(kN);
      n = kBlock;
    } else if (use_graph) {
      MT3_CUDA_CHECK(cudaGraphLaunch(g1, s));
      count_launch(k1);
    } else {
      MT3_TRY(decode_step_impl(m, m->tok_cur, m->dlogits, mode, nullptr, 1, m->tokens, s, true, scored, biased));
    }
    step += n;
    ran += n;
    m->host_pos += n;
    if (stop && (((step - start) & 15) == 0 || step == num_steps)) {
      MT3_CUDA_CHECK(cudaMemcpyAsync(m->h_flag, m->state + 2, sizeof(int), cudaMemcpyDeviceToHost, s));
      MT3_CUDA_CHECK(cudaStreamSynchronize(s));
      if (m->h_flag[0]) break;
    }
  }
  if (mode == 2) {
    MT3_TRY(launch_beam1_finalize(m->tokens, m->B, m->L, ran, m->beam_i, scored ? m->tok_scores : nullptr, m->beam_f, m->fin_lp_eos,
                                  scored ? m->seq_scores : nullptr, s));
  } else if (scored) {
    MT3_TRY(launch_seq_score(m->tok_scores, m->B, m->L, m->seq_scores, s));
  }
  MT3_CUDA_CHECK(cudaMemcpyAsync(tokens_out, m->tokens, (size_t)m->B * m->L * sizeof(int), cudaMemcpyDeviceToDevice, s));
  if (token_scores_out)
    MT3_CUDA_CHECK(cudaMemcpyAsync(token_scores_out, m->tok_scores, (size_t)m->B * m->L * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (scores_out) MT3_CUDA_CHECK(cudaMemcpyAsync(scores_out, m->seq_scores, (size_t)m->B * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (steps_run) *steps_run = ran;
  return MT3_OK;
}

extern "C" int mt3_generate(mt3_model* h, const float* x, int32_t num_steps, int32_t flags, int32_t* tokens_out,
                            int32_t* steps_run, void* stream) {
  return generate_impl("mt3_generate", h, x, num_steps, flags, nullptr, 0, tokens_out, nullptr, nullptr, steps_run, nullptr, 0, nullptr,
                       stream);
}

extern "C" int mt3_generate_scored(mt3_model* h, const float* x, int32_t num_steps, int32_t flags, int32_t* tokens_out,
                                   float* token_scores_out, float* scores_out, int32_t* steps_run, void* stream) {
  return generate_impl("mt3_generate_scored", h, x, num_steps, flags, nullptr, 0, tokens_out, token_scores_out, scores_out, steps_run,
                       nullptr, 0, nullptr, stream);
}

extern "C" int mt3_generate_prompted(mt3_model* h, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt,
                                     int32_t prompt_len, int32_t* tokens_out, float* token_scores_out, float* scores_out,
                                     int32_t* steps_run, void* workspace, int64_t workspace_bytes, void* stream) {
  return generate_impl("mt3_generate_prompted", h, x, num_steps, flags, prompt, prompt_len, tokens_out, token_scores_out, scores_out,
                       steps_run, workspace, workspace_bytes, nullptr, stream);
}

extern "C" int mt3_generate_sampled(mt3_model* h, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt,
                                    int32_t prompt_len, int32_t* tokens_out, float* token_scores_out, float* scores_out,
                                    int32_t* steps_run, void* workspace, int64_t workspace_bytes, const mt3_sample_params* params,
                                    void* stream) {
  return generate_impl("mt3_generate_sampled", h, x, num_steps, flags, prompt, prompt_len, tokens_out, token_scores_out, scores_out,
                       steps_run, workspace, workspace_bytes, params, stream);
}

extern "C" int mt3_generate_biased(mt3_model* h, const float* x, int32_t num_steps, int32_t flags, const int32_t* prompt,
                                   int32_t prompt_len, int32_t* tokens_out, float* token_scores_out, float* scores_out,
                                   int32_t* steps_run, void* workspace, int64_t workspace_bytes, const mt3_sample_params* params,
                                   const float* logit_bias, int64_t bias_ld, void* stream) {
  return generate_impl("mt3_generate_biased", h, x, num_steps, flags, prompt, prompt_len, tokens_out, token_scores_out, scores_out,
                       steps_run, workspace, workspace_bytes, params, stream, logit_bias, bias_ld);
}

extern "C" int64_t mt3_teacher_forced_workspace_bytes(const mt3_model* h, int32_t batch, int32_t input_length, int32_t target_length) {
  if (!h) return -1;
  const Model* m = reinterpret_cast<const Model*>(h);
  if (batch <= 0 || batch > m->cfg.max_batch || input_length <= 0 || input_length > m->cfg.max_input_length || target_length <= 0 ||
      target_length > m->L)
    return -1;
  return tf_workspace_bytes(m, batch, input_length, target_length);
}

extern "C" int mt3_decode_teacher_forced(mt3_model* h, const float* encoded, int32_t batch, int32_t input_length,
                                         const int32_t* decoder_input_tokens, const int32_t* decoder_target_tokens,
                                         const int32_t* loss_weights, int32_t target_length, float* logits, float* token_scores,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
  MT3_REQUIRE(h && encoded && decoder_input_tokens && decoder_target_tokens, MT3_ERR_BAD_ARG, "mt3_decode_teacher_forced: null argument");
  MT3_REQUIRE(logits || token_scores, MT3_ERR_BAD_ARG, "mt3_decode_teacher_forced: logits and token_scores are both NULL");
  MT3_REQUIRE(((uintptr_t)logits & 15) == 0, MT3_ERR_BAD_ARG, "mt3_decode_teacher_forced: logits must be 16-byte aligned");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_REQUIRE(batch > 0 && batch <= m->cfg.max_batch, MT3_ERR_SHAPE, "batch %d outside (0, max_batch=%d]", batch, m->cfg.max_batch);
  MT3_REQUIRE(input_length > 0 && input_length <= m->cfg.max_input_length, MT3_ERR_SHAPE,
              "input_length %d outside (0, max_input_length=%d]", input_length, m->cfg.max_input_length);
  MT3_REQUIRE(target_length > 0 && target_length <= m->L, MT3_ERR_SHAPE, "target_length %d outside (0, max_decode_length=%d]",
              target_length, m->L);
  MT3_TRY(check_tf_workspace(m, "mt3_decode_teacher_forced", workspace, workspace_bytes, batch, input_length, target_length));
  MT3_REQUIRE(tf_supported(m, input_length, target_length), MT3_ERR_UNSUPPORTED,
              "mt3_decode_teacher_forced: target_length %d or input_length %d too long for the exact-fp32 attention kernel", target_length,
              input_length);
  // the wgmma GEMM's N tiling of the logits projection
  MT3_REQUIRE(!m->tc || m->V % 32 == 0, MT3_ERR_UNSUPPORTED, "mt3_decode_teacher_forced: the wgmma logits GEMM needs vocab %% 32 == 0");
  cudaStream_t s = (cudaStream_t)stream;
  MT3_TRY(ensure_tf_weights(m, s));
  return teacher_forced_impl(m, encoded, batch, input_length, decoder_input_tokens, decoder_target_tokens, loss_weights, target_length, logits,
                             token_scores, (char*)workspace, s);
}

extern "C" int mt3_vocab_decode(const int32_t* ids, int32_t batch, int32_t length, int32_t num_regular_tokens, int32_t* out,
                                void* stream) {
  MT3_REQUIRE(ids && out, MT3_ERR_BAD_ARG, "mt3_vocab_decode: null argument");
  MT3_REQUIRE(batch >= 0 && length >= 0 && num_regular_tokens >= 0, MT3_ERR_BAD_ARG, "mt3_vocab_decode: negative size");
  if (batch == 0 || length == 0) return MT3_OK;
  vocab_decode_kernel<<<cdiv(batch, 64), 64, 0, (cudaStream_t)stream>>>(ids, batch, length, num_regular_tokens, out);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

extern "C" int mt3_dot_product_attention_f32(const float* q, const float* k, const float* v, const float* bias, int32_t batch,
                                             int32_t q_len, int32_t kv_len, int32_t num_heads, int32_t head_dim, float* out,
                                             void* stream) {
  MT3_REQUIRE(q && k && v && out, MT3_ERR_BAD_ARG, "mt3_dot_product_attention_f32: null argument");
  MT3_REQUIRE(batch >= 0 && q_len >= 0 && kv_len > 0 && num_heads > 0 && head_dim > 0, MT3_ERR_BAD_ARG,
              "mt3_dot_product_attention_f32: non-positive size");
  MT3_REQUIRE(kv_len <= 8192, MT3_ERR_UNSUPPORTED, "mt3_dot_product_attention_f32: kv_len %d above 8192", kv_len);
  const long long items = (long long)batch * num_heads * q_len;
  if (items == 0) return MT3_OK;
  const size_t smem = (size_t)4 * kv_len * sizeof(float);
  static size_t attr_smem = 48 * 1024;
  if (smem > attr_smem) {
    MT3_CUDA_CHECK(cudaFuncSetAttribute(dot_product_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_smem = smem;
  }
  dot_product_attention_kernel<<<(unsigned)((items + 3) / 4), 128, smem, (cudaStream_t)stream>>>(q, k, v, bias, batch, q_len, kv_len,
                                                                                                 num_heads, head_dim, out);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

__global__ void trace_reset_kernel(unsigned long long* t, int n_slots) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_slots * mt3::kTraceWords) t[i] = (i % mt3::kTraceWords == 0) ? ~0ull : 0ull;
}

extern "C" int mt3_debug_trace_step(mt3_model* h, int32_t pos, uint64_t* out, int32_t max_slots, char* names,
                                    int32_t names_bytes, int32_t* n_slots, void* stream) {
  MT3_REQUIRE(h && out && names && n_slots, MT3_ERR_BAD_ARG, "mt3_debug_trace_step: null argument");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  MT3_REQUIRE(pos >= 2 && pos < m->L, MT3_ERR_BAD_ARG, "mt3_debug_trace_step: pos must be in [2, %d)", m->L);
  cudaStream_t s = (cudaStream_t)stream;
  if (!m->trace) MT3_CUDA_CHECK(cudaMalloc(&m->trace, sizeof(unsigned long long) * kTraceSlots * kTraceWords));
  if (!m->cap_stream) MT3_CUDA_CHECK(cudaStreamCreateWithFlags(&m->cap_stream, cudaStreamNonBlocking));
  // capture one greedy step with a trace slot baked into every GEMM / attention node
  m->trace_names.clear();
  m->tracing = true;
  const uint64_t before = g_launch_count.load();
  MT3_CUDA_CHECK(cudaStreamBeginCapture(m->cap_stream, cudaStreamCaptureModeThreadLocal));
  const int r = decode_step_impl(m, m->tok_cur, m->dlogits, 1, nullptr, 1, m->tokens, m->cap_stream, true);
  cudaGraph_t g = nullptr;
  const cudaError_t e = cudaStreamEndCapture(m->cap_stream, &g);
  m->tracing = false;
  g_launch_count.store(before);
  if (r != MT3_OK || e != cudaSuccess) {
    if (g) cudaGraphDestroy(g);
    return r != MT3_OK ? r : fail(MT3_ERR_CUDA, "mt3_debug_trace_step: capture -> %s", cudaGetErrorString(e));
  }
  cudaGraphExec_t ge = nullptr;
  MT3_CUDA_CHECK(cudaGraphInstantiate(&ge, g, 0));
  const int n = (int)m->trace_names.size();
  const int start_pos = pos - 2;                      // two warm replays, the third one (at `pos`) is read back
  MT3_CUDA_CHECK(cudaMemcpyAsync(m->state, &start_pos, sizeof(int), cudaMemcpyHostToDevice, s));
  MT3_CUDA_CHECK(cudaMemsetAsync(m->finished, 0, sizeof(int) * m->B, s));
  for (int it = 0; it < 3; ++it) {
    trace_reset_kernel<<<cdiv(kTraceSlots * kTraceWords, 256), 256, 0, s>>>(m->trace, kTraceSlots);
    MT3_CUDA_CHECK(cudaGraphLaunch(ge, s));
  }
  MT3_CUDA_CHECK(cudaStreamSynchronize(s));
  const int n_out = std::min(n, (int)max_slots);
  MT3_CUDA_CHECK(cudaMemcpy(out, m->trace, sizeof(unsigned long long) * n_out * kTraceWords, cudaMemcpyDeviceToHost));
  std::string all;
  for (int i = 0; i < n_out; ++i) { all += m->trace_names[i]; all += '\n'; }
  snprintf(names, names_bytes, "%s", all.c_str());
  *n_slots = n_out;
  cudaGraphExecDestroy(ge);
  cudaGraphDestroy(g);
  return MT3_OK;
}

extern "C" int mt3_debug_launch(mt3_model* h, int32_t kind, int32_t pos, int32_t iters, void* stream) {
  MT3_REQUIRE(h, MT3_ERR_BAD_ARG, "mt3_debug_launch: null model");
  Model* m = reinterpret_cast<Model*>(h);
  MT3_NEED_WS(m);
  MT3_REQUIRE(pos >= 0 && pos < m->L && iters > 0, MT3_ERR_BAD_ARG, "mt3_debug_launch: bad pos/iters");
  cudaStream_t s = (cudaStream_t)stream;
  const int D = m->D, Q = m->Q, L = m->L, T = m->T;
  for (int it = 0; it < iters; ++it) {
    const int l = it % m->Ld;
    switch (kind) {
      case MT3_K_DEC_SELF_ATTN: {
        MT3_TRY(dec_attention(m, m->dq, kv_layer(m, m->skv, l, L), L, nullptr, pos + 1, m->dao, s));
        break;
      }
      case MT3_K_DEC_CROSS_ATTN: {
        MT3_TRY(dec_attention(m, m->dq, kv_layer(m, m->ckv, l, T), T, nullptr, T, m->dao, s));
        break;
      }
      case MT3_K_DEC_QKV_GEMM: {
        // scratch output: the encoder qkv buffer (B*T rows >= B).  Not the cache: after a full generate, *state is
        // max_decode_length, and an append there would write past it.
        MT3_TRY(dec_gemm(m, "gemm_qkv", m->dy, D, m->dec[l].wqkv, 3 * Q, D, 1, EPI_STORE, m->ea.qkv.hi, 3 * Q, 3 * Q, nullptr, nullptr, s));
        break;
      }
      case MT3_K_ENC_QKV_GEMM: {
        const EncLayer& w = m->enc[it % std::max(1, m->Le)];
        MT3_TRY(seq_qkv(m, m->ea, w.wqkv, w.t_wqkv, s));
        break;
      }
      case MT3_K_ENC_ATTN: {
        MT3_TRY(seq_self_attention(m, m->ea, nullptr, 0, false, s));
        break;
      }
      default:
        return fail(MT3_ERR_BAD_ARG, "mt3_debug_launch: unknown kind %d", kind);
    }
  }
  return MT3_OK;
}
