// Non-GEMM kernels of the MT3 encoder/decoder blocks (sm_90a): RMSNorm statistics,
// full-sequence attention in fp32 (encoder, teacher-forced decoder), token embedding,
// greedy argmax with EOS bookkeeping, vocabulary decode, weight re-layout.
#pragma once

#include "common.cuh"
#include "philox.cuh"

namespace mt3 {

// ---------------------------------------------------------------------------------
// RMSNorm (layers.py:604-621): rstd[m] = 1/sqrt(mean(x[m,:]^2) + eps).  One warp per row.
// ---------------------------------------------------------------------------------
// x_lo != null: the row is stored as a tf32 hi/lo pair (x = x_hi + x_lo exactly).
__global__ void row_rstd_kernel(const float* __restrict__ x, const float* __restrict__ x_lo, int ld, int M, int D,
                                float eps, float* __restrict__ rstd) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* p = reinterpret_cast<const float4*>(x + (long long)row * ld);
  const float4* pl = x_lo ? reinterpret_cast<const float4*>(x_lo + (long long)row * ld) : nullptr;
  float s = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    float4 v = p[i];
    if (pl) {
      const float4 w = pl[i];
      v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    }
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  s = warp_sum(s);
  if (lane == 0) rstd[row] = 1.0f / sqrtf(s / (float)D + eps);
}

inline int launch_row_rstd(const float* x, const float* x_lo, int ld, int M, int D, float eps, float* rstd, cudaStream_t s) {
  row_rstd_kernel<<<cdiv(M, 8), 256, 0, s>>>(x, x_lo, ld, M, D, eps, rstd);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// y = x * rstd * g  (materialised only where the reference's API returns the normed
// tensor itself: `encoded`, network.py:192).
__global__ void rmsnorm_kernel(const float* __restrict__ x, const float* __restrict__ x_lo, int ldx, int M, int D,
                               float eps, const float* __restrict__ g, float* __restrict__ y, int ldy) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* p = reinterpret_cast<const float4*>(x + (long long)row * ldx);
  const float4* pl = x_lo ? reinterpret_cast<const float4*>(x_lo + (long long)row * ldx) : nullptr;
  auto ld4 = [&](int i) {
    float4 v = p[i];
    if (pl) {
      const float4 w = pl[i];
      v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    }
    return v;
  };
  float s = 0.f;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 v = ld4(i);
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  s = warp_sum(s);
  const float r = 1.0f / sqrtf(s / (float)D + eps);
  float4* q = reinterpret_cast<float4*>(y + (long long)row * ldy);
  const float4* gg = reinterpret_cast<const float4*>(g);
  for (int i = lane; i < D / 4; i += 32) {
    const float4 v = ld4(i);
    const float4 w = __ldg(gg + i);
    q[i] = make_float4(v.x * r * w.x, v.y * r * w.y, v.z * r * w.z, v.w * r * w.w);
  }
}

inline int launch_rmsnorm(const float* x, const float* x_lo, int ldx, int M, int D, float eps, const float* g, float* y, int ldy,
                          cudaStream_t s) {
  rmsnorm_kernel<<<cdiv(M, 8), 256, 0, s>>>(x, x_lo, ldx, M, D, eps, g, y, ldy);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// Full-sequence attention, exact fp32 (layers.py:85-157): softmax(q k^T) v, no 1/sqrt(d)
// scaling (layers.py:230-234); the encoder's mask is all ones (network.py:283-289).
// One CTA = 32 query rows of one (b, h); scores for all Tk keys live in shared memory.
// ---------------------------------------------------------------------------------
constexpr int kHD = 64;   // head_dim the kernels are specialised for (gin/model.gin:54)

// Queries of head h at columns q_col0 + 64 h of q's rows [b Tq, (b + 1) Tq) (row pitch ldq), keys / values at k_col0 /
// v_col0 + 64 h of kv's rows [b Tk, (b + 1) Tk) (row pitch ldkv).  CAUSAL: query i sees key j iff j <= i, j < n_valid and
// key_valid[b * n_valid + j] > 0; key tiles past the CTA's last query are not read, and a row with no visible key writes 0.
template <bool CAUSAL>
__global__ void __launch_bounds__(256)
attention_fp32_kernel(const float* __restrict__ q, int ldq, int q_col0, const float* __restrict__ kv, int ldkv, int k_col0, int v_col0,
                      int Tq, int Tk, int H, float* __restrict__ out, float* __restrict__ out_lo, int ldo,
                      const int* __restrict__ key_valid, int n_valid) {
  extern __shared__ __align__(16) float sm[];
  constexpr int QT = 32, KT = 64;
  const int SP = Tk + 4;
  float* sQ = sm;                 // [QT][64]
  float* sS = sQ + QT * kHD;      // [QT][Tk+4]
  float* sT = sS + QT * SP;       // [64][KT+4]  K tile transposed ([d][k]) / V tile [k][d+4]
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QT;
  const int tid = threadIdx.x;
  const int qoff = q_col0 + h * kHD, koff = k_col0 + h * kHD, voff = v_col0 + h * kHD;
  const float* qbase = q + (long long)b * Tq * ldq;
  const float* base = kv + (long long)b * Tk * ldkv;
  const int kend = CAUSAL ? min(Tk, q0 + QT) : Tk;      // keys any row of this CTA can see lie below kend

  for (int i = tid; i < QT * kHD / 4; i += 256) {
    const int r = i / (kHD / 4), c4 = i % (kHD / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < Tq) v = *reinterpret_cast<const float4*>(qbase + (long long)(q0 + r) * ldq + qoff + c4 * 4);
    *reinterpret_cast<float4*>(sQ + r * kHD + c4 * 4) = v;
  }
  // S = Q K^T : thread -> 2 query rows x 4 keys
  const int tq = tid / 16, tk = tid % 16;     // tq in [0,16): rows tq, tq+16 ; tk: keys tk*4..+3
  for (int k0 = 0; k0 < kend; k0 += KT) {
    __syncthreads();
    for (int i = tid; i < KT * kHD / 4; i += 256) {
      const int r = i / (kHD / 4), c4 = i % (kHD / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + r < kend) v = *reinterpret_cast<const float4*>(base + (long long)(k0 + r) * ldkv + koff + c4 * 4);
      sT[(c4 * 4 + 0) * (KT + 4) + r] = v.x;
      sT[(c4 * 4 + 1) * (KT + 4) + r] = v.y;
      sT[(c4 * 4 + 2) * (KT + 4) + r] = v.z;
      sT[(c4 * 4 + 3) * (KT + 4) + r] = v.w;
    }
    __syncthreads();
    float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int d = 0; d < kHD; ++d) {
      const float q_0 = sQ[tq * kHD + d], q_1 = sQ[(tq + 16) * kHD + d];
      const float4 kv4 = *reinterpret_cast<const float4*>(sT + d * (KT + 4) + tk * 4);
      a0[0] = fmaf(q_0, kv4.x, a0[0]); a0[1] = fmaf(q_0, kv4.y, a0[1]);
      a0[2] = fmaf(q_0, kv4.z, a0[2]); a0[3] = fmaf(q_0, kv4.w, a0[3]);
      a1[0] = fmaf(q_1, kv4.x, a1[0]); a1[1] = fmaf(q_1, kv4.y, a1[1]);
      a1[2] = fmaf(q_1, kv4.z, a1[2]); a1[3] = fmaf(q_1, kv4.w, a1[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tk * 4 + j;
      if (k < kend) {
        if (CAUSAL) {
          const bool ok = k < n_valid && key_valid[(long long)b * n_valid + k] > 0;
          sS[tq * SP + k] = (ok && k <= q0 + tq) ? a0[j] : -INFINITY;
          sS[(tq + 16) * SP + k] = (ok && k <= q0 + tq + 16) ? a1[j] : -INFINITY;
        } else {
          sS[tq * SP + k] = a0[j];
          sS[(tq + 16) * SP + k] = a1[j];
        }
      }
    }
  }
  __syncthreads();
  // softmax over keys: warp w handles rows w*4 .. w*4+3
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int r = warp * 4; r < warp * 4 + 4; ++r) {
      float* row = sS + r * SP;
      float mx = -INFINITY;
      for (int k = lane; k < kend; k += 32) mx = fmaxf(mx, row[k]);
      mx = warp_max(mx);
      if (CAUSAL && mx == -INFINITY) mx = 0.f;         // no visible key: every weight is exp(-inf) = 0
      float sum = 0.f;
      for (int k = lane; k < kend; k += 32) {
        const float e = expf(row[k] - mx);
        row[k] = e;
        sum += e;
      }
      sum = warp_sum(sum);
      const float inv = (CAUSAL && !(sum > 0.f)) ? 0.f : 1.0f / sum;
      for (int k = lane; k < kend; k += 32) row[k] *= inv;
    }
  }
  // O = P V : thread -> 2 query rows x 4 dims
  float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
  const int td = tid % 16;   // dims td*4..+3
  for (int k0 = 0; k0 < kend; k0 += KT) {
    __syncthreads();
    for (int i = tid; i < KT * kHD / 4; i += 256) {
      const int r = i / (kHD / 4), c4 = i % (kHD / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + r < kend) v = *reinterpret_cast<const float4*>(base + (long long)(k0 + r) * ldkv + voff + c4 * 4);
      *reinterpret_cast<float4*>(sT + r * (kHD + 4) + c4 * 4) = v;
    }
    __syncthreads();
    const int kmax = min(KT, kend - k0);
    for (int k = 0; k < kmax; ++k) {
      const float p0 = sS[tq * SP + k0 + k], p1 = sS[(tq + 16) * SP + k0 + k];
      const float4 vv = *reinterpret_cast<const float4*>(sT + k * (kHD + 4) + td * 4);
      o0[0] = fmaf(p0, vv.x, o0[0]); o0[1] = fmaf(p0, vv.y, o0[1]);
      o0[2] = fmaf(p0, vv.z, o0[2]); o0[3] = fmaf(p0, vv.w, o0[3]);
      o1[0] = fmaf(p1, vv.x, o1[0]); o1[1] = fmaf(p1, vv.y, o1[1]);
      o1[2] = fmaf(p1, vv.z, o1[2]); o1[3] = fmaf(p1, vv.w, o1[3]);
    }
  }
  const long long obase = (long long)b * Tq * ldo + h * kHD + td * 4;
  auto store = [&](int row, const float (&o)[4]) {
    if (row >= Tq) return;
    const long long off = obase + (long long)row * ldo;
    if (out_lo) {
      float hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split_tf32(o[j], hi[j], lo[j]);
      *reinterpret_cast<float4*>(out + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<float4*>(out_lo + off) = make_float4(lo[0], lo[1], lo[2], lo[3]);
    } else {
      *reinterpret_cast<float4*>(out + off) = make_float4(o[0], o[1], o[2], o[3]);
    }
  };
  store(q0 + tq, o0);
  store(q0 + tq + 16, o1);
}

// Shared memory of attention_fp32_kernel: sQ, sS and sT.  The row of scores over all Tk keys (sS) bounds Tk.
constexpr size_t kAttFp32MaxSmem = 200 * 1024;
inline size_t attention_fp32_smem(int Tk) { return (size_t)(32 * kHD + 32 * (Tk + 4) + 64 * 68) * sizeof(float); }

// Encoder self-attention over the [B*T, 3Q] qkv rows (q = kv = qkv, k_col0 = Q, v_col0 = 2Q); the teacher-forced decoder's
// causal self-attention with per-key validity (key_valid != null), and its cross-attention of q [B*Tq, ldq] over
// kv [B*Tk, ldkv].  out [B*Tq, H*64].
inline int launch_attention_fp32(const float* q, int ldq, int q_col0, const float* kv, int ldkv, int k_col0, int v_col0, int Tq, int Tk, int H,
                                 int B, float* out, float* out_lo, int ldo, const int* key_valid, int n_valid, cudaStream_t s) {
  const size_t smem = attention_fp32_smem(Tk);
  MT3_REQUIRE(smem <= kAttFp32MaxSmem, MT3_ERR_UNSUPPORTED, "fp32 attention: Tk=%d too long", Tk);
  const dim3 grid(cdiv(Tq, 32), H, B);
  if (key_valid) {
    MT3_TRY(set_max_dynamic_smem<attention_fp32_kernel<true>>((int)kAttFp32MaxSmem));
    attention_fp32_kernel<true><<<grid, 256, smem, s>>>(q, ldq, q_col0, kv, ldkv, k_col0, v_col0, Tq, Tk, H, out, out_lo, ldo, key_valid, n_valid);
  } else {
    MT3_TRY(set_max_dynamic_smem<attention_fp32_kernel<false>>((int)kAttFp32MaxSmem));
    attention_fp32_kernel<false><<<grid, 256, smem, s>>>(q, ldq, q_col0, kv, ldkv, k_col0, v_col0, Tq, Tk, H, out, out_lo, ldo, nullptr, 0);
  }
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// Decoder input: y[b,:] = E[tok[b],:] + PE[pos,:]  (Embed one-hot == row gather,
// layers.py:516-537; FixedEmbed decode branch, layers.py:589-596).
// ---------------------------------------------------------------------------------
__global__ void embed_kernel(const int* __restrict__ tok, const float* __restrict__ emb, int D, int vocab,
                             const float* __restrict__ pe, const int* __restrict__ pos_ptr, float* __restrict__ y, int b0) {
  pdl_wait();
  pdl_trigger();
  const int b = b0 + blockIdx.x;       // b0: first sequence of this sub-batch (decode streams)
  int t = tok[b];
  t = min(max(t, 0), vocab - 1);
  const int pos = *pos_ptr;
  const float4* e = reinterpret_cast<const float4*>(emb + (long long)t * D);
  const float4* p = reinterpret_cast<const float4*>(pe + (long long)pos * D);
  float4* o = reinterpret_cast<float4*>(y + (long long)b * D);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 a = __ldg(e + i), c = __ldg(p + i);
    o[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
  }
}

// sequences b0 .. b0 + n_cta - 1
inline int launch_embed(const int* tok, const float* emb, int D, int vocab, const float* pe, const int* pos_ptr, float* y, int b0,
                        int n_cta, cudaStream_t s) {
  MT3_CUDA_CHECK(launch_kernel(embed_kernel, dim3(n_cta), dim3(128), 0, s, false, tok, emb, D, vocab, pe, pos_ptr, y, b0));
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// logsumexp(x[0 .. V)) in a CTA of 256 threads, the one log-sum-exp of the greedy token scores and of the teacher-forced
// token scores, so that one logits row gives the same bits in both: the row maximum (fmaxf, so NaN is skipped), then
// sum expf(x - max) per thread in id order, a warp tree and the 8 warp sums in order.  A NaN in the row makes the sum, and
// the result, NaN.  Every thread calls it (it synchronises the CTA) and every thread gets the result.  red: 8 shared floats.
// BIAS: over the biased row biased_logit(x, bias) instead of x (mt3_generate_biased).
// ---------------------------------------------------------------------------------
// The logit a token picker sees under a logit bias c: -inf where c is -inf (a suppressed id, whatever the model's logit,
// NaN included), else one float32 add.  A zero bias gives x back bit for bit for every x but -0.0, which compares equal.
__device__ __forceinline__ float biased_logit(float x, float c) { return c == -INFINITY ? -INFINITY : x + c; }

template <bool BIAS = false>
__device__ __forceinline__ float block_logsumexp(const float* __restrict__ x, int V, float* red, const float* __restrict__ bias = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float mx = -INFINITY;
  for (int c = tid; c < V; c += 256) mx = fmaxf(mx, BIAS ? biased_logit(x[c], bias[c]) : x[c]);
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float se = 0.f;
  for (int c = tid; c < V; c += 256) se += expf((BIAS ? biased_logit(x[c], bias[c]) : x[c]) - mx);
  se = warp_sum(se);
  if (lane == 0) red[warp] = se;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < 8; ++w) tot += red[w];
  return mx + logf(tot);
}

// ---------------------------------------------------------------------------------
// Greedy pick + loop bookkeeping (stands in for t5x's decode loop at num_decodes=1,
// models.py:127): next = argmax(logits), like np/jnp.argmax: the first maximum wins, and
// the first NaN wins over every number (tracked apart from the maximum, so the common
// all-finite path keeps its short compare chain); finished sequences emit PAD; EOS
// (id 1, vocabularies.py:157-159) marks finished.
// The last CTA to arrive advances the shared position and publishes all_finished.
// state: [0] pos, [1] arrival counter, [2] all_finished
// token_scores (optional, row stride out_ld): [b, pos] = logits[next] - logsumexp(logits row) (block_logsumexp), 0 for a
// sequence that had finished before this step (it emits PAD); NaN when the row holds a NaN.
// y_next (optional) = E[next] + PE[pos + 1], skipped at the last step, where pos + 1 = pe_rows has no PE row.
// plen (optional, [B]): forced prompt lengths (mt3_generate_prompted).  At pos < plen[b] the sequence emits the token the
// caller put at tokens_out[b, pos] instead of its argmax: score 0, no finish; tok_cur and y_next follow that token.
// BIAS (argmax_step_biased_kernel): every read of the logits row is biased_logit(logits[b, i], bias[b, i]), bias [B, V]
// (mt3_generate_biased); argmax_step_kernel is the body at BIAS = false, as it was before the bias existed.
// ---------------------------------------------------------------------------------
template <bool BIAS>
__device__ __forceinline__ void
argmax_step_body(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur,
                 int* __restrict__ finished, int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld,
                 const int* __restrict__ plen, int* __restrict__ tok_out_user, int* __restrict__ state, int advance, int b0,
                 const float* __restrict__ emb,
                 const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next, const float* __restrict__ bias) {
  __shared__ float sv[8], slse[8];
  __shared__ int si[8], snan[8];
  __shared__ int s_next[2];
  // B = sequences in the whole batch (the arrival counter spans every sub-batch), b0 = first sequence of this launch
  const int b = b0 + blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // plen is written before the encoder runs, never by the kernel this one may start under: its load goes ahead of the wait
  const int pl = (plen && tid == 0) ? plen[b] : 0;
  pdl_wait();
  pdl_trigger();
  const float* l = logits + (long long)b * V;
  const float* bb = BIAS ? bias + (long long)b * V : nullptr;
  // every number beats the start (-inf, 0x7fffffff), so bi stays out of range only when the whole row is NaN, and then
  // nan_i = 0 replaces it
  float best = -INFINITY;
  int bi = 0x7fffffff, nan_i = 0x7fffffff;
  for (int i = tid; i < V; i += 256) {
    const float v = BIAS ? biased_logit(l[i], bb[i]) : l[i];
    if (v > best || (v == best && i < bi)) { best = v; bi = i; }
    if (v != v) nan_i = min(nan_i, i);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  nan_i = __reduce_min_sync(0xffffffffu, nan_i);
  if (lane == 0) { sv[warp] = best; si[warp] = bi; snan[warp] = nan_i; }
  __syncthreads();
  const float lse = token_scores ? block_logsumexp<BIAS>(l, V, slse, bb) : 0.f;
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) {
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
      nan_i = min(nan_i, snan[w]);
    }
    if (nan_i != 0x7fffffff) bi = nan_i;
    const int pos = state[0];
    int nxt = bi;
    float lp = token_scores ? (BIAS ? biased_logit(l[bi], bb[bi]) : l[bi]) - lse : 0.f;
    if (pos < pl) {                       // forced: the prompt token (never EOS), so the sequence cannot finish here
      nxt = tokens_out[(long long)b * out_ld + pos];
      lp = 0.f;
    } else if (finished) {
      if (finished[b]) { nxt = 0; lp = 0.f; }
      if (nxt == 1) finished[b] = 1;
    }
    s_next[0] = nxt;
    s_next[1] = pos + 1;
    if (tok_cur) tok_cur[b] = nxt;
    if (tokens_out) tokens_out[(long long)b * out_ld + pos] = nxt;
    if (token_scores) token_scores[(long long)b * out_ld + pos] = lp;
    if (tok_out_user) tok_out_user[b] = nxt;
    if (advance) {
      __threadfence();
      const int done = atomicAdd(&state[1], 1);
      if (done == B - 1) {
        __threadfence();
        int all = 1;
        if (finished) {
          for (int i = 0; i < B; ++i) all &= (*(volatile int*)&finished[i]) != 0;
        } else {
          all = 0;
        }
        state[2] = all;
        state[1] = 0;
        state[0] = pos + 1;
      }
    }
  }
  // generate loop: the next step's decoder input  y[b,:] = E[next,:] + PE[pos + 1,:]  (embed_kernel's work, layers.py:516-537,
  // :589-596) is written here, which takes one launch out of every step.  pos was read before this CTA arrived at the
  // counter, i.e. before the last CTA advances it.
  if (y_next) {
    __syncthreads();
    const int t = min(max(s_next[0], 0), V - 1), p1 = s_next[1];
    if (p1 >= pe_rows) return;
    const float4* e = reinterpret_cast<const float4*>(emb + (long long)t * D);
    const float4* pp = reinterpret_cast<const float4*>(pe + (long long)p1 * D);
    float4* o = reinterpret_cast<float4*>(y_next + (long long)b * D);
    for (int i = tid; i < D / 4; i += 256) {
      const float4 a = __ldg(e + i), c = __ldg(pp + i);
      o[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    }
  }
}

__global__ void __launch_bounds__(256)
argmax_step_kernel(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur,
                   int* __restrict__ finished, int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld,
                   const int* __restrict__ plen, int* __restrict__ tok_out_user, int* __restrict__ state, int advance, int b0,
                   const float* __restrict__ emb,
                   const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next) {
  argmax_step_body<false>(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, tok_out_user, state, advance, b0, emb,
                          pe, pe_rows, D, y_next, nullptr);
}

__global__ void __launch_bounds__(256)
argmax_step_biased_kernel(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur,
                          int* __restrict__ finished, int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld,
                          const int* __restrict__ plen, int* __restrict__ tok_out_user, int* __restrict__ state, int advance, int b0,
                          const float* __restrict__ emb, const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next,
                          const float* __restrict__ bias) {
  argmax_step_body<true>(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, tok_out_user, state, advance, b0, emb,
                         pe, pe_rows, D, y_next, bias);
}

// sequences b0 .. b0 + n_cta - 1 of a batch of B; bias [B, V] or null (the unbiased kernel)
inline int launch_argmax_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                              int out_ld, const int* plen, int* tok_out_user, int* state, int advance, int b0, const float* emb,
                              const float* pe, int pe_rows, int D, float* y_next, int n_cta, const float* bias, cudaStream_t s) {
  if (bias)
    MT3_CUDA_CHECK(launch_kernel(argmax_step_biased_kernel, dim3(n_cta), dim3(256), 0, s, false, logits, V, B, tok_cur, finished,
                                 tokens_out, token_scores, out_ld, plen, tok_out_user, state, advance, b0, emb, pe, pe_rows, D, y_next,
                                 bias));
  else
    MT3_CUDA_CHECK(launch_kernel(argmax_step_kernel, dim3(n_cta), dim3(256), 0, s, false, logits, V, B, tok_cur, finished, tokens_out,
                                 token_scores, out_ld, plen, tok_out_user, state, advance, b0, emb, pe, pe_rows, D, y_next));
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// T5X decoding.beam_search at num_decodes = 1 (the reference's decode_fn, models.py:127), one CTA per sequence.
// With one live beam the search keeps the 2 best extensions of the live prefix per step:
//   live     continues with the best token that is NOT EOS (cumulative log-probability live_lp);
//   finished whenever EOS is among the 2 best, the hypothesis "prefix + EOS" competes with the best finished one so far on
//            (live_lp_before + log p(EOS)) / brevity_penalty(alpha, length),  brevity_penalty = ((5 + n) / 6)^alpha;
//   a sequence is settled once its finished score beats what the live prefix can still reach,
//            live_lp / brevity_penalty(alpha, max_len)   (`finished[b]`, feeds the loop's all-finished flag).
// tokens_out holds the LIVE sequence; beam1_finalize_kernel cuts it at the winning finish.  Ties follow the reference's
// stable top-k (lower vocabulary id first; an existing finished hypothesis beats an equal newcomer).
// NaN logits: candidates are ranked by cand_better, so every emitted id is in [0, V).  An all-NaN row continues with
// id 0, the first non-EOS id of a stable top-2 over NaN scores (ids 0 and 1), and finishes nothing (the EOS candidate's
// score is NaN).  A row that is only partly NaN makes the log-sum-exp NaN; what T5X does then depends on its NaN
// ordering, which is not pinned here, so such rows carry no parity claim.
// beam_f [B][2] = {live_lp, finished score}, beam_i [B] = length of the best finished hypothesis (0 = none yet).
// token_scores (optional, row stride out_ld): [b, pos] = the live token's log-probability v1 - lse; with it, fin_lp_eos [B]
// keeps the EOS log-probability of the best finished hypothesis, which beam1_finalize_kernel puts at its last position.
// y_next and plen as in argmax_step_kernel: at a forced position the live prefix takes the prompt token with
// log-probability 0 (T5X's convention for prompts: forced tokens are not the model's choices), and no "prefix + EOS"
// hypothesis is made, so the live log-probability is still 0 when the prompt ends.
// ---------------------------------------------------------------------------------
// Candidate order: larger value first, NaN above every number, lower id first among equals (and among NaNs).  The
// candidates start from (-inf, 0x7fffffff), which every real candidate beats.
__device__ __forceinline__ bool cand_better(float v, int i, float ov, int oi) {
  if (isnan(v)) return !isnan(ov) || i < oi;
  return !isnan(ov) && (v > ov || (v == ov && i < oi));
}

// BIAS (beam1_step_biased_kernel): every read of the logits row is biased_logit(logits[b, i], bias[b, i]), as in
// argmax_step_body.
template <bool BIAS>
__device__ __forceinline__ void
beam1_step_body(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur, int* __restrict__ finished,
                int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                int* __restrict__ state, float* __restrict__ beam_f, float* __restrict__ fin_lp_eos, int* __restrict__ beam_i, float alpha, int max_len,
                const float* __restrict__ emb, const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next,
                const float* __restrict__ bias) {
  __shared__ float s1v[8], s2v[8], smx[8], ssum[8];
  __shared__ int s1i[8], s2i[8];
  __shared__ int s_next[2];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pl = (plen && tid == 0) ? plen[b] : 0;      // ahead of the wait, as in argmax_step_kernel
  pdl_wait();
  pdl_trigger();
  const float* l = logits + (long long)b * V;
  const float* bb = BIAS ? bias + (long long)b * V : nullptr;
  // best and second-best NON-EOS candidates (value, id), and the running maximum over everything for the log-sum-exp
  float v1 = -INFINITY, v2 = -INFINITY, mx = -INFINITY;
  int i1 = 0x7fffffff, i2 = 0x7fffffff;
  for (int i = tid; i < V; i += 256) {
    const float v = BIAS ? biased_logit(l[i], bb[i]) : l[i];
    mx = fmaxf(mx, v);
    if (i == 1) continue;                        // EOS (vocabularies.py:157-159) is handled separately
    if (cand_better(v, i, v1, i1)) { v2 = v1; i2 = i1; v1 = v; i1 = i; }
    else if (cand_better(v, i, v2, i2)) { v2 = v; i2 = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov1 = __shfl_xor_sync(0xffffffffu, v1, o), ov2 = __shfl_xor_sync(0xffffffffu, v2, o);
    const int oi1 = __shfl_xor_sync(0xffffffffu, i1, o), oi2 = __shfl_xor_sync(0xffffffffu, i2, o);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (cand_better(ov1, oi1, v1, i1)) {         // theirs wins: second = better of (mine first, their second)
      if (cand_better(v1, i1, ov2, oi2)) { v2 = v1; i2 = i1; } else { v2 = ov2; i2 = oi2; }
      v1 = ov1; i1 = oi1;
    } else if (cand_better(ov1, oi1, v2, i2)) { v2 = ov1; i2 = oi1; }
  }
  if (lane == 0) { s1v[warp] = v1; s1i[warp] = i1; s2v[warp] = v2; s2i[warp] = i2; smx[warp] = mx; }
  __syncthreads();
  float gmx = smx[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) gmx = fmaxf(gmx, smx[w]);
  float se = 0.f;
  for (int i = tid; i < V; i += 256) se += expf((BIAS ? biased_logit(l[i], bb[i]) : l[i]) - gmx);
  se = warp_sum(se);
  if (lane == 0) ssum[warp] = se;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) {
      const float ov1 = s1v[w], ov2 = s2v[w];
      const int oi1 = s1i[w], oi2 = s2i[w];
      if (cand_better(ov1, oi1, v1, i1)) {
        if (cand_better(v1, i1, ov2, oi2)) { v2 = v1; i2 = i1; } else { v2 = ov2; i2 = oi2; }
        v1 = ov1; i1 = oi1;
      } else if (cand_better(ov1, oi1, v2, i2)) { v2 = ov1; i2 = oi1; }
    }
    float tot = 0.f;
    for (int w = 0; w < 8; ++w) tot += ssum[w];
    const float lse = gmx + logf(tot);
    const float veos = BIAS ? biased_logit(l[1], bb[1]) : l[1];
    const int pos = state[0];
    const float live_prev = beam_f[2 * b];
    float fin_score = beam_f[2 * b + 1];
    const bool forced = pos < pl;
    if (forced) i1 = tokens_out[(long long)b * out_ld + pos];
    // EOS is one of the 2 best extensions iff it beats the second-best non-EOS candidate
    if (!forced && cand_better(veos, 1, v2, i2)) {
      const float cand = (live_prev + (veos - lse)) / powf((5.0f + (float)(pos + 1)) / 6.0f, alpha);
      if (cand > fin_score) {
        fin_score = cand;
        beam_f[2 * b + 1] = cand;
        beam_i[b] = pos + 1;
        if (token_scores) fin_lp_eos[b] = veos - lse;
      }
    }
    const float live = forced ? live_prev : live_prev + (v1 - lse);
    beam_f[2 * b] = live;
    tok_cur[b] = i1;
    tokens_out[(long long)b * out_ld + pos] = i1;
    if (token_scores) token_scores[(long long)b * out_ld + pos] = forced ? 0.f : v1 - lse;
    finished[b] = (beam_i[b] > 0 && fin_score > live / powf((5.0f + (float)max_len) / 6.0f, alpha)) ? 1 : 0;
    s_next[0] = i1;
    s_next[1] = pos + 1;
    __threadfence();
    const int done = atomicAdd(&state[1], 1);
    if (done == B - 1) {
      __threadfence();
      int all = 1;
      for (int i = 0; i < B; ++i) all &= (*(volatile int*)&finished[i]) != 0;
      state[2] = all;
      state[1] = 0;
      state[0] = pos + 1;
    }
  }
  if (y_next) {
    __syncthreads();
    const int t = min(max(s_next[0], 0), V - 1), p1 = s_next[1];
    if (p1 >= pe_rows) return;
    const float4* e = reinterpret_cast<const float4*>(emb + (long long)t * D);
    const float4* pp = reinterpret_cast<const float4*>(pe + (long long)p1 * D);
    float4* o = reinterpret_cast<float4*>(y_next + (long long)b * D);
    for (int i = tid; i < D / 4; i += 256) {
      const float4 a = __ldg(e + i), c = __ldg(pp + i);
      o[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    }
  }
}

__global__ void __launch_bounds__(256)
beam1_step_kernel(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur, int* __restrict__ finished,
                  int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                  int* __restrict__ state, float* __restrict__ beam_f, float* __restrict__ fin_lp_eos, int* __restrict__ beam_i, float alpha, int max_len,
                  const float* __restrict__ emb, const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next) {
  beam1_step_body<false>(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i, alpha,
                         max_len, emb, pe, pe_rows, D, y_next, nullptr);
}

__global__ void __launch_bounds__(256)
beam1_step_biased_kernel(const float* __restrict__ logits, int V, int B, int* __restrict__ tok_cur, int* __restrict__ finished,
                         int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                         int* __restrict__ state, float* __restrict__ beam_f, float* __restrict__ fin_lp_eos, int* __restrict__ beam_i,
                         float alpha, int max_len, const float* __restrict__ emb, const float* __restrict__ pe, int pe_rows, int D,
                         float* __restrict__ y_next, const float* __restrict__ bias) {
  beam1_step_body<true>(logits, V, B, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i, alpha,
                        max_len, emb, pe, pe_rows, D, y_next, bias);
}

// bias [B, V] or null (the unbiased kernel)
inline int launch_beam1_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                             int out_ld, const int* plen, int* state, float* beam_f, float* fin_lp_eos, int* beam_i, float alpha,
                             int max_len, const float* emb, const float* pe, int pe_rows, int D, float* y_next, const float* bias,
                             cudaStream_t s) {
  if (bias)
    MT3_CUDA_CHECK(launch_kernel(beam1_step_biased_kernel, dim3(B), dim3(256), 0, s, false, logits, V, B, tok_cur, finished, tokens_out,
                                 token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i, alpha, max_len, emb, pe, pe_rows, D,
                                 y_next, bias));
  else
    MT3_CUDA_CHECK(launch_kernel(beam1_step_kernel, dim3(B), dim3(256), 0, s, false, logits, V, B, tok_cur, finished, tokens_out,
                                 token_scores, out_ld, plen, state, beam_f, fin_lp_eos, beam_i, alpha, max_len, emb, pe, pe_rows, D,
                                 y_next));
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// the best finished hypothesis = the live prefix up to its finish + EOS, zeros after; a sequence that never finished keeps
// its live tokens (the reference returns the live beam when nothing finished).
// token_scores (optional, [B, L], as beam1_step_kernel wrote them) get the same cut: fin_lp_eos[b] at n - 1, zeros after.
// scores (optional, [B]) = T5X beam_search's score: the best finished score of beam_f, or the live log-probability when
// nothing finished.
__global__ void beam1_finalize_kernel(int* __restrict__ tokens, int B, int L, int steps, const int* __restrict__ beam_i,
                                      float* __restrict__ token_scores, const float* __restrict__ beam_f,
                                      const float* __restrict__ fin_lp_eos, float* __restrict__ scores) {
  const int b = blockIdx.x;
  const int n = beam_i[b];
  if (scores && threadIdx.x == 0) scores[b] = n > 0 ? beam_f[2 * b + 1] : beam_f[2 * b];
  const int from = n > 0 ? n : steps;
  if (n > 0 && threadIdx.x == 0) {
    tokens[(long long)b * L + n - 1] = 1;
    if (token_scores) token_scores[(long long)b * L + n - 1] = fin_lp_eos[b];
  }
  for (int i = from + threadIdx.x; i < L; i += blockDim.x) {
    tokens[(long long)b * L + i] = 0;
    if (token_scores) token_scores[(long long)b * L + i] = 0.f;
  }
}

inline int launch_beam1_finalize(int* tokens, int B, int L, int steps, const int* beam_i, float* token_scores, const float* beam_f,
                                 const float* fin_lp_eos, float* scores, cudaStream_t s) {
  beam1_finalize_kernel<<<B, 128, 0, s>>>(tokens, B, L, steps, beam_i, token_scores, beam_f, fin_lp_eos, scores);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// scores[b] = the sum of token_scores[b, 0 .. L) (greedy sequence score), in one fixed order whatever the steps ran: each
// of 128 threads sums ids tid, tid + 128, ... in order, then a warp tree and the 4 warp sums in order.
__global__ void __launch_bounds__(128) seq_score_kernel(const float* __restrict__ token_scores, int L, float* __restrict__ scores) {
  __shared__ float red[4];
  const int b = blockIdx.x, tid = threadIdx.x;
  float s = 0.f;
  for (int i = tid; i < L; i += 128) s += token_scores[(long long)b * L + i];
  s = warp_sum(s);
  if ((tid & 31) == 0) red[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) scores[b] = ((red[0] + red[1]) + red[2]) + red[3];
}

inline int launch_seq_score(const float* token_scores, int B, int L, float* scores, cudaStream_t s) {
  seq_score_kernel<<<B, 128, 0, s>>>(token_scores, L, scores);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// T5X decoding.temperature_sample's pick (mt3_generate_sampled), one CTA per sequence, parameters from sp (device):
//   z = logits / temperature (IEEE division), kept in shared memory;
//   top-k (0 < topk < V): keep every id whose z is >= the k-th largest z (ties at the k-th value are all kept);
//   top-p (0 < topp < 1), after top-k: keep id i iff the softmax mass of the kept ids with z_j > z_i is below topp;
//   next = argmax_i (z_i + g_i) over the kept ids (the first id wins a tie), g_i = -log(-log(u_i)), u_i from
//     Philox4x32-10 with key sp->key and counter (i / 4, pos, sp->row0 + b, 0), word i % 4 (philox.cuh): a row's
//     numbers depend only on (key, stream, position).
// The filters sort (order-preserving key of z, id) pairs, V padded to a power of two (nsort), with a bitonic network in
// shared memory, then cut the sorted row at the k-th value and at the first tie group whose preceding mass, summed in one
// fixed order, reaches topp: both cuts are deterministic.  The dropped ids become -inf in the z row.
// token_scores: sp->rescale_log_probs != 0: z[next] - logsumexp(kept z); else logits[next] - logsumexp(logits row), greedy's
// bits.  Both through block_logsumexp.  A row with a NaN emits its first NaN id with a NaN score, as argmax_step_kernel.
// The bookkeeping (finished rows emit PAD with score 0, EOS finishes, forced prompt positions, the arrival counter that
// advances state, y_next) is argmax_step_kernel's.
// ---------------------------------------------------------------------------------
constexpr int kSampleMaxSortV = 4096;          // the largest vocabulary the top-k / top-p filters sort
constexpr int kSampleMaxSmem = 200 * 1024;

// nsort: the sort's padded length (0 when V is too large to sort); the dynamic shared memory is nsort pairs and the z row
inline int sample_sort_n(int V) {
  if (V > kSampleMaxSortV) return 0;
  int n = 256;
  while (n < V) n <<= 1;
  return n;
}
inline size_t sample_step_smem(int V) { return (size_t)sample_sort_n(V) * 8 + (size_t)V * 4; }

// ascending in the result = descending in z (-0.0 after +0.0; NaN never reaches the sort)
__device__ __forceinline__ uint32_t z_order_desc(float z) {
  const uint32_t u = __float_as_uint(z);
  return (u & 0x80000000u) ? u : ~(u | 0x80000000u);
}

// BIAS (sample_step_biased_kernel): every read of the logits row is biased_logit(logits[b, i], bias[b, i]), as in
// argmax_step_body: z = biased logits / temperature, and the unrescaled scores are taken over the biased row.
template <bool BIAS>
__device__ __forceinline__ void
sample_step_body(const float* __restrict__ logits, int V, int B, int nsort, int* __restrict__ tok_cur, int* __restrict__ finished,
                 int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                 int* __restrict__ state, const mt3_sample_params* __restrict__ sp, const float* __restrict__ emb,
                 const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next, const float* __restrict__ bias,
                 unsigned char* smem_raw) {
  unsigned long long* skey = reinterpret_cast<unsigned long long*>(smem_raw);   // [nsort] (z order << 32 | id)
  float* z = reinterpret_cast<float*>(smem_raw + (size_t)nsort * 8);              // [V]
  __shared__ float sv[8], slse[8], sscan[8];
  __shared__ int si[8], snan[8];
  __shared__ int s_cut[2];
  __shared__ int s_next[2];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // plen and the parameters are written before the encoder runs: their loads go ahead of the wait
  const int pl = (plen && tid == 0) ? plen[b] : 0;
  const float temp = sp->temperature, topp = sp->topp;
  const int topk = sp->topk, rescale = sp->rescale_log_probs;
  const uint32_t k0 = sp->key[0], k1 = sp->key[1], stream = sp->row0 + (uint32_t)b;
  pdl_wait();
  pdl_trigger();
  const float* l = logits + (long long)b * V;
  const float* bb = BIAS ? bias + (long long)b * V : nullptr;
  // read by every thread before its CTA arrives at the counter (the barriers below), so before the last CTA advances it
  const int pos = state[0];
  int nan_i = 0x7fffffff;
  for (int i = tid; i < V; i += 256) {
    const float v = BIAS ? biased_logit(l[i], bb[i]) : l[i];
    z[i] = v / temp;
    if (v != v) nan_i = min(nan_i, i);
  }
  nan_i = __reduce_min_sync(0xffffffffu, nan_i);
  if (lane == 0) snan[warp] = nan_i;
  if (tid == 0) { s_cut[0] = V; s_cut[1] = V; }
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 8; ++w) nan_i = min(nan_i, snan[w]);
  const bool has_nan = nan_i != 0x7fffffff;
  const bool use_k = topk > 0 && topk < V, use_p = topp > 0.f && topp < 1.f;
  if (!has_nan && (use_k || use_p) && nsort >= V) {
    for (int j = tid; j < nsort; j += 256)
      skey[j] = j < V ? ((unsigned long long)z_order_desc(z[j]) << 32) | (unsigned)j : ~0ull;
    __syncthreads();
    for (int k = 2; k <= nsort; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int t = tid; t < nsort / 2; t += 256) {
          const int i = 2 * t - (t & (j - 1)), p = i + j;
          const unsigned long long a = skey[i], c = skey[p];
          if ((a > c) == ((i & k) == 0)) { skey[i] = c; skey[p] = a; }
        }
        __syncthreads();
      }
    }
    auto zs = [&](int j) { return z[(int)(skey[j] & 0xffffffffu)]; };
    if (use_k) {     // the one sorted position where the run of values >= the k-th value ends
      const float zk = zs(topk - 1);
      for (int j = topk - 1 + tid; j < V; j += 256)
        if (zs(j) >= zk && (j + 1 == V || zs(j + 1) < zk)) s_cut[0] = j + 1;
      __syncthreads();
    }
    const int n1 = s_cut[0];
    if (use_p) {
      // thread t holds sorted positions [t c, t c + c): its sum in order, an exclusive scan of the 256 sums (warp shuffles,
      // then the 8 warp totals in order), then its own positions again in order
      const int c = nsort / 256;
      const float z0 = zs(0);
      float run = 0.f;
      for (int q = 0; q < c; ++q) {
        const int j = tid * c + q;
        if (j < n1) run += expf(zs(j) - z0);
      }
      float incl = run;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      float m = __shfl_up_sync(0xffffffffu, incl, 1);
      if (lane == 0) m = 0.f;
      if (lane == 31) sscan[warp] = incl;
      __syncthreads();
      float base = 0.f, tot = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        if (w == warp) base = tot;
        tot += sscan[w];
      }
      m += base;
      const float thr = topp * tot;
      for (int q = 0; q < c; ++q) {
        const int j = tid * c + q;
        if (j >= n1) break;
        const float zj = zs(j);
        if (j > 0 && zj < zs(j - 1) && m >= thr) { atomicMin(&s_cut[1], j); break; }
        m += expf(zj - z0);
      }
      __syncthreads();
    }
    // the kept ids are the sorted prefix [0, n): z >= its last value.  That id's z is kept, so no thread overwrites it.
    const float zc = zs(min(n1, s_cut[1]) - 1);
    for (int i = tid; i < V; i += 256)
      if (!(z[i] >= zc)) z[i] = -INFINITY;
    __syncthreads();
  }
  // Gumbel-max: thread t draws the ids 4 j .. 4 j + 3 of the Philox blocks j = t, t + 256, ...
  float best = -INFINITY;
  int bi = 0x7fffffff;
  if (!has_nan) {
    for (int j = tid; 4 * j < V; j += 256) {
      uint32_t w[4];
      philox4x32_10((uint32_t)j, (uint32_t)pos, stream, 0u, k0, k1, w);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = 4 * j + q;
        if (i < V) {
          const float v = z[i] + (-logf(-logf(philox_uniform(w[q]))));
          if (v > best || (v == best && i < bi)) { best = v; bi = i; }
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  float lse = 0.f;
  if constexpr (BIAS) {
    if (token_scores && !has_nan) lse = rescale ? block_logsumexp(z, V, slse) : block_logsumexp<true>(l, V, slse, bb);
  } else {
    lse = (token_scores && !has_nan) ? block_logsumexp(rescale ? z : l, V, slse) : 0.f;
  }
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] > best || (sv[w] == best && si[w] < bi)) { best = sv[w]; bi = si[w]; }
    int nxt = has_nan ? nan_i : bi;
    float lp = 0.f;
    if (token_scores)
      lp = has_nan ? __int_as_float(0x7fffffff) : (rescale ? z[nxt] : (BIAS ? biased_logit(l[nxt], bb[nxt]) : l[nxt])) - lse;
    if (pos < pl) {                       // forced: the prompt token (never EOS), so the sequence cannot finish here
      nxt = tokens_out[(long long)b * out_ld + pos];
      lp = 0.f;
    } else {
      if (finished[b]) { nxt = 0; lp = 0.f; }
      if (nxt == 1) finished[b] = 1;
    }
    s_next[0] = nxt;
    s_next[1] = pos + 1;
    tok_cur[b] = nxt;
    tokens_out[(long long)b * out_ld + pos] = nxt;
    if (token_scores) token_scores[(long long)b * out_ld + pos] = lp;
    __threadfence();
    const int done = atomicAdd(&state[1], 1);
    if (done == B - 1) {
      __threadfence();
      int all = 1;
      for (int i = 0; i < B; ++i) all &= (*(volatile int*)&finished[i]) != 0;
      state[2] = all;
      state[1] = 0;
      state[0] = pos + 1;
    }
  }
  if (y_next) {
    __syncthreads();
    const int t = min(max(s_next[0], 0), V - 1), p1 = s_next[1];
    if (p1 >= pe_rows) return;
    const float4* e = reinterpret_cast<const float4*>(emb + (long long)t * D);
    const float4* pp = reinterpret_cast<const float4*>(pe + (long long)p1 * D);
    float4* o = reinterpret_cast<float4*>(y_next + (long long)b * D);
    for (int i = tid; i < D / 4; i += 256) {
      const float4 a = __ldg(e + i), c = __ldg(pp + i);
      o[i] = make_float4(a.x + c.x, a.y + c.y, a.z + c.z, a.w + c.w);
    }
  }
}

__global__ void __launch_bounds__(256)
sample_step_kernel(const float* __restrict__ logits, int V, int B, int nsort, int* __restrict__ tok_cur, int* __restrict__ finished,
                   int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                   int* __restrict__ state, const mt3_sample_params* __restrict__ sp, const float* __restrict__ emb,
                   const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  sample_step_body<false>(logits, V, B, nsort, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D,
                          y_next, nullptr, smem_raw);
}

__global__ void __launch_bounds__(256)
sample_step_biased_kernel(const float* __restrict__ logits, int V, int B, int nsort, int* __restrict__ tok_cur, int* __restrict__ finished,
                          int* __restrict__ tokens_out, float* __restrict__ token_scores, int out_ld, const int* __restrict__ plen,
                          int* __restrict__ state, const mt3_sample_params* __restrict__ sp, const float* __restrict__ emb,
                          const float* __restrict__ pe, int pe_rows, int D, float* __restrict__ y_next, const float* __restrict__ bias) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  sample_step_body<true>(logits, V, B, nsort, tok_cur, finished, tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D,
                         y_next, bias, smem_raw);
}

// every sequence of a batch of B; sp DEV; bias [B, V] or null (the unbiased kernel).  Top-k / top-p at V > kSampleMaxSortV are
// refused by the caller, which knows sp.
inline int launch_sample_step(const float* logits, int V, int B, int* tok_cur, int* finished, int* tokens_out, float* token_scores,
                              int out_ld, const int* plen, int* state, const mt3_sample_params* sp, const float* emb, const float* pe,
                              int pe_rows, int D, float* y_next, const float* bias, cudaStream_t s) {
  const size_t smem = sample_step_smem(V);
  MT3_REQUIRE(smem <= (size_t)kSampleMaxSmem, MT3_ERR_UNSUPPORTED, "sampling: vocabulary %d too large for one CTA's row", V);
  if (bias) {
    MT3_TRY(set_max_dynamic_smem<sample_step_biased_kernel>(kSampleMaxSmem));
    MT3_CUDA_CHECK(launch_kernel(sample_step_biased_kernel, dim3(B), dim3(256), smem, s, false, logits, V, B, sample_sort_n(V), tok_cur,
                                 finished, tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D, y_next, bias));
  } else {
    MT3_TRY(set_max_dynamic_smem<sample_step_kernel>(kSampleMaxSmem));
    MT3_CUDA_CHECK(launch_kernel(sample_step_kernel, dim3(B), dim3(256), smem, s, false, logits, V, B, sample_sort_n(V), tok_cur, finished,
                                 tokens_out, token_scores, out_ld, plen, state, sp, emb, pe, pe_rows, D, y_next));
  }
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// layers.dot_product_attention (layers.py:85-157) as a standalone op, exact fp32, any head_dim, optional additive bias
// [b, h, q, kv] (layers.py:143-146: combined mask / relative-position bias).  No 1/sqrt(d) scaling (the reference folds it
// into the query initialiser, layers.py:230-234).  One warp per (batch, head, query); scores in shared memory.
// q [b, tq, h, d], k / v [b, tk, h, d], out [b, tq, h, d].
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
dot_product_attention_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                             const float* __restrict__ bias, int B, int TQ, int TK, int H, int D, float* __restrict__ out) {
  extern __shared__ float att_sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long item = (long long)blockIdx.x * 4 + warp;          // (b, h, qi)
  if (item >= (long long)B * H * TQ) return;
  const int qi = (int)(item % TQ), h = (int)((item / TQ) % H), b = (int)(item / ((long long)TQ * H));
  float* sc = att_sm + (size_t)warp * TK;
  const float* qr = q + (((long long)b * TQ + qi) * H + h) * D;
  float mx = -INFINITY;
  for (int j = lane; j < TK; j += 32) {
    const float* kr = k + (((long long)b * TK + j) * H + h) * D;
    float s = 0.f;
    for (int d = 0; d < D; ++d) s = fmaf(qr[d], kr[d], s);
    if (bias) s += bias[(((long long)b * H + h) * TQ + qi) * TK + j];
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < TK; j += 32) {
    const float e = expf(sc[j] - mx);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.0f / sum;
  float* orow = out + (((long long)b * TQ + qi) * H + h) * D;
  for (int d = lane; d < D; d += 32) {
    float acc = 0.f;
    for (int j = 0; j < TK; ++j) acc = fmaf(sc[j], v[(((long long)b * TK + j) * H + h) * D + d], acc);
    orow[d] = acc * inv;
  }
}

// advance the position without an argmax (decode_step called with tok_out == NULL)
__global__ void advance_pos_kernel(int* state) {
  pdl_wait();
  state[0] += 1;
}

// GenericTokenVocabulary._decode_tf (vocabularies.py:241-271).
__global__ void vocab_decode_kernel(const int* __restrict__ ids, int B, int L, int num_regular, int* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  bool eos = false;
  for (int i = 0; i < L; ++i) {
    const int id = ids[(long long)b * L + i];
    eos = eos || (id == 1);
    int o;
    if (eos) o = -1;
    else if (id >= 3 && id < 3 + num_regular) o = id - 3;
    else o = -2;
    out[(long long)b * L + i] = o;
  }
}

// dst[k, col_off + n*col_stride] = src[k, n] * (g ? g[k] : 1)   -- weight re-layout at model creation
__global__ void scale_copy_cols_kernel(const float* __restrict__ src, int K, int N, const float* __restrict__ g,
                                       float* __restrict__ dst, int ldd, int col_off, int col_stride) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)K * N) return;
  const int k = (int)(i / N), n = (int)(i % N);
  dst[(long long)k * ldd + col_off + (long long)n * col_stride] = src[i] * (g ? g[k] : 1.f);
}

// hi/lo split of a dense fp32 array (tf32x3 operands)
__global__ void split_pair_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = reinterpret_cast<const float4*>(x)[i];
  float4 h, l;
  split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
  reinterpret_cast<float4*>(hi)[i] = h;
  reinterpret_cast<float4*>(lo)[i] = l;
}

// src [K, N] row-major -> dst_hi (/dst_lo) [N, K]: the K-major ("transposed") weight layout the wgmma B operand reads.
__global__ void transpose_split_kernel(const float* __restrict__ src, int K, int N, float* __restrict__ dst_hi,
                                       float* __restrict__ dst_lo) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? src[(long long)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) {
      const float v = tile[threadIdx.x][i];
      if (dst_lo) {
        float h, l;
        split_tf32(v, h, l);
        dst_hi[(long long)n * K + k] = h;
        dst_lo[(long long)n * K + k] = l;
      } else {
        dst_hi[(long long)n * K + k] = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// Teacher-forced decoder input: y[b * Lp + i, :] = E[tok[b, i], :] + PE[i, :] for i < L (network.py:211-217; positions
// are arange(L)), 0 for the padding rows L <= i < Lp.  Ids outside [0, vocab) are clamped as in embed_kernel.
// y_lo != null: the row is written as a tf32 hi/lo pair.  One CTA per row.
// ---------------------------------------------------------------------------------
__global__ void embed_seq_kernel(const int* __restrict__ tok, int L, int Lp, const float* __restrict__ emb, int D, int vocab,
                                 const float* __restrict__ pe, float* __restrict__ y, float* __restrict__ y_lo) {
  const int row = blockIdx.x, b = row / Lp, i = row % Lp;
  float4* o = reinterpret_cast<float4*>(y + (long long)row * D);
  float4* ol = y_lo ? reinterpret_cast<float4*>(y_lo + (long long)row * D) : nullptr;
  if (i >= L) {
    for (int c = threadIdx.x; c < D / 4; c += blockDim.x) {
      o[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ol) ol[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    return;
  }
  const int t = min(max(tok[(long long)b * L + i], 0), vocab - 1);
  const float4* e = reinterpret_cast<const float4*>(emb + (long long)t * D);
  const float4* p = reinterpret_cast<const float4*>(pe + (long long)i * D);
  for (int c = threadIdx.x; c < D / 4; c += blockDim.x) {
    const float4 a = __ldg(e + c), q = __ldg(p + c);
    const float4 v = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
    if (ol) {
      float4 h, l;
      split_tf32(v.x, h.x, l.x); split_tf32(v.y, h.y, l.y); split_tf32(v.z, h.z, l.z); split_tf32(v.w, h.w, l.w);
      o[c] = h;
      ol[c] = l;
    } else {
      o[c] = v;
    }
  }
}

inline int launch_embed_seq(const int* tok, int B, int L, int Lp, const float* emb, int D, int vocab, const float* pe, float* y, float* y_lo,
                            cudaStream_t s) {
  embed_seq_kernel<<<B * Lp, 128, 0, s>>>(tok, L, Lp, emb, D, vocab, pe, y, y_lo);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

// ---------------------------------------------------------------------------------
// Token score of T5X score_batch (z_loss = 0): score[b, i] = (x[t] - logsumexp(x)) * w over the logits row x of position
// (b, i), t = target[b, i] (clamped into [0, V)), w = weight[b, i] or, without weights, target > 0; a weight of 0 scores
// exactly 0.  One CTA per row of a chunk of padded rows: logits [n, V] hold rows row0 .. row0 + n - 1 of [B * Lp]; rows
// with i >= L are padding and skipped.  logits_out [B, L, V] (optional) receives a copy of each row.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
token_score_kernel(const float* __restrict__ logits, int V, int row0, int Lp, int L, const int* __restrict__ target,
                   const int* __restrict__ weight, float* __restrict__ scores, float* __restrict__ logits_out) {
  __shared__ float red[8];
  const int g = row0 + blockIdx.x;
  const int b = g / Lp, i = g % Lp;
  if (i >= L) return;
  const int tid = threadIdx.x;
  const float* x = logits + (long long)blockIdx.x * V;
  const long long pos = (long long)b * L + i;
  if (logits_out) {
    const float4* src = reinterpret_cast<const float4*>(x);
    float4* dst = reinterpret_cast<float4*>(logits_out + pos * V);
    for (int c = tid; c < V / 4; c += 256) dst[c] = src[c];
  }
  if (!scores) return;
  const float lse = block_logsumexp(x, V, red);
  if (tid == 0) {
    const int tg = target[pos];
    const float wt = weight ? (float)weight[pos] : (tg > 0 ? 1.f : 0.f);
    const int t = min(max(tg, 0), V - 1);
    scores[pos] = wt != 0.f ? (x[t] - lse) * wt : 0.f;
  }
}

inline int launch_token_score(const float* logits, int V, int row0, int n_rows, int Lp, int L, const int* target, const int* weight,
                              float* scores, float* logits_out, cudaStream_t s) {
  if (n_rows <= 0) return MT3_OK;
  token_score_kernel<<<n_rows, 256, 0, s>>>(logits, V, row0, Lp, L, target, weight, scores, logits_out);
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

}  // namespace mt3
