// K4: attention on the Hopper tensor cores (wgmma + TMA), sm_90a: the encoder's self-attention and the teacher-forced
// decoder's causal self-attention and cross-attention (attention_tc_kernel, launch_attention_tc).
//
// Reference: dot_product_attention (layers.py:85-157): softmax_k(q . k^T) . v, logits NOT scaled by
// 1/sqrt(d) (layers.py:230-234), mask all ones in the encoder (network.py:283-289).
//
// One work item = 128 query rows of one (batch, head); T <= 256 keys, head_dim 64.  Two consumer warpgroups take 64
// query rows each; everything between the two MMAs stays in registers.
//   S[64 q, T k]   = Q . K^T   wgmma m64n128k8 tf32 per 128-key chunk, K=64 (8 k-steps), A and B from shared memory;
//                               error-compensated (Qhi.Khi + Qhi.Klo + Qlo.Khi) when hi/lo operands are given
//   P = exp(S - rowmax)         in the accumulator registers: a row lives in the four lanes of a quad, so the row
//                               maximum and sum are two shuffles; P (rounded to tf32, unnormalised) overwrites S
//   O[64 q, 64 d]  = P . V      wgmma m64n64k8 with the A operand taken from those registers.  B operand = V^T tiles
//                               [64 d x 32 keys] (keys contiguous, K-major), written per head by the QKV GEMM epilogue
//                               (TcGemmArgs::VT_*) with the keys of every group of 8 in the order vt_key_slot() gives:
//                               that is the order in which an accumulator thread's columns form an A fragment.
//                               P . Vhi + P . Vlo; 1/rowsum is applied in the epilogue.
// Shared memory (192 KB): [ Q hi/lo 64 KB | slot0 64 KB | slot1 64 KB ]; slots hold K chunk c (hi/lo) and later
// V chunk c (hi/lo).  384 threads: warps 0..7 = the two consumer warpgroups, warps 8..11 = the producer warpgroup (one
// thread of it issues TMA); the producer hands most of its registers to the consumers (setmaxnreg).
// Operands come straight from the qkv buffers the QKV GEMM epilogue wrote ([B*T, 3*H*64] hi and lo)
// through two TMA tensor maps; output is [B*T, H*64] (hi/lo split for the out-projection GEMM).
#pragma once

#include "common.cuh"
#include "gemm_tc.cuh"
#include "tc.cuh"

namespace mt3 {

__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

constexpr int kAtQ = 128;                 // query rows per work item
constexpr int kAtKC = 128;                // keys per chunk
constexpr int kAtSub = 128 * 32 * 4;      // one [128 x 32] fp32 sub-tile = 16 KB
constexpr int kVSub = 64 * 32 * 4;        // one [64 d x 32 keys] V^T sub-tile = 8 KB
constexpr int kAtSmem = 3 * 4 * kAtSub + 256;   // 196 864 B of the 232 448 a CTA may have
constexpr int kAtThreads = 384;           // warps 0..7: two consumer warpgroups, warps 8..11: producer warpgroup (TMA)

// s += S chunk (128 keys) of this warpgroup's 64 query rows.
template <bool SPLIT3>
__device__ __forceinline__ void at_qk(float (&s)[64], uint32_t q_addr, uint32_t k_addr) {
  tc::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {                           // 64 d = 2 sub-tiles x 4 k-steps of 8
    const uint32_t off = (ks >> 2) * kAtSub + (ks & 3) * 32;
    const uint64_t a_hi = tc::smem_desc_k_sw128(q_addr + off);
    const uint64_t b_hi = tc::smem_desc_k_sw128(k_addr + off);
    if (SPLIT3) {
      tc::wgmma_tf32_m64n128(s, tc::smem_desc_k_sw128(q_addr + 2 * kAtSub + off), b_hi);
      tc::wgmma_tf32_m64n128(s, a_hi, tc::smem_desc_k_sw128(k_addr + 2 * kAtSub + off));
    }
    tc::wgmma_tf32_m64n128(s, a_hi, b_hi);
  }
  tc::wgmma_commit();
}

// O += P chunk . V chunk: k-step j takes the accumulator's 8-column block j as its A fragment (see vt_key_slot()).
template <bool SPLIT3>
__device__ __forceinline__ void at_pv(float (&o)[32], const float (&p)[64], uint32_t v_addr) {
  tc::wgmma_fence();
#pragma unroll
  for (int j = 0; j < 16; ++j) {                             // sub-tile j / 4 (32 keys), k-step j % 4 inside it
    const uint32_t b = v_addr + (j >> 2) * kVSub + (j & 3) * 32;
    const uint32_t a0 = __float_as_uint(p[4 * j]), a1 = __float_as_uint(p[4 * j + 2]);
    const uint32_t a2 = __float_as_uint(p[4 * j + 1]), a3 = __float_as_uint(p[4 * j + 3]);
    tc::wgmma_tf32_m64n64_rs(o, a0, a1, a2, a3, tc::smem_desc_k_sw128(b));
    if (SPLIT3) tc::wgmma_tf32_m64n64_rs(o, a0, a1, a2, a3, tc::smem_desc_k_sw128(b + 4 * kVSub));
  }
  tc::wgmma_commit();
}

// Row maxima of one S chunk over the columns < TK; mx0 = row lane / 4, mx1 = that row + 8 (this thread's columns only).
__device__ __forceinline__ void at_chunk_max(const float (&s)[64], int col0, int TK, float& mx0, float& mx1) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e)
      if (col0 + 8 * j + e < TK) {
        mx0 = fmaxf(mx0, s[4 * j + e]);
        mx1 = fmaxf(mx1, s[4 * j + 2 + e]);
      }
}

// S chunk -> P chunk in place: exp(s - max) rounded to tf32 (exactly what the tensor core will read), 0 beyond TK.
// ROUND = false: P stays fp32, for the split P . V of at_pv_lo().
template <bool ROUND = true>
__device__ __forceinline__ void at_chunk_exp(float (&s)[64], int col0, int TK, float mx0, float mx1, float& sum0, float& sum1) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = col0 + 8 * j + e < TK;
      // ex2.approx (2 ulp) is ample: the value is rounded to tf32 (2^-11) right after, or split into tf32 hi + lo
      const float p0 = ok ? (ROUND ? round_tf32(exp2f((s[4 * j + e] - mx0) * 1.4426950408889634f))
                                   : exp2f((s[4 * j + e] - mx0) * 1.4426950408889634f)) : 0.f;
      const float p1 = ok ? (ROUND ? round_tf32(exp2f((s[4 * j + 2 + e] - mx1) * 1.4426950408889634f))
                                   : exp2f((s[4 * j + 2 + e] - mx1) * 1.4426950408889634f)) : 0.f;
      s[4 * j + e] = p0;
      s[4 * j + 2 + e] = p1;
      sum0 += p0;
      sum1 += p1;
    }
}

// The lo half of a split P . V: once the MMAs that read the fp32 P as its tf32 hi part (the tensor core ignores the low
// 13 mantissa bits) have completed, P becomes P - hi (exact) in place and O += P_lo . V_hi.
__device__ __forceinline__ void at_pv_lo(float (&o)[32], float (&p)[64], uint32_t v_addr) {
#pragma unroll
  for (int i = 0; i < 64; ++i) p[i] -= __uint_as_float(__float_as_uint(p[i]) & 0xffffe000u);
  at_pv<false>(o, p, v_addr);
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Mask kinds of the attention kernel.  NONE: every key below the item's key count is visible (encoder, cross-attention).
// CAUSAL: query i sees key j iff j <= i, j < n_valid and key_valid[b][j] > 0 (the teacher-forced decoder's
// make_decoder_mask); a row whose every key is masked writes 0.
constexpr int kAtMaskNone = 0, kAtMaskCausal = 1;

// s = -inf where the key is masked for the row: this thread's rows i0 and i0 + 8 (sequence positions), columns
// j0 + 8 j + {0, 1} of the chunk (key positions).
__device__ __forceinline__ void at_chunk_mask(float (&s)[64], int j0, int i0, const int* __restrict__ kv, int n_valid) {
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int key = j0 + 8 * j + e;
      const bool ok = key < n_valid && __ldg(kv + key) > 0;
      if (!ok || key > i0) s[4 * j + e] = -INFINITY;
      if (!ok || key > i0 + 8) s[4 * j + 2 + e] = -INFINITY;
    }
}

// PERSISTENT: one CTA per SM walks over work items (sequence b, head h, 128-query tile) with stride gridDim.x.  All
// mbarriers complete exactly once per item, so the wait parity is (item counter & 1).  The TMA thread streams ahead of
// the consumers: Q of item i+1 as soon as both warpgroups have finished S(i), K of item i+1 as soon as they have
// finished P.V(i), i.e. under the epilogue of i; V(i) replaces K(i) in the slots as soon as S(i) is complete.
// NCHUNK = 128-key chunks per item (1: TK <= 128, 2: TK <= 256): compile-time, so that every wgmma sits on a uniform path.
// Q of head h: columns q_col0 + 64 h of the rows [b Tq, (b + 1) Tq) of tq_*; K: columns k_col0 + 64 h of the rows
// [b Tk, (b + 1) Tk) of tk_*.  Under CAUSAL the items of key parts that lie wholly above the diagonal are skipped (the
// item counter does not advance for them, in the producer and the consumers alike).
// PSPLIT: P . V in 3xTF32 too (P_hi V_hi + P_hi V_lo + P_lo V_hi, P kept in fp32) instead of P rounded to tf32.  The
// teacher-forced pass splits P so that the decoder's logits stay within the float32 bar of DESIGN.md section 4 (P rounded
// to tf32 moves them by about 1e-4 of their scale); the encoder rounds P, and its accuracy bar and speed were measured so.
template <bool SPLIT3, bool KSPLIT, int NCHUNK, int MASK, bool PSPLIT>
__global__ void __launch_bounds__(kAtThreads, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tq_hi, const __grid_constant__ CUtensorMap tq_lo,
                    const __grid_constant__ CUtensorMap tk_hi, const __grid_constant__ CUtensorMap tk_lo,
                    const __grid_constant__ CUtensorMap tv_hi, const __grid_constant__ CUtensorMap tv_lo, int q_col0, int k_col0, int Tq,
                    int Tk, int H, int B, float* __restrict__ out_hi, float* __restrict__ out_lo, int ldo, int TK_arg, int KS_arg,
                    float* __restrict__ part_o, float2* __restrict__ part_ml, const int* __restrict__ key_valid, int n_valid) {
  const int KS = KSPLIT ? KS_arg : 1, TK = KSPLIT ? TK_arg : Tk;      // compile-time 1 / Tk in the common single-pass form
  // TK = keys per work item (<= 256), KS = key parts per query tile (Tk <= KS * TK).  KS == 1: the item covers all keys and
  // writes the normalised output.  KS > 1 (T = 512, ismir2021; the decoder's L > 256): an item covers keys
  // [ks TK, (ks + 1) TK) and writes its UNNORMALISED O tile plus (row max, row sum) to part_o / part_ml; the combine kernel
  // merges the parts (softmax is associative over key blocks: O = sum_k e^(m_k - m) O_k / sum_k e^(m_k - m) l_k).
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((tc::smem_u32(smem) & 1023u) != 0) __trap();          // the swizzled tiles need 1024-byte alignment
  uint8_t* sQ = smem;                       // Q hi: 2 sub-tiles, Q lo: 2 sub-tiles (64 KB)
  uint8_t* slot[2] = {smem + 4 * kAtSub, smem + 8 * kAtSub};
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 12 * kAtSub);
  uint64_t* q_full = bars;                  // Q landed
  uint64_t* k_full = bars + 1;              // [2] K chunk landed
  uint64_t* v_full = bars + 3;              // [2] V chunk landed
  uint64_t* s_done = bars + 5;              // the S MMAs have read Q and K (256 arrivals)
  uint64_t* pv_done = bars + 6;             // the P.V MMAs have read V (256 arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int nchunk = NCHUNK;
  const int ntile = (Tq + kAtQ - 1) / kAtQ;
  const int n_items = B * H * ntile * KS;
  constexpr uint32_t kSubBytes = kAtSub;
  const uint32_t lo_tiles = SPLIT3 ? 2u : 1u;

  if (warp == 8 && lane == 0) {
    tc::prefetch_tmap(&tq_hi);
    tc::prefetch_tmap(&tk_hi);
    tc::prefetch_tmap(&tv_hi);
    if (SPLIT3) {
      tc::prefetch_tmap(&tq_lo);
      tc::prefetch_tmap(&tk_lo);
      tc::prefetch_tmap(&tv_lo);
    }
    tc::mbar_init(q_full, 1);
    for (int c = 0; c < 2; ++c) {
      tc::mbar_init(&k_full[c], 1);
      tc::mbar_init(&v_full[c], 1);
    }
    tc::mbar_init(s_done, 256);
    tc::mbar_init(pv_done, 256);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 8 && tc::elect_one()) {
      int it = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
        const uint32_t ph = it & 1, pph = ph ^ 1;
        const int ks = item % KS, it2 = item / KS;
        const int qt = it2 % ntile, h = (it2 / ntile) % H, b = it2 / (ntile * H);
        const int qrow0 = b * Tq, q0 = qt * kAtQ, koff = ks * TK;
        const int krow0 = b * Tk;
        if (MASK == kAtMaskCausal && koff > q0 + kAtQ - 1) { --it; continue; }
        // Q: the region is free since the previous item's S MMAs (s_done, waited for before that item's V was loaded)
        tc::mbar_arrive_expect_tx(q_full, 2 * lo_tiles * kSubBytes);
        for (int sub = 0; sub < 2; ++sub) {
          tc::tma_load_2d(sQ + sub * kAtSub, &tq_hi, q_full, q_col0 + h * 64 + sub * 32, qrow0 + q0);
          if (SPLIT3) tc::tma_load_2d(sQ + (2 + sub) * kAtSub, &tq_lo, q_full, q_col0 + h * 64 + sub * 32, qrow0 + q0);
        }
        // K chunks -> slots: free once the previous item's P.V MMAs have read V out of them
        if (it > 0) tc::mbar_wait(pv_done, pph);
        for (int c = 0; c < nchunk; ++c) {
          tc::mbar_arrive_expect_tx(&k_full[c], 2 * lo_tiles * kSubBytes);
          for (int sub = 0; sub < 2; ++sub) {
            tc::tma_load_2d(slot[c] + sub * kAtSub, &tk_hi, &k_full[c], k_col0 + h * 64 + sub * 32, krow0 + koff + c * kAtKC);
            if (SPLIT3) tc::tma_load_2d(slot[c] + (2 + sub) * kAtSub, &tk_lo, &k_full[c], k_col0 + h * 64 + sub * 32, krow0 + koff + c * kAtKC);
          }
        }
        // V^T chunks reuse the slots once every S MMA of THIS item has read K
        tc::mbar_wait(s_done, ph);
        const int vrow = (b * H + h) * 64;
        for (int c = 0; c < nchunk; ++c) {
          tc::mbar_arrive_expect_tx(&v_full[c], 4 * lo_tiles * kVSub);
          for (int sub = 0; sub < 4; ++sub) {
            tc::tma_load_2d(slot[c] + sub * kVSub, &tv_hi, &v_full[c], koff + c * kAtKC + sub * 32, vrow);
            if (SPLIT3) tc::tma_load_2d(slot[c] + (4 + sub) * kVSub, &tv_lo, &v_full[c], koff + c * kAtKC + sub * 32, vrow);
          }
        }
      }
    }
  } else {
    // ---- consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile; this thread rows r and r + 8,
    // columns 8 j + 2 (lane % 4) + {0, 1} of every 8-column block j ----
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2;
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    const uint32_t q_addr = tc::smem_u32(sQ) + wg * 64 * 128;    // 64 rows of 128 B into each sub-tile
    int it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
      const uint32_t ph = it & 1;
      const int ks = item % KS, it2 = item / KS;
      const int qt = it2 % ntile, h = (it2 / ntile) % H, b = it2 / (ntile * H);
      const int row0 = b * Tq, q0 = qt * kAtQ;
      if (MASK == kAtMaskCausal && ks * TK > q0 + kAtQ - 1) { --it; continue; }
      float s0[64], s1[64], o[32];
      // ---- S = Q K^T ----
#pragma unroll
      for (int i = 0; i < 64; ++i) s0[i] = s1[i] = 0.f;
      tc::mbar_wait(q_full, ph);
      tc::mbar_wait(&k_full[0], ph);
      at_qk<SPLIT3>(s0, q_addr, tc::smem_u32(slot[0]));
      if (nchunk > 1) {
        tc::mbar_wait(&k_full[1], ph);
        at_qk<SPLIT3>(s1, q_addr, tc::smem_u32(slot[1]));
      }
      tc::wgmma_wait<0>();
      tc::mbar_arrive(s_done);
      if (MASK == kAtMaskCausal) {
        const int* kv = key_valid + (long long)b * n_valid;
        at_chunk_mask(s0, ks * TK + cq, q0 + r, kv, n_valid);
        if (nchunk > 1) at_chunk_mask(s1, ks * TK + kAtKC + cq, q0 + r, kv, n_valid);
      }
      // ---- P = exp(S - rowmax), in place ----
      float mx0 = -INFINITY, mx1 = -INFINITY;
      at_chunk_max(s0, cq, TK, mx0, mx1);
      if (nchunk > 1) at_chunk_max(s1, kAtKC + cq, TK, mx0, mx1);
      mx0 = quad_max(mx0);
      mx1 = quad_max(mx1);
      float sum0 = 0.f, sum1 = 0.f;
      // a row with every key of this item masked has max -inf: exp(-inf - 0) = 0 instead of exp(-inf + inf) = NaN
      const float me0 = (MASK != kAtMaskNone && mx0 == -INFINITY) ? 0.f : mx0;
      const float me1 = (MASK != kAtMaskNone && mx1 == -INFINITY) ? 0.f : mx1;
      at_chunk_exp<!PSPLIT>(s0, cq, TK, me0, me1, sum0, sum1);
      if (nchunk > 1) at_chunk_exp<!PSPLIT>(s1, kAtKC + cq, TK, me0, me1, sum0, sum1);
      // ---- O = P V ----
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      tc::mbar_wait(&v_full[0], ph);
      at_pv<SPLIT3>(o, s0, tc::smem_u32(slot[0]));
      if (nchunk > 1) {
        tc::mbar_wait(&v_full[1], ph);
        at_pv<SPLIT3>(o, s1, tc::smem_u32(slot[1]));
      }
      if (PSPLIT) {                 // the MMAs above read P as its hi part; they must be done before P becomes P_lo
        tc::wgmma_wait<0>();
        at_pv_lo(o, s0, tc::smem_u32(slot[0]));
        if (nchunk > 1) at_pv_lo(o, s1, tc::smem_u32(slot[1]));
      }
      sum0 = quad_sum(sum0);
      sum1 = quad_sum(sum1);
      tc::wgmma_wait<0>();
      tc::mbar_arrive(pv_done);
      // ---- epilogue: a quad stores 32 contiguous bytes of a row per 8-column block ----
      // key parts stay unnormalised: the combine kernel divides; a row with no visible key writes 0
      const float inv0 = KS == 1 ? ((MASK != kAtMaskNone && !(sum0 > 0.f)) ? 0.f : 1.0f / sum0) : 1.0f;
      const float inv1 = KS == 1 ? ((MASK != kAtMaskNone && !(sum1 > 0.f)) ? 0.f : 1.0f / sum1) : 1.0f;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int q = q0 + r + 8 * half;
        if (q >= Tq) continue;
        const float inv = half ? inv1 : inv0;
        if (KS > 1 && (lane & 3) == 0)
          part_ml[(((long long)ks * B + b) * H + h) * Tq + q] = make_float2(half ? mx1 : mx0, half ? sum1 : sum0);
        const long long off = (long long)(row0 + q) * ldo + h * 64 + cq;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float x = o[4 * j + 2 * half] * inv, y = o[4 * j + 2 * half + 1] * inv;
          if (KS > 1) {
            *reinterpret_cast<float2*>(part_o + (long long)ks * B * Tq * ldo + off + 8 * j) = make_float2(x, y);
          } else if (out_lo) {
            float xh, xl, yh, yl;
            split_tf32(x, xh, xl);
            split_tf32(y, yh, yl);
            *reinterpret_cast<float2*>(out_hi + off + 8 * j) = make_float2(xh, yh);
            *reinterpret_cast<float2*>(out_lo + off + 8 * j) = make_float2(xl, yl);
          } else {
            *reinterpret_cast<float2*>(out_hi + off + 8 * j) = make_float2(x, y);
          }
        }
      }
    }
  }
}

// Merge of KS key parts: out[row, h, :] = sum_k e^(m_k - m) O_k / sum_k e^(m_k - m) l_k.  One warp per (row, head).
// CAUSAL: row t reads only the parts that start at or before t (the others were skipped or are wholly masked for it), a
// part with no visible key (m_k = -inf) weighs 0, and a row with none at all writes 0.
template <bool CAUSAL>
__global__ void attention_combine_kernel(const float* __restrict__ part_o, const float2* __restrict__ part_ml, int B, int T, int H, int KS,
                                         int TK, float* __restrict__ out_hi, float* __restrict__ out_lo) {
  const long long item = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);     // (b, t, h)
  const int lane = threadIdx.x & 31;
  if (item >= (long long)B * T * H) return;
  const int h = (int)(item % H);
  const long long row = item / H;                      // b * T + t
  const int b = (int)(row / T), t = (int)(row % T);
  const int ldo = H * 64;
  const int ks_end = CAUSAL ? min(KS, t / TK + 1) : KS;
  float m = -INFINITY;
  for (int k = 0; k < ks_end; ++k) m = fmaxf(m, part_ml[(((long long)k * B + b) * H + h) * T + t].x);
  float den = 0.f;
  float2 acc = make_float2(0.f, 0.f);
  for (int k = 0; k < ks_end; ++k) {
    const float2 ml = part_ml[(((long long)k * B + b) * H + h) * T + t];
    const float w = (CAUSAL && ml.x == -INFINITY) ? 0.f : expf(ml.x - m);
    den = fmaf(w, ml.y, den);
    const float2 o = *reinterpret_cast<const float2*>(part_o + (long long)k * B * T * ldo + row * ldo + h * 64 + lane * 2);
    acc.x = fmaf(w, o.x, acc.x);
    acc.y = fmaf(w, o.y, acc.y);
  }
  const float inv = (CAUSAL && !(den > 0.f)) ? 0.f : 1.0f / den;
  const float x = acc.x * inv, y = acc.y * inv;
  const long long off = row * ldo + h * 64 + lane * 2;
  if (out_lo) {
    float xh, xl, yh, yl;
    split_tf32(x, xh, xl);
    split_tf32(y, yh, yl);
    *reinterpret_cast<float2*>(out_hi + off) = make_float2(xh, yh);
    *reinterpret_cast<float2*>(out_lo + off) = make_float2(xl, yl);
  } else {
    *reinterpret_cast<float2*>(out_hi + off) = make_float2(x, y);
  }
}

// Items of at most 256 keys; the key-split form (parts of 256 keys, unnormalised, merged by the combine kernel) when there
// are more.
//   causal:     Tq = Tk = a multiple of 128 (the sequence padded to the query tile: padded rows come after every real
//               position, so causality hides them); key j of sequence b is visible to query i iff j <= i, j < n_valid and
//               key_valid[b * n_valid + j] > 0.  The parts wholly above the diagonal are skipped.
//   otherwise:  all Tk keys visible to every query (the encoder: Tq = Tk = T; cross-attention: Tk = T); Tk <= 256 and a
//               multiple of 8, or a multiple of 256 (ismir2021: 512).
inline int attention_tc_parts(int Tk, bool causal) {
  if (Tk <= 2 * kAtKC) return 1;
  return causal ? cdiv(Tk, 2 * kAtKC) : Tk / (2 * kAtKC);
}
// floats of scratch the key-split form needs: KS unnormalised O tiles + KS (max, sum) pairs per (row, head)
inline int64_t attention_tc_scratch_floats(int B, int Tq, int Tk, int H, bool causal) {
  const int64_t KS = attention_tc_parts(Tk, causal);
  if (KS == 1) return 0;
  return KS * (int64_t)B * Tq * H * 64 + KS * (int64_t)B * H * Tq * 2;
}
inline bool attention_tc_supported(int Tq, int Tk, bool causal) {
  if (causal) return Tq == Tk && Tq % kAtQ == 0;
  return Tk % 8 == 0 && (Tk <= 2 * kAtKC || Tk % (2 * kAtKC) == 0);
}

// q: an operand whose rows [b Tq, (b + 1) Tq) hold sequence b's queries, head h at columns q_col0 + 64 h; k likewise with
// Tk and k_col0; vt: V^T [B*H*64, Tk] (box rows 64, keys in vt_key_slot() order); out [B*Tq, H*64] (out_lo optional).
// split_p: P . V in 3xTF32 as well (the kernel's PSPLIT); ignored unless split3.  scratch: attention_tc_scratch_floats()
// floats for the key-split form.
inline int launch_attention_tc(const TcOperand& q, int q_col0, int Tq, const TcOperand& k, int k_col0, int Tk, const TcOperand& vt, int B,
                               int H, float* out_hi, float* out_lo, bool split3, bool split_p, bool causal, const int* key_valid, int n_valid,
                               cudaStream_t s, float* scratch) {
  MT3_REQUIRE(attention_tc_supported(Tq, Tk, causal), MT3_ERR_UNSUPPORTED, "tc attention: Tq=%d Tk=%d causal=%d is not supported", Tq, Tk,
              (int)causal);
  MT3_REQUIRE(!causal || key_valid != nullptr, MT3_ERR_BAD_ARG, "tc attention: the causal form needs key_valid");
  MT3_REQUIRE(!split3 || (q.has_lo && k.has_lo && vt.has_lo), MT3_ERR_BAD_ARG, "tc attention: TF32X3 needs hi/lo operands");
  const int KS = attention_tc_parts(Tk, causal);
  const int TK = KS == 1 ? Tk : 2 * kAtKC;
  const int nchunk = cdiv(TK, kAtKC);
  MT3_REQUIRE(KS == 1 || scratch != nullptr, MT3_ERR_WORKSPACE, "tc attention: Tk=%d needs the key-split scratch buffer", Tk);
  float* part_o = scratch;
  float2* part_ml = KS > 1 ? reinterpret_cast<float2*>(scratch + (int64_t)KS * B * Tq * H * 64) : nullptr;
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    MT3_CUDA_CHECK(cudaGetDevice(&dev));
    MT3_CUDA_CHECK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
  }
  const int n_items = B * H * cdiv(Tq, kAtQ) * KS;
  dim3 grid(n_items < sm_count ? n_items : sm_count);       // one persistent CTA per SM (192 KB of shared memory each)
  const CUtensorMap& q_lo = split3 ? q.lo : q.hi;
  const CUtensorMap& k_lo = split3 ? k.lo : k.hi;
  const CUtensorMap& v_lo = split3 ? vt.lo : vt.hi;
#define MT3_AT_LAUNCH(S3, KSP, NC, MK, PS)                                                                                            \
  do {                                                                                                                                \
    MT3_TRY((set_max_dynamic_smem<attention_tc_kernel<S3, KSP, NC, MK, PS>>(kAtSmem)));                                               \
    attention_tc_kernel<S3, KSP, NC, MK, PS><<<grid, kAtThreads, kAtSmem, s>>>(q.hi, q_lo, k.hi, k_lo, vt.hi, v_lo, q_col0, k_col0, Tq, Tk, \
                                                                               H, B, out_hi, out_lo, H * 64, TK, KS, part_o, part_ml,  \
                                                                               key_valid, n_valid);                                    \
  } while (0)
  // causal: items of two chunks always take the key-split instantiation, which writes the normalised output itself when
  // KS == 1 (Tk = 256); the single-pass two-chunk form spills with the mask's registers
#define MT3_AT_FORMS(S3, PS)                                                  \
  if (causal && nchunk > 1) MT3_AT_LAUNCH(S3, true, 2, kAtMaskCausal, PS);    \
  else if (causal) MT3_AT_LAUNCH(S3, false, 1, kAtMaskCausal, PS);            \
  else if (KS > 1) MT3_AT_LAUNCH(S3, true, 2, kAtMaskNone, PS);               \
  else if (nchunk > 1) MT3_AT_LAUNCH(S3, false, 2, kAtMaskNone, PS);          \
  else MT3_AT_LAUNCH(S3, false, 1, kAtMaskNone, PS);
  if (split3 && split_p) { MT3_AT_FORMS(true, true) }
  else if (split3) { MT3_AT_FORMS(true, false) }
  else { MT3_AT_FORMS(false, false) }
#undef MT3_AT_FORMS
#undef MT3_AT_LAUNCH
  MT3_LAUNCH_CHECK();
  if (KS > 1) {
    const long long items = (long long)B * Tq * H;
    if (causal)
      attention_combine_kernel<true><<<(unsigned)((items + 7) / 8), 256, 0, s>>>(part_o, part_ml, B, Tq, H, KS, TK, out_hi, out_lo);
    else
      attention_combine_kernel<false><<<(unsigned)((items + 7) / 8), 256, 0, s>>>(part_o, part_ml, B, Tq, H, KS, TK, out_hi, out_lo);
    MT3_LAUNCH_CHECK();
  }
  return MT3_OK;
}

}  // namespace mt3
