// Exact-fp32 CUDA-core GEMM with the fused epilogues the MT3 blocks need.
// This is the parity anchor (MT3_GEMM_FP32_SIMT): same arithmetic type as the
// reference's DenseGeneral (layers.py:373-418, lax.dot_general in float32), used to
// validate the wgmma path and as the small-M decode GEMM.
//
//   C[M,N] = epilogue( row_scale[m] * (A[M,K] . B[K,N]) )
//
// Epilogues (all fused, nothing re-read from HBM):
//   EPI_STORE       plain store
//   EPI_RESIDUAL    + R[m,n]                     (x + Attn(..), x + MLP(..): network.py:68,83)
//   EPI_ADD_PE      + PE[m % pe_T, n]            (FixedEmbed add, network.py:180)
//   EPI_GATED_GELU  B's columns are interleaved (wi_0[j], wi_1[j]); writes
//                   gelu_tanh(c0) * c1 into C[m, j]  (MlpBlock, layers.py:459-476)
//   split store     columns >= n_split go to C1 at row offset *c1_pos: the fused
//                   self-attention K/V cache append (layers.py:272-289)
// row_scale carries the RMSNorm factor rsqrt(mean(x^2)+eps) (layers.py:613-616); the
// norm's learned scale is folded into B's rows when the model is created.
#pragma once

#include <cuda_fp16.h>

#include "common.cuh"

namespace mt3 {

enum { EPI_STORE = 0, EPI_RESIDUAL = 1, EPI_ADD_PE = 2, EPI_GATED_GELU = 3 };

struct GemmArgs {
  const float* A; int lda;
  const float* B; int ldb;
  int M, N, K;
  const float* row_scale;      // [M] or null
  int epi;
  const float* R; int ldr;     // EPI_RESIDUAL
  const float* pe; int pe_T; int pe_ld;  // EPI_ADD_PE
  float* C; int ldc;
  int n_split;                 // columns >= n_split -> head-major K/V store at C1 (N if unused)
  void* C1; int kv_fmt; int hm_rows_per_b; int hm_cap; int hm_H; const int* hm_pos;   // head-major K/V store, see kv_dest()
};

// Head-major K/V layout shared by the self-attention cache and the hoisted cross K/V:
//   kv[b][which(0=K,1=V)][head][cap] rows of 64 elements
// Row m of the GEMM is (b, t) = (m / rows_per_b, m % rows_per_b + pos); column c (relative to n_split) is
// (which, head, d) = (c / (H*64), (c % (H*64)) / 64, c % 64).  Decode: rows_per_b = 1, pos = cache index
// (the fused KV-cache append, layers.py:272-289); cross K/V: rows_per_b = T, pos = 0.
// kv_fmt (mt3_model_config.kv_cache_format) is the storage format of a row:
//   0  64 x float                                                           256 B
//   1  64 x __half                                                          128 B
//   2  "p24": 64 x u16 (bits 31..16 of the float) then 64 x u8 (bits 15..8)  192 B.  The decoder rebuilds a float
//      with ONE byte permute per element by repeating the third byte as the fourth (value bits = hi16:lo8:lo8), and
//      the encoder picks the nearest value of that form.  Within a binade those values are 257 ulps apart (1 ulp where
//      the low byte wraps from 0xFF to 0x00), so the nearest one is at most 128 ulps away: relative error < 2^-16.
//      Neighbouring values are an odd number of ulps apart, so there are no ties.
__host__ __device__ __forceinline__ int kv_row_bytes(int kv_fmt) { return kv_fmt == 0 ? 256 : (kv_fmt == 1 ? 128 : 192); }

__device__ __forceinline__ long long kv_dest(int m, int c, int rows_per_b, int cap, int H, int pos, int kv_fmt, int& d) {
  const int b = m / rows_per_b, t = m % rows_per_b + pos;
  const int which = c / (H * 64), h = (c % (H * 64)) >> 6;
  d = c & 63;
  return ((((long long)b * 2 + which) * H + h) * cap + t) * kv_row_bytes(kv_fmt);
}

// the 24 stored bits (hi16 << 8 | lo8) of the p24 value nearest to x: the candidates are the codes t = bits >> 8 and
// t +- 1 (t - 1 only while it keeps the sign); on equal distance the earlier of t, t + 1, t - 1 would be kept
__device__ __forceinline__ uint32_t p24_encode(float x) {
  const uint32_t bits = __float_as_uint(x);
  const uint32_t t = bits >> 8;
  uint32_t best = t;
  uint32_t v = (t << 8) | (t & 255u);
  uint32_t err = v > bits ? v - bits : bits - v;
  const uint32_t tu = t + 1;                                   // same sign: the sign bit is far above the carry
  v = (tu << 8) | (tu & 255u);
  uint32_t e = v > bits ? v - bits : bits - v;
  if (e < err) { err = e; best = tu; }
  if ((t & 0x7fffffu) != 0u) {
    const uint32_t td = t - 1;
    v = (td << 8) | (td & 255u);
    e = v > bits ? v - bits : bits - v;
    if (e < err) best = td;
  }
  return best;
}
__device__ __forceinline__ float p24_decode(uint32_t t) { return __uint_as_float((t << 8) | (t & 255u)); }

// store N (1, 2 or 4) consecutive elements d..d+N-1 (d % N == 0) of one K/V row
template <int N>
__device__ __forceinline__ void kv_store(char* row, int kv_fmt, int d, const float* v) {
  if (kv_fmt == 0) {
    float* dst = reinterpret_cast<float*>(row) + d;
    if (N == 4) *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
    else if (N == 2) *reinterpret_cast<float2*>(dst) = make_float2(v[0], v[1]);
    else dst[0] = v[0];
  } else if (kv_fmt == 1) {
    __half* dst = reinterpret_cast<__half*>(row) + d;
    if (N == 1) dst[0] = __float2half_rn(v[0]);
#pragma unroll
    for (int i = 0; i + 1 < N; i += 2) reinterpret_cast<__half2*>(dst)[i / 2] = __floats2half2_rn(v[i], v[i + 1]);
  } else {
    uint32_t t[N];
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = p24_encode(v[i]);
    unsigned short* hi = reinterpret_cast<unsigned short*>(row) + d;
    unsigned char* lo = reinterpret_cast<unsigned char*>(row) + 128 + d;
    if (N == 4) {
      *reinterpret_cast<uint2*>(hi) = make_uint2((t[0] >> 8) | ((t[1] >> 8) << 16), (t[2] >> 8) | ((t[3] >> 8) << 16));
      *reinterpret_cast<uint32_t*>(lo) = (t[0] & 255u) | ((t[1] & 255u) << 8) | ((t[2] & 255u) << 16) | ((t[3] & 255u) << 24);
    } else if (N == 2) {
      *reinterpret_cast<uint32_t*>(hi) = (t[0] >> 8) | ((t[1] >> 8) << 16);
      *reinterpret_cast<unsigned short*>(lo) = (unsigned short)((t[0] & 255u) | ((t[1] & 255u) << 8));
    } else {
      hi[0] = (unsigned short)(t[0] >> 8);
      lo[0] = (unsigned char)(t[0] & 255u);
    }
  }
}

__device__ __forceinline__ float gelu_tanh(float x) {
  // flax.linen.gelu(approximate=True): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))
  const float c = 0.7978845608028654f;
  return 0.5f * x * (1.f + tanhf(c * (x + 0.044715f * x * x * x)));
}

// Thread tile = (TM/4 x TN/4) blocks of 4x4, blocks BM/(TM/4) rows / BN/(TN/4) cols apart so
// that every shared-memory read is a conflict-free 16-byte access.
template <int BM, int BN, int BK, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
sgemm_kernel(const GemmArgs p) {
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int TX = BN / TN;
  constexpr int RB = TM / 4, CB = TN / 4;
  constexpr int RSTEP = BM / RB, CSTEP = BN / CB;
  constexpr int APAD = 4;
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  constexpr int A_F4 = BM * BK / 4, B_F4 = BK * BN / 4;
  constexpr int A_PER = (A_F4 + NT - 1) / NT, B_PER = (B_F4 + NT - 1) / NT;
  float4 ra[A_PER], rb[B_PER];

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      const int idx = tid + i * NT;
      const int row = idx / (BK / 4), kq = idx % (BK / 4);
      ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < A_F4 && m0 + row < p.M)
        ra[i] = __ldg(reinterpret_cast<const float4*>(p.A + (long long)(m0 + row) * p.lda + k0 + kq * 4));
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      const int idx = tid + i * NT;
      const int kr = idx / (BN / 4), nq = idx % (BN / 4);
      rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < B_F4 && n0 + nq * 4 < p.N)
        rb[i] = __ldg(reinterpret_cast<const float4*>(p.B + (long long)(k0 + kr) * p.ldb + n0 + nq * 4));
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      const int idx = tid + i * NT;
      if (idx < A_F4) {
        const int row = idx / (BK / 4), kq = idx % (BK / 4);
        As[buf][kq * 4 + 0][row] = ra[i].x;
        As[buf][kq * 4 + 1][row] = ra[i].y;
        As[buf][kq * 4 + 2][row] = ra[i].z;
        As[buf][kq * 4 + 3][row] = ra[i].w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      const int idx = tid + i * NT;
      if (idx < B_F4) {
        const int kr = idx / (BN / 4), nq = idx % (BN / 4);
        *reinterpret_cast<float4*>(&Bs[buf][kr][nq * 4]) = rb[i];
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int nk = p.K / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        const float4 v = *reinterpret_cast<const float4*>(&As[buf][k][r * RSTEP + ty * 4]);
        a[r * 4 + 0] = v.x; a[r * 4 + 1] = v.y; a[r * 4 + 2] = v.z; a[r * 4 + 3] = v.w;
      }
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        const float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][c * CSTEP + tx * 4]);
        b[c * 4 + 0] = v.x; b[c * 4 + 1] = v.y; b[c * 4 + 2] = v.z; b[c * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

  // ---- epilogue ----
#pragma unroll
  for (int r = 0; r < RB; ++r) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + r * RSTEP + ty * 4 + i;
      if (m >= p.M) continue;
      const float rs = p.row_scale ? p.row_scale[m] : 1.f;
#pragma unroll
      for (int c = 0; c < CB; ++c) {
        const int n = n0 + c * CSTEP + tx * 4;
        if (n >= p.N) continue;
        float4 v = make_float4(acc[r * 4 + i][c * 4 + 0] * rs, acc[r * 4 + i][c * 4 + 1] * rs,
                               acc[r * 4 + i][c * 4 + 2] * rs, acc[r * 4 + i][c * 4 + 3] * rs);
        if (p.epi == EPI_GATED_GELU) {
          float2 o = make_float2(gelu_tanh(v.x) * v.y, gelu_tanh(v.z) * v.w);
          *reinterpret_cast<float2*>(p.C + (long long)m * p.ldc + (n >> 1)) = o;
          continue;
        }
        if (p.epi == EPI_RESIDUAL) {
          const float4 q = *reinterpret_cast<const float4*>(p.R + (long long)m * p.ldr + n);
          v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
        } else if (p.epi == EPI_ADD_PE) {
          const float4 q = __ldg(reinterpret_cast<const float4*>(p.pe + (long long)(m % p.pe_T) * p.pe_ld + n));
          v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
        }
        if (n < p.n_split) {
          *reinterpret_cast<float4*>(p.C + (long long)m * p.ldc + n) = v;
        } else {
          const int pos = p.hm_pos ? *p.hm_pos : 0;
          int d;
          char* row = reinterpret_cast<char*>(p.C1) + kv_dest(m, n - p.n_split, p.hm_rows_per_b, p.hm_cap, p.hm_H, pos, p.kv_fmt, d);
          const float v4[4] = {v.x, v.y, v.z, v.w};
          kv_store<4>(row, p.kv_fmt, d, v4);
        }
      }
    }
  }
}

// Host-side dispatch: big tiles for the encoder-sized GEMMs (M = B*T), a narrow tile for
// the decode step (M = B) so that N/32 CTAs stream the weight matrix.
inline int launch_sgemm(const GemmArgs& a, cudaStream_t s) {
  MT3_REQUIRE(a.K % 16 == 0 && a.N % 4 == 0 && a.lda % 4 == 0 && a.ldb % 4 == 0 && a.ldc % 2 == 0, MT3_ERR_UNSUPPORTED,
              "sgemm: K=%d must be a multiple of 16 and N=%d, lda=%d, ldb=%d of 4", a.K, a.N, a.lda, a.ldb);
  MT3_REQUIRE(a.n_split % 4 == 0, MT3_ERR_UNSUPPORTED, "sgemm: n_split must be a multiple of 4");
  if (a.M > 128) {
    dim3 grid(cdiv(a.N, 128), cdiv(a.M, 128));
    sgemm_kernel<128, 128, 16, 8, 8><<<grid, 256, 0, s>>>(a);
  } else {
    dim3 grid(cdiv(a.N, 32), cdiv(a.M, 64));
    sgemm_kernel<64, 32, 16, 4, 4><<<grid, 128, 0, s>>>(a);
  }
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}

}  // namespace mt3
