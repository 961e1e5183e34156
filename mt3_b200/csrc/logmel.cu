// K1: fused log-mel frontend for sm_90a.
//
// Replaces spectrograms.compute_spectrogram (spectrograms.py:64-73) ->
// spectral_ops.compute_logmel/compute_mel/compute_mag/stft/safe_log
// (spectral_ops.py:29-88): frame (hop 128, pad_end) -> periodic Hann -> rFFT-2048 ->
// |.| -> mel filterbank (on magnitude) -> log(where(x<=0, eps, x)).
//
// Design (one warp per frame, nothing but the audio is read and only the log-mel
// frames are written -- the reference materialises a [B,256,1025] complex64
// spectrum, 134 MB at B=64):
//   * the CTA stages the audio span of its frames in shared memory (each sample is
//     shared by 16 overlapping frames) together with the Hann window;
//   * a 2048-point real FFT is a 1024-point complex FFT of z[n] = x[2n] + i x[2n+1]
//     plus an untangling pass.  1024 = 32 x 32: lane n2 holds z[32 n1 + n2] and
//     runs a radix-2 DIF 32-point FFT entirely in registers (twiddles are
//     compile-time constants), multiplies by W_1024^(n2 k1), the 32x32 block is
//     transposed through padded shared memory, and a second in-register 32-point
//     FFT yields Z[k1 + 32 k2] in lane k1;
//   * the untangle step X[k] = E[k] + W_2048^k O[k] needs Z[1024-k], which lives
//     in lane (32 - k1) mod 32: fetched with warp shuffles;
//   * magnitudes go to shared memory; the mel "matmul" (99.6 % zeros: <= 2 non-zeros
//     per FFT bin, <= 10 per mel bin) is a banded gather-FMA, lane m handles mel bins
//     m, m+32, ..., so the final store is coalesced.
// Roofline: 655 360 algorithmic bytes and ~14.4 MFLOP of butterflies per mt3
// segment; with hop 128 every sample feeds 16 frames, so the kernel is bound by
// fp32 issue / shared memory, not HBM (DESIGN.md, "K1").
// Range: every kernel here takes |X| of each bin other than DC and Nyquist as
// sqrtf(Xr^2 + Xi^2), which is exact to rounding for about 2^-63 <= |X| <= 2^64.  Below,
// Xr^2 + Xi^2 is subnormal and loses relative precision (under ~2^-75 it rounds to 0); above,
// it overflows to +inf.  DC and Nyquist are real, |Z0.x +/- Z0.y|, and have neither limit;
// nor do tf.abs and the float64 oracle.  Audio in [-1, 1] gives |X| <= N/2 <= 2^13.
#include <math.h>
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace mt3 {

struct Frontend {
  mt3_frontend_config cfg;
  int n_bins;              // fft/2 + 1
  float* d_window;         // [fft]
  float2* d_tw1024;        // [32 k1][32 lane]  W_1024^(lane*k1)
  int* d_mel_off = nullptr;    // [n_mel + 1] CSR offsets into d_mel_csr (compact per-mel-bin taps, no padding)
  float* d_mel_csr = nullptr;  // [nnz span] weights of mel bin m for FFT bins bin0[m] .. bin0[m] + cnt - 1
  int* d_mel_lo = nullptr;     // [n_mel] first non-zero FFT bin of mel bin m (un-clamped)
  float2* d_tw_nc = nullptr;   // [R k1][32 lane]  W_NC^(lane*k1), NC = fft/2 = 32 R (fft 1024 / 4096 kernels)
  float2* d_rtw;           // [1024]            W_2048^k
  int* d_mel_bin0;         // [n_mel] first FFT bin of the tap window
  float* d_mel_w;          // [taps][n_mel] zero-padded band of the mel matrix
  int taps;                // taps per mel bin (max support width)
  int csr_len = 0;         // floats in d_mel_csr
  int nnz;
};

namespace {

__host__ __device__ constexpr int brev5(int r) {
  return ((r & 1) << 4) | ((r & 2) << 2) | (r & 4) | ((r & 8) >> 2) | ((r & 16) >> 4);
}

// W_32^m = (cos(2 pi m/32), -sin(2 pi m/32)); returns c = cos, s = sin.
__device__ __forceinline__ void tw32(int m, float& c, float& s) {
  switch (m) {
    case 1: c = 0.98078528040323043f; s = 0.19509032201612825f; break;
    case 2: c = 0.92387953251128674f; s = 0.38268343236508978f; break;
    case 3: c = 0.83146961230254524f; s = 0.55557023301960218f; break;
    case 4: c = 0.70710678118654757f; s = 0.70710678118654757f; break;
    case 5: c = 0.55557023301960218f; s = 0.83146961230254524f; break;
    case 6: c = 0.38268343236508978f; s = 0.92387953251128674f; break;
    case 7: c = 0.19509032201612825f; s = 0.98078528040323043f; break;
    case 9: c = -0.19509032201612825f; s = 0.98078528040323043f; break;
    case 10: c = -0.38268343236508978f; s = 0.92387953251128674f; break;
    case 11: c = -0.55557023301960218f; s = 0.83146961230254524f; break;
    case 12: c = -0.70710678118654757f; s = 0.70710678118654757f; break;
    case 13: c = -0.83146961230254524f; s = 0.55557023301960218f; break;
    case 14: c = -0.92387953251128674f; s = 0.38268343236508978f; break;
    case 15: c = -0.98078528040323043f; s = 0.19509032201612825f; break;
    default: c = 1.f; s = 0.f; break;
  }
}

// In-register 32-point forward FFT, radix-2 decimation in frequency.
// Output is bit-reversed: x[r] holds X[brev5(r)].
__device__ __forceinline__ void fft32(float (&xr)[32], float (&xi)[32]) {
#pragma unroll
  for (int stage = 0; stage < 5; ++stage) {
    const int span = 16 >> stage;
#pragma unroll
    for (int a = 0; a < 32; ++a) {
      if ((a & span) == 0) {
        const int b = a + span;
        const int m = (a & (span - 1)) * (16 / span);
        const float tr = xr[a] - xr[b];
        const float ti = xi[a] - xi[b];
        xr[a] += xr[b];
        xi[a] += xi[b];
        if (m == 0) {
          xr[b] = tr;
          xi[b] = ti;
        } else if (m == 8) {  // * (-i)
          xr[b] = ti;
          xi[b] = -tr;
        } else {
          float c, s;
          tw32(m, c, s);
          xr[b] = tr * c + ti * s;
          xi[b] = ti * c - tr * s;
        }
      }
    }
  }
}

constexpr int kFft = 2048;
constexpr int kHalf = 1024;
constexpr int kScratchF2 = 32 * 33;  // padded 32x32 complex transpose buffer per warp

template <int FRAMES_PER_CTA, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 2)
logmel2048_kernel(const float* __restrict__ audio, long long audio_stride, int n_samples, int hop,
                  const int* __restrict__ n_valid_frames, int T, const float* __restrict__ window,
                  const float2* __restrict__ tw1024, const float2* __restrict__ rtw,
                  const int* __restrict__ mel_bin0, const float* __restrict__ mel_wpad, int mel_taps, int mel_in_smem,
                  int n_mel, float log_eps, float* __restrict__ out) {
  // Every lookup table lives in shared memory: with ~100 KB of it carved out per CTA the L1 that is left
  // (~20 KB) cannot hold the 40 KB of twiddle / mel tables, and their loads would each pay an L2 round trip.
  extern __shared__ __align__(16) float smem[];
  const int chunk = (FRAMES_PER_CTA - 1) * hop + kFft;     // samples staged per CTA
  const int chunk_pad = (chunk + 3) & ~3;
  float* s_audio = smem;                                   // [chunk_pad]
  float* s_win = s_audio + chunk_pad;                      // [2048]
  float2* s_tw = reinterpret_cast<float2*>(s_win + kFft);  // [32][32]  W_1024^(lane*k1)
  float2* s_rtw = s_tw + 1024;                             // [1024]    W_2048^k
  float2* s_scratch = s_rtw + 1024;                        // [WARPS][32*33]
  int* s_bin0 = reinterpret_cast<int*>(s_scratch + WARPS * kScratchF2);   // [n_mel]
  float* s_melw = reinterpret_cast<float*>(s_bin0 + ((n_mel + 3) & ~3));  // [mel_taps][n_mel] (if it fits)

  const int seg = blockIdx.y;
  const int t0 = blockIdx.x * FRAMES_PER_CTA;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  constexpr int NTHR = WARPS * 32;

  const float* a = audio + (long long)seg * audio_stride;
  const long long s0 = (long long)t0 * hop;
  for (int i = tid; i < chunk; i += NTHR) {
    const long long g = s0 + i;
    s_audio[i] = (g < n_samples) ? __ldg(a + g) : 0.f;   // pad_end=True zeros
  }
  for (int i = tid; i < kFft; i += NTHR) s_win[i] = __ldg(window + i);
  for (int i = tid; i < 1024; i += NTHR) {
    s_tw[i] = __ldg(tw1024 + i);
    s_rtw[i] = __ldg(rtw + i);
  }
  for (int i = tid; i < n_mel; i += NTHR) s_bin0[i] = __ldg(mel_bin0 + i);
  if (mel_in_smem)
    for (int i = tid; i < mel_taps * n_mel; i += NTHR) s_melw[i] = __ldg(mel_wpad + i);
  __syncthreads();
  const float* melw = mel_in_smem ? s_melw : mel_wpad;

  const int n_valid = n_valid_frames ? n_valid_frames[seg] : T;
  float2* scratch = s_scratch + warp * kScratchF2;
  float* mag = reinterpret_cast<float*>(scratch);          // reused: [1025] magnitudes

  for (int f = warp; f < FRAMES_PER_CTA; f += WARPS) {
    const int t = t0 + f;
    if (t >= T) break;
    float* orow = out + ((long long)seg * T + t) * n_mel;
    if (t >= n_valid) {                                    // feature-converter zero padding
      for (int m = lane; m < n_mel; m += 32) orow[m] = 0.f;
      continue;
    }
    float xr[32], xi[32];
    {
      const float2* fa = reinterpret_cast<const float2*>(s_audio + f * hop);
      const float2* fw = reinterpret_cast<const float2*>(s_win);
#pragma unroll
      for (int n1 = 0; n1 < 32; ++n1) {
        const float2 v = fa[32 * n1 + lane];
        const float2 w = fw[32 * n1 + lane];
        xr[n1] = v.x * w.x;
        xi[n1] = v.y * w.y;
      }
    }
    fft32(xr, xi);   // over n1: x[r] = A[k1 = brev5(r)] for n2 = lane
#pragma unroll
    for (int r = 0; r < 32; ++r) {
      const int k1 = brev5(r);
      float vr = xr[r], vi = xi[r];
      if (k1 != 0) {
        const float2 w = s_tw[k1 * 32 + lane];
        const float nr = vr * w.x - vi * w.y;
        vi = vr * w.y + vi * w.x;
        vr = nr;
      }
      scratch[k1 * 33 + lane] = make_float2(vr, vi);
    }
    __syncwarp();
#pragma unroll
    for (int n2 = 0; n2 < 32; ++n2) {
      const float2 v = scratch[lane * 33 + n2];
      xr[n2] = v.x;
      xi[n2] = v.y;
    }
    __syncwarp();
    fft32(xr, xi);   // over n2: x[r] = Z[lane + 32 * brev5(r)]

    // untangle: X[k] = E[k] + W_2048^k O[k], E = (Z[k] + conj Z[N-k]) / 2, O = (Z[k] - conj Z[N-k]) / (2i)
    const int partner = (32 - lane) & 31;
#pragma unroll
    for (int r = 0; r < 32; ++r) {
      const int k2 = brev5(r);
      const int r0 = brev5((32 - k2) & 31);   // what lane 0 must publish (Z[32 (32-k2)])
      const float pr = (lane == 0) ? xr[r0] : xr[31 - r];
      const float pi = (lane == 0) ? xi[r0] : xi[31 - r];
      const float qr = __shfl_sync(0xffffffffu, pr, partner);
      const float qi = __shfl_sync(0xffffffffu, pi, partner);
      const float zr = xr[r], zi = xi[r];
      const int k = lane + 32 * k2;
      const float er = 0.5f * (zr + qr), ei = 0.5f * (zi - qi);
      const float orr = 0.5f * (zi + qi), oi = -0.5f * (zr - qr);
      const float2 w = s_rtw[k];
      const float Xr = er + (w.x * orr - w.y * oi);
      const float Xi = ei + (w.x * oi + w.y * orr);
      mag[k] = sqrtf(Xr * Xr + Xi * Xi);
      if (r == 0 && lane == 0) mag[kHalf] = fabsf(zr - zi);   // Nyquist bin
    }
    __syncwarp();
    // banded mel: every mel bin reads the same number of taps (zero-padded), ascending FFT bin order;
    // weights are laid out [tap][mel] so that a warp's reads are consecutive.
    for (int m = lane; m < n_mel; m += 32) {
      const float* mg = mag + s_bin0[m];
      float acc = 0.f;
#pragma unroll 5
      for (int j = 0; j < mel_taps; ++j) acc = fmaf(mg[j], melw[j * n_mel + m], acc);
      orow[m] = logf(acc <= 0.f ? log_eps : acc);      // safe_log: replace, not add
    }
    __syncwarp();
  }
}


// ---------------------------------------------------------------------------------------------
// The same warp-per-frame scheme for FFT sizes 1024 and 4096 (BASELINE configs[3] sweeps 1024 / 2048 / 4096 at hop 128; the
// reference itself only ever uses 2048).  A real FFT of size 64 R is a complex FFT of NC = 32 R points, R in {16, 64}:
//   stage 1   lane n2 holds z[32 n1 + n2], n1 < R, and runs an R-point radix-2 DIF FFT in registers (twiddles are
//             immediates from a constant table), multiplies by W_NC^(n2 k1);
//   transpose through a padded [R][33] shared-memory tile;
//   stage 2   lane k1 (and k1 + 32 for R = 64; only 16 lanes for R = 16) runs the 32-point in-register FFT over n2 and
//             writes Z[k1 + R k2] to a linear shared-memory array;
//   untangle  X[k] = E[k] + W_N^k O[k] from Z[k] and Z[NC - k] read back from shared memory, magnitudes, banded mel, log.
// ---------------------------------------------------------------------------------------------
__constant__ float2 kTw64[32] = {{1.f, 0.f}, {0.99518472667219693f, 0.098017140329560604f}, {0.98078528040323043f, 0.19509032201612825f}, {0.95694033573220882f, 0.29028467725446233f}, {0.92387953251128674f, 0.38268343236508978f}, {0.88192126434835505f, 0.47139673682599764f}, {0.83146961230254524f, 0.55557023301960218f}, {0.77301045336273699f, 0.63439328416364549f}, {0.70710678118654757f, 0.70710678118654746f}, {0.63439328416364549f, 0.77301045336273699f}, {0.55557023301960229f, 0.83146961230254524f}, {0.47139673682599781f, 0.88192126434835494f}, {0.38268343236508984f, 0.92387953251128674f}, {0.29028467725446233f, 0.95694033573220894f}, {0.19509032201612833f, 0.98078528040323043f}, {0.09801714032956077f, 0.99518472667219682f}, {0.f, 1.f}, {-0.098017140329560645f, 0.99518472667219693f}, {-0.19509032201612819f, 0.98078528040323043f}, {-0.29028467725446216f, 0.95694033573220894f}, {-0.38268343236508973f, 0.92387953251128674f}, {-0.4713967368259977f, 0.88192126434835505f}, {-0.55557023301960196f, 0.83146961230254546f}, {-0.63439328416364538f, 0.7730104533627371f}, {-0.70710678118654746f, 0.70710678118654757f}, {-0.77301045336273699f, 0.63439328416364549f}, {-0.83146961230254535f, 0.55557023301960218f}, {-0.88192126434835494f, 0.47139673682599786f}, {-0.92387953251128674f, 0.38268343236508989f}, {-0.95694033573220882f, 0.29028467725446239f}, {-0.98078528040323043f, 0.19509032201612861f}, {-0.99518472667219682f, 0.098017140329560826f}};        // (cos, sin)(2 pi m / 64)

template <int R> __host__ __device__ constexpr int brev_r(int r) {
  int o = 0;
  for (int b = 1, t = R >> 1; b < R; b <<= 1, t >>= 1)
    if (r & b) o |= t;
  return o;
}

// In-register R-point forward FFT, radix-2 decimation in frequency; output bit-reversed: x[r] holds X[brev_r<R>(r)].
template <int R>
__device__ __forceinline__ void fft_reg(float (&xr)[R], float (&xi)[R]) {
#pragma unroll
  for (int span = R / 2; span >= 1; span >>= 1) {
#pragma unroll
    for (int a = 0; a < R; ++a) {
      if ((a & span) == 0) {
        const int b = a + span;
        const int m = (a & (span - 1)) * (R / 2 / span);          // W_R^m
        const float tr = xr[a] - xr[b];
        const float ti = xi[a] - xi[b];
        xr[a] += xr[b];
        xi[a] += xi[b];
        if (m == 0) {
          xr[b] = tr;
          xi[b] = ti;
        } else if (m == R / 4) {  // * (-i)
          xr[b] = ti;
          xi[b] = -tr;
        } else {
          const float c = kTw64[m * (64 / R)].x, sn = kTw64[m * (64 / R)].y;
          xr[b] = tr * c + ti * sn;
          xi[b] = ti * c - tr * sn;
        }
      }
    }
  }
}

template <int R, int FRAMES_PER_CTA, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
logmel_r_kernel(const float* __restrict__ audio, long long audio_stride, int n_samples, int hop,
                const int* __restrict__ n_valid_frames, int T, const float* __restrict__ window,
                const float2* __restrict__ tw_nc, const float2* __restrict__ rtw, const int* __restrict__ mel_lo,
                const int* __restrict__ mel_off, const float* __restrict__ mel_csr, int mel_nnz, int n_mel, float log_eps,
                float* __restrict__ out) {
  constexpr int NC = 32 * R, FFT = 2 * NC;
  constexpr int J = (R + 31) / 32;                         // stage-2 passes per lane
  constexpr int kT = R * 33;                               // transpose tile (float2)
  constexpr int kScr = kT + NC;                            // per-warp scratch (float2): tile + linear Z
  extern __shared__ __align__(16) float smem[];
  const int chunk = (FRAMES_PER_CTA - 1) * hop + FFT;
  const int chunk_pad = (chunk + 3) & ~3;
  float* s_audio = smem;                                   // [chunk_pad]
  float* s_win = s_audio + chunk_pad;                      // [FFT]
  float2* s_tw = reinterpret_cast<float2*>(s_win + FFT);   // [R][32]  W_NC^(lane*k1)
  float2* s_rtw = s_tw + R * 32;                           // [NC]     W_FFT^k
  float2* s_scratch = s_rtw + NC;                          // [WARPS][kScr]
  // mel filterbank in compact CSR form (the fixed-tap padded band of the 2048 kernel would be 80 KB at FFT 4096)
  int* s_lo = reinterpret_cast<int*>(s_scratch + WARPS * kScr);            // [n_mel] first FFT bin
  int* s_off = s_lo + ((n_mel + 3) & ~3);                                  // [n_mel + 1]
  float* s_csr = reinterpret_cast<float*>(s_off + ((n_mel + 4) & ~3));     // [mel_nnz]

  const int seg = blockIdx.y;
  const int t0 = blockIdx.x * FRAMES_PER_CTA;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  constexpr int NTHR = WARPS * 32;

  const float* a = audio + (long long)seg * audio_stride;
  const long long s0 = (long long)t0 * hop;
  for (int i = tid; i < chunk; i += NTHR) {
    const long long g = s0 + i;
    s_audio[i] = (g < n_samples) ? __ldg(a + g) : 0.f;   // pad_end=True zeros
  }
  for (int i = tid; i < FFT; i += NTHR) s_win[i] = __ldg(window + i);
  for (int i = tid; i < R * 32; i += NTHR) s_tw[i] = __ldg(tw_nc + i);
  for (int i = tid; i < NC; i += NTHR) s_rtw[i] = __ldg(rtw + i);
  for (int i = tid; i < n_mel; i += NTHR) s_lo[i] = __ldg(mel_lo + i);
  for (int i = tid; i <= n_mel; i += NTHR) s_off[i] = __ldg(mel_off + i);
  for (int i = tid; i < mel_nnz; i += NTHR) s_csr[i] = __ldg(mel_csr + i);
  __syncthreads();

  const int n_valid = n_valid_frames ? n_valid_frames[seg] : T;
  float2* tile = s_scratch + warp * kScr;                  // [R][33]
  float2* zs = tile + kT;                                  // [NC] Z in natural order
  float* mag = reinterpret_cast<float*>(tile);             // reused after stage 2: [NC + 1] magnitudes (NC + 1 <= 2 kT)

  for (int f = warp; f < FRAMES_PER_CTA; f += WARPS) {
    const int t = t0 + f;
    if (t >= T) break;
    float* orow = out + ((long long)seg * T + t) * n_mel;
    if (t >= n_valid) {                                    // feature-converter zero padding
      for (int m = lane; m < n_mel; m += 32) orow[m] = 0.f;
      continue;
    }
    {
      float xr[R], xi[R];
      const float2* fa = reinterpret_cast<const float2*>(s_audio + f * hop);
      const float2* fw = reinterpret_cast<const float2*>(s_win);
#pragma unroll
      for (int n1 = 0; n1 < R; ++n1) {
        const float2 v = fa[32 * n1 + lane];
        const float2 w = fw[32 * n1 + lane];
        xr[n1] = v.x * w.x;
        xi[n1] = v.y * w.y;
      }
      fft_reg<R>(xr, xi);   // over n1: x[r] = A[k1 = brev_r(r)] for n2 = lane
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int k1 = brev_r<R>(r);
        float vr = xr[r], vi = xi[r];
        if (k1 != 0) {
          const float2 w = s_tw[k1 * 32 + lane];
          const float nr = vr * w.x - vi * w.y;
          vi = vr * w.y + vi * w.x;
          vr = nr;
        }
        tile[k1 * 33 + lane] = make_float2(vr, vi);
      }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int k1 = lane + 32 * j;
      if (k1 < R) {
        float xr[32], xi[32];
#pragma unroll
        for (int n2 = 0; n2 < 32; ++n2) {
          const float2 v = tile[k1 * 33 + n2];
          xr[n2] = v.x;
          xi[n2] = v.y;
        }
        fft32(xr, xi);   // over n2: x[r] = Z[k1 + R * brev5(r)]
#pragma unroll
        for (int r = 0; r < 32; ++r) zs[k1 + R * brev5(r)] = make_float2(xr[r], xi[r]);
      }
    }
    __syncwarp();
    // untangle: X[k] = E[k] + W_FFT^k O[k], E = (Z[k] + conj Z[NC-k]) / 2, O = (Z[k] - conj Z[NC-k]) / (2i)
    for (int k = lane; k < NC; k += 32) {
      const float2 zk = zs[k];
      if (k == 0) {
        mag[0] = fabsf(zk.x + zk.y);
        mag[NC] = fabsf(zk.x - zk.y);                      // Nyquist bin
        continue;
      }
      const float2 zq = zs[NC - k];
      const float er = 0.5f * (zk.x + zq.x), ei = 0.5f * (zk.y - zq.y);
      const float orr = 0.5f * (zk.y + zq.y), oi = -0.5f * (zk.x - zq.x);
      const float2 w = s_rtw[k];
      const float Xr = er + (w.x * orr - w.y * oi);
      const float Xi = ei + (w.x * oi + w.y * orr);
      mag[k] = sqrtf(Xr * Xr + Xi * Xi);
    }
    __syncwarp();
    for (int m = lane; m < n_mel; m += 32) {           // ascending FFT bin order, like the padded band
      const float* mg = mag + s_lo[m];
      const float* w = s_csr + s_off[m];
      const int cnt = s_off[m + 1] - s_off[m];
      float acc = 0.f;
      for (int j = 0; j < cnt; ++j) acc = fmaf(mg[j], w[j], acc);
      orow[m] = logf(acc <= 0.f ? log_eps : acc);      // safe_log: replace, not add
    }
    __syncwarp();
  }
}

// Any OTHER power-of-two FFT size (BASELINE configs[3] sweeps 1024 / 2048 / 4096, which have the kernels above; the reference
// itself only ever uses 2048, spectrograms.py:27-28).  Same arithmetic contract, plain structure: one CTA per frame,
// real FFT of size N as a complex radix-2 DIF FFT of size N/2 in shared memory (output bit-reversed, read back through
// the bit-reversed index), untangle, magnitude, banded mel, safe log.  Tables (window, W_N^k) come from global memory.
template <int NTHR>
__global__ void __launch_bounds__(NTHR)
logmel_pow2_kernel(const float* __restrict__ audio, long long audio_stride, int n_samples, int hop, int fft, int log2_nc,
                   const int* __restrict__ n_valid_frames, int T, const float* __restrict__ window,
                   const float2* __restrict__ rtw, const int* __restrict__ mel_bin0, const float* __restrict__ mel_wpad,
                   int mel_taps, int n_mel, float log_eps, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  const int nc = fft >> 1;
  float2* z = reinterpret_cast<float2*>(smem);             // [nc]
  float* mag = smem + 2 * nc;                              // [nc + 1]
  const int seg = blockIdx.y, t = blockIdx.x, tid = threadIdx.x;
  float* orow = out + ((long long)seg * T + t) * n_mel;
  const int n_valid = n_valid_frames ? n_valid_frames[seg] : T;
  if (t >= n_valid) {                                      // feature-converter zero padding
    for (int m = tid; m < n_mel; m += NTHR) orow[m] = 0.f;
    return;
  }
  const float* a = audio + (long long)seg * audio_stride;
  const long long s0 = (long long)t * hop;
  for (int n = tid; n < nc; n += NTHR) {
    const long long g = s0 + 2 * n;
    const float x0 = (g < n_samples) ? __ldg(a + g) : 0.f;             // pad_end=True zeros
    const float x1 = (g + 1 < n_samples) ? __ldg(a + g + 1) : 0.f;
    z[n] = make_float2(x0 * __ldg(window + 2 * n), x1 * __ldg(window + 2 * n + 1));
  }
  __syncthreads();
  // radix-2 decimation in frequency: stage with half-span h: (a, b) -> (a + b, (a - b) W_nc^(j * nc / (2h)))
  for (int h = nc >> 1; h >= 1; h >>= 1) {
    const int tw_step = (nc / (2 * h)) * 2;                // W_nc^m = W_fft^(2m): index into rtw (W_fft^k, k < fft/2)
    for (int i = tid; i < (nc >> 1); i += NTHR) {
      const int j = i & (h - 1);
      const int ia = ((i - j) << 1) + j, ib = ia + h;
      const float2 va = z[ia], vb = z[ib];
      const float dr = va.x - vb.x, di = va.y - vb.y;
      const float2 w = __ldg(rtw + j * tw_step);
      z[ia] = make_float2(va.x + vb.x, va.y + vb.y);
      z[ib] = make_float2(dr * w.x - di * w.y, dr * w.y + di * w.x);
    }
    __syncthreads();
  }
  // untangle: X[k] = E[k] + W_fft^k O[k], E = (Z[k] + conj Z[nc-k]) / 2, O = (Z[k] - conj Z[nc-k]) / (2i); Z[k] = z[brev(k)]
  const int shift = 32 - log2_nc;
  for (int k = tid; k <= nc; k += NTHR) {
    if (k == 0 || k == nc) {
      const float2 z0 = z[0];
      mag[k] = (k == 0) ? fabsf(z0.x + z0.y) : fabsf(z0.x - z0.y);
      continue;
    }
    const float2 zk = z[__brev((unsigned)k) >> shift];
    const float2 zq = z[__brev((unsigned)(nc - k)) >> shift];
    const float er = 0.5f * (zk.x + zq.x), ei = 0.5f * (zk.y - zq.y);
    const float orr = 0.5f * (zk.y + zq.y), oi = -0.5f * (zk.x - zq.x);
    const float2 w = __ldg(rtw + k);
    const float Xr = er + (w.x * orr - w.y * oi);
    const float Xi = ei + (w.x * oi + w.y * orr);
    mag[k] = sqrtf(Xr * Xr + Xi * Xi);
  }
  __syncthreads();
  for (int m = tid; m < n_mel; m += NTHR) {
    const float* mg = mag + __ldg(mel_bin0 + m);
    float acc = 0.f;
    for (int j = 0; j < mel_taps; ++j) acc = fmaf(mg[j], __ldg(mel_wpad + j * n_mel + m), acc);
    orow[m] = logf(acc <= 0.f ? log_eps : acc);            // safe_log: replace, not add
  }
}

}  // namespace

}  // namespace mt3

using namespace mt3;

extern "C" int mt3_frontend_create(const mt3_frontend_config* cfg, const float* mel_matrix, mt3_frontend** out) {
  MT3_REQUIRE(cfg && mel_matrix && out, MT3_ERR_BAD_ARG, "mt3_frontend_create: null argument");
  const int fft = cfg->fft_size;
  MT3_REQUIRE(fft >= 64 && fft <= 16384 && (fft & (fft - 1)) == 0, MT3_ERR_UNSUPPORTED,
              "mt3_frontend_create: fft_size %d unsupported (power of two in [64, 16384]; the reference fixes 2048, "
              "spectrograms.py:27-28)", fft);
  MT3_REQUIRE(cfg->hop_width > 0 && cfg->hop_width % 2 == 0 && cfg->hop_width <= fft, MT3_ERR_BAD_ARG,
              "mt3_frontend_create: hop_width %d must be even and in (0, %d]", cfg->hop_width, fft);
  MT3_REQUIRE(cfg->num_mel_bins > 0 && cfg->sample_rate > 0, MT3_ERR_BAD_ARG, "mt3_frontend_create: bad sizes");
  Frontend* fe = new Frontend();
  fe->cfg = *cfg;
  fe->n_bins = cfg->fft_size / 2 + 1;
  const int n_mel = cfg->num_mel_bins;

  std::vector<float> win(fft);
  for (int i = 0; i < fft; ++i) win[i] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / fft));  // periodic Hann
  std::vector<float2> tw(32 * 32), rt(fft / 2);
  for (int k1 = 0; k1 < 32; ++k1)
    for (int l = 0; l < 32; ++l) {
      const double th = -2.0 * M_PI * (double)(k1 * l) / 1024.0;
      tw[k1 * 32 + l] = make_float2((float)cos(th), (float)sin(th));
    }
  for (int k = 0; k < fft / 2; ++k) {                       // W_fft^k
    const double th = -2.0 * M_PI * (double)k / (double)fft;
    rt[k] = make_float2((float)cos(th), (float)sin(th));
  }
  // banded form of the [n_bins, n_mel] matrix: per mel bin the contiguous span of non-zero FFT bins, padded
  // with zeros to a common width `taps` (window start clamped so that it stays inside the spectrum)
  std::vector<int> lo(n_mel, -1), hi(n_mel, -1), bin0(n_mel, 0);
  int taps = 1, nnz = 0;
  for (int m = 0; m < n_mel; ++m) {
    for (int b = 0; b < fe->n_bins; ++b)
      if (mel_matrix[(size_t)b * n_mel + m] != 0.f) {
        if (lo[m] < 0) lo[m] = b;
        hi[m] = b;
        ++nnz;
      }
    if (lo[m] >= 0) taps = std::max(taps, hi[m] - lo[m] + 1);
  }
  std::vector<float> w((size_t)taps * n_mel, 0.f);
  for (int m = 0; m < n_mel; ++m) {
    if (lo[m] < 0) continue;
    bin0[m] = std::min(lo[m], fe->n_bins - taps);
    for (int j = 0; j < taps; ++j) w[(size_t)j * n_mel + m] = mel_matrix[(size_t)(bin0[m] + j) * n_mel + m];
  }
  fe->taps = taps;
  fe->nnz = nnz;
  // compact form: per mel bin the span [lo, hi] only
  std::vector<int> off(n_mel + 1, 0), lo0(n_mel, 0);
  std::vector<float> csr;
  for (int m = 0; m < n_mel; ++m) {
    off[m] = (int)csr.size();
    if (lo[m] >= 0) {
      lo0[m] = lo[m];
      for (int b = lo[m]; b <= hi[m]; ++b) csr.push_back(mel_matrix[(size_t)b * n_mel + m]);
    }
  }
  off[n_mel] = (int)csr.size();
  if (csr.empty()) csr.push_back(0.f);

#define FE_ALLOC_COPY(dst, vec)                                                            \
  MT3_CUDA_CHECK(cudaMalloc((void**)&(dst), (vec).size() * sizeof((vec)[0])));            \
  MT3_CUDA_CHECK(cudaMemcpy((dst), (vec).data(), (vec).size() * sizeof((vec)[0]), cudaMemcpyHostToDevice))
  FE_ALLOC_COPY(fe->d_window, win);
  FE_ALLOC_COPY(fe->d_tw1024, tw);
  FE_ALLOC_COPY(fe->d_rtw, rt);
  if (fft == 1024 || fft == 4096) {
    const int R = fft / 64, NC = fft / 2;
    std::vector<float2> twn((size_t)R * 32);
    for (int k1 = 0; k1 < R; ++k1)
      for (int l = 0; l < 32; ++l) {
        const double th = -2.0 * M_PI * (double)(k1 * l) / (double)NC;
        twn[(size_t)k1 * 32 + l] = make_float2((float)cos(th), (float)sin(th));
      }
    FE_ALLOC_COPY(fe->d_tw_nc, twn);
  }
  FE_ALLOC_COPY(fe->d_mel_bin0, bin0);
  FE_ALLOC_COPY(fe->d_mel_w, w);
  FE_ALLOC_COPY(fe->d_mel_off, off);
  FE_ALLOC_COPY(fe->d_mel_csr, csr);
  FE_ALLOC_COPY(fe->d_mel_lo, lo0);
  fe->csr_len = off[n_mel];
#undef FE_ALLOC_COPY
  *out = reinterpret_cast<mt3_frontend*>(fe);
  return MT3_OK;
}

extern "C" int mt3_frontend_destroy(mt3_frontend* h) {
  if (!h) return MT3_OK;
  Frontend* fe = reinterpret_cast<Frontend*>(h);
  cudaFree(fe->d_window);
  cudaFree(fe->d_tw1024);
  cudaFree(fe->d_tw_nc);
  cudaFree(fe->d_mel_off);
  cudaFree(fe->d_mel_csr);
  cudaFree(fe->d_mel_lo);
  cudaFree(fe->d_rtw);
  cudaFree(fe->d_mel_bin0);
  cudaFree(fe->d_mel_w);
  delete fe;
  return MT3_OK;
}

extern "C" int mt3_frontend_num_frames(const mt3_frontend* h, int64_t n_samples) {
  if (!h || n_samples < 0) return fail(MT3_ERR_BAD_ARG, "mt3_frontend_num_frames: bad argument");
  const Frontend* fe = reinterpret_cast<const Frontend*>(h);
  return (int)((n_samples + fe->cfg.hop_width - 1) / fe->cfg.hop_width);
}

extern "C" int mt3_logmel_f32(const mt3_frontend* h, const float* audio, int64_t audio_stride, int32_t num_segments,
                              int32_t n_samples, const int32_t* n_valid_frames, float* out, void* stream) {
  MT3_REQUIRE(h && out, MT3_ERR_BAD_ARG, "mt3_logmel_f32: null handle/output");
  MT3_REQUIRE(num_segments >= 0 && n_samples >= 0, MT3_ERR_BAD_ARG, "mt3_logmel_f32: negative size");
  if (num_segments == 0 || n_samples == 0) return MT3_OK;  // empty input -> zero frames (tf.signal.frame)
  MT3_REQUIRE(audio, MT3_ERR_BAD_ARG, "mt3_logmel_f32: null audio");
  MT3_REQUIRE(audio_stride >= n_samples, MT3_ERR_SHAPE, "mt3_logmel_f32: audio_stride %lld < n_samples %d",
              (long long)audio_stride, n_samples);
  MT3_REQUIRE(num_segments <= 65535, MT3_ERR_SHAPE, "mt3_logmel_f32: more than 65535 segments per call");
  const Frontend* fe = reinterpret_cast<const Frontend*>(h);
  const int hop = fe->cfg.hop_width;
  const int T = (n_samples + hop - 1) / hop;
  if ((fe->cfg.fft_size == 1024 || fe->cfg.fft_size == 4096) && fe->d_tw_nc) {
    // warp-per-frame kernels for the other two sizes of BASELINE configs[3]
    const int fft = fe->cfg.fft_size, n_mel = fe->cfg.num_mel_bins;
    auto launch_r = [&](auto kern, int R, int F, int W) -> int {
      const int NC = 32 * R;
      const int chunk = (F - 1) * hop + fft;
      const size_t smem = (size_t)(((chunk + 3) & ~3) + fft) * sizeof(float) + (size_t)(R * 32 + NC) * sizeof(float2) +
                          (size_t)W * (R * 33 + NC) * sizeof(float2) + (size_t)(((n_mel + 3) & ~3) + ((n_mel + 4) & ~3)) * sizeof(int) +
                          (size_t)fe->csr_len * sizeof(float);
      MT3_REQUIRE(smem <= 227 * 1024, MT3_ERR_UNSUPPORTED, "mt3_logmel_f32: hop %d needs %zu B of shared memory", hop, smem);
      MT3_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      dim3 grid((T + F - 1) / F, num_segments);
      kern<<<grid, W * 32, smem, (cudaStream_t)stream>>>(audio, audio_stride, n_samples, hop, n_valid_frames, T, fe->d_window,
                                                         fe->d_tw_nc, fe->d_rtw, fe->d_mel_lo, fe->d_mel_off, fe->d_mel_csr, fe->csr_len,
                                                         n_mel, fe->cfg.log_eps, out);
      return MT3_OK;
    };
    const int rc = fft == 1024 ? launch_r(logmel_r_kernel<16, 16, 8>, 16, 16, 8) : launch_r(logmel_r_kernel<64, 8, 4>, 64, 8, 4);
    if (rc != MT3_OK) return rc;
    MT3_LAUNCH_CHECK();
    return MT3_OK;
  }
  if (fe->cfg.fft_size != kFft) {
    const int fft = fe->cfg.fft_size, nc = fft / 2;
    int log2_nc = 0;
    while ((1 << log2_nc) < nc) ++log2_nc;
    constexpr int NT = 256;
    const size_t smem_g = (size_t)(2 * nc + nc + 4) * sizeof(float);
    static bool attr_g = false;
    if (!attr_g) {
      MT3_CUDA_CHECK(cudaFuncSetAttribute(logmel_pow2_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      attr_g = true;
    }
    MT3_REQUIRE(T <= 2147483647 / 2 && smem_g <= 200 * 1024, MT3_ERR_UNSUPPORTED, "mt3_logmel_f32: fft %d too large", fft);
    logmel_pow2_kernel<NT><<<dim3(T, num_segments), NT, smem_g, (cudaStream_t)stream>>>(
        audio, audio_stride, n_samples, hop, fft, log2_nc, n_valid_frames, T, fe->d_window, fe->d_rtw, fe->d_mel_bin0, fe->d_mel_w,
        fe->taps, fe->cfg.num_mel_bins, fe->cfg.log_eps, out);
    MT3_LAUNCH_CHECK();
    return MT3_OK;
  }
  // 12 frames per CTA on 6 warps (~111 KB of smem incl. all tables, two CTAs per SM = 12 warps per SM, 168 registers per
  // thread): 134 us per 64 segments (the earlier 16 frames on 4 warps: 175 us)
  static bool attr_set = false;
  const int n_mel = fe->cfg.num_mel_bins;
  auto launch = [&](auto kern, int F, int W) -> int {
    const int chunk = (F - 1) * hop + kFft;
    const size_t base = (size_t)(((chunk + 3) & ~3) + kFft) * sizeof(float) + 2 * 1024 * sizeof(float2) +
                        (size_t)W * kScratchF2 * sizeof(float2) + (size_t)((n_mel + 3) & ~3) * sizeof(int);
    const size_t mel_bytes = (size_t)fe->taps * n_mel * sizeof(float);
    const int mel_in_smem = base + mel_bytes <= 113 * 1024;
    const size_t smem = base + (mel_in_smem ? mel_bytes : 0);
    MT3_REQUIRE(smem <= 227 * 1024, MT3_ERR_UNSUPPORTED, "mt3_logmel_f32: hop %d needs %zu B of shared memory", hop, smem);
    if (!attr_set) {
      MT3_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set = true;
    }
    dim3 grid((T + F - 1) / F, num_segments);
    kern<<<grid, W * 32, smem, (cudaStream_t)stream>>>(audio, audio_stride, n_samples, hop, n_valid_frames, T, fe->d_window,
                                                       fe->d_tw1024, fe->d_rtw, fe->d_mel_bin0, fe->d_mel_w, fe->taps,
                                                       mel_in_smem, n_mel, fe->cfg.log_eps, out);
    return MT3_OK;
  };
  const int rc = launch(logmel2048_kernel<12, 6>, 12, 6);
  if (rc != MT3_OK) return rc;
  MT3_LAUNCH_CHECK();
  return MT3_OK;
}
