"""The log-mel frontend kernels (K1, mt3_b200/csrc/logmel.cu) run alone through `mt3_frontend_create` / `mt3_logmel_f32`
with hand-built float32 mel matrices, against a float64 numpy restatement of exactly what the kernel consumes:

  float32 audio, framed as tf.signal.frame(pad_end=True) does; the float32 periodic Hann window the library builds,
  (float)(0.5 - 0.5 cos(2 pi i / N)); |rfft| in float64; the float32 mel matrix cast to float64;
  log(where(x <= 0, eps, x)); rows >= n_valid_frames[s] written as +0.0.

Every case names the kernel and branch it reaches (`kernel_path` restates the launcher's choice, and a CPU test pins each
case to its branch):
  2048/smem    logmel2048_kernel, the padded mel band staged in shared memory
  2048/global  logmel2048_kernel, the band read from global memory (base + band > 113 KB)
  r16, r64     logmel_r_kernel<16, ...> (FFT 1024) and logmel_r_kernel<64, ...> (FFT 4096), compact CSR band
  pow2         logmel_pow2_kernel (FFT 64, 128, 256, 512, 8192, 16384)

Bars (u = 2^-24), per element, derived from the arithmetic:
  FFT bin b of frame t   bar_b = tol * u * (log2 N * |X_b| + sqrt(N) * ||xw_t||_2) + 2^-75
                         the first term is the relative error a radix-2 fp32 FFT carries on a loud bin.  The second is the
                         floor every bin of the frame carries: sqrt(N) ||xw_t|| = ||X_t||_2 (Parseval; xw_t is the frame's
                         windowed samples) is the scale of the FFT's norm-wise error bound, and one bin can hold that
                         much: on a tone the rounding of the large intermediates lands coherently in the quiet bins
                         (measured 0.5 - 0.9 u ||X_t|| at every N; a floor of u ||xw_t|| fails tones by up to 55x).  The
                         last term is the rounding of Xr^2 + Xi^2 when it is subnormal (<= 2^-150, which moves |X| by
                         <= 2^-75): a zero crossing of a cosine under the window's first taps gets there
  mel bin m (linear)     sum_b |W_bm| bar_b  +  n_fma * u * sum_b |W_bm X_b|  +  mel (|ln mel| + 1) 2u
                         (the FMA chain over the band: n_fma = the padded tap count at 2048 / pow2, the column's CSR length
                         at 1024 / 4096; then the rounding of logf and of its result)
  exact zeros            where the exact mel is 0 because every term of it is (all-zero frames, empty columns), the
                         output must be logf(eps) to within 1 ulp, with eps the configured log_eps
  negative mel           an output of logf(eps) is accepted when the exact mel is below its bar (the kernel's sum may have
                         been <= 0); where the exact mel is negative by more than its bar, anything else fails.
The comparison is made in the linear domain: |exp(got) - mel| against the bar.  Every output must be finite.

Audio rows sit `audio_stride > n_samples` apart with NaN in every gap and after the last row, so a frame that read past
its segment would produce NaN; the output buffer is surrounded by NaN guards that must stay NaN; and every launch is
repeated and must be bit-identical.

`tol` per kernel is set from a measurement on an H100 80GB HBM3 at a 700 W power limit.  The worst err/bar of each case
at that tol is in the comments of CASES and in the docstrings below: 0.42 (logmel2048_kernel), 0.48 (logmel_r_kernel) and
0.41 (logmel_pow2_kernel) at worst, so every bar sits within 10x of its kernel's worst measured ratio.  Cases that measure
far below that (HTK bands over quiet bins, one-frame segments) share their kernel's bar rather than get one of their own.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse

from oracle import mt3_oracle as O

U = 2.0 ** -24
SUBNORMAL = 2.0 ** -75          # sqrt of half the smallest subnormal float
EPS = 1e-5                      # the library's default log_eps (spectral_ops.compute_logmel)


def log_eps(eps):
    """What logf(eps) rounds to, to within 1 ulp."""
    return np.float32(np.log(np.float64(np.float32(eps))))


DEV = "cuda:0"
SR = 16000
# FFT error constant per kernel family (the `tol` of bar_b above).  Worst err/bar at tol = 1 over every case below, on
# an H100 80GB HBM3 at a 700 W power limit: 0.85 (logmel2048_kernel), 0.96 (logmel_r_kernel), 0.83 (logmel_pow2_kernel)
TOL_FFT = {"2048": 2.0, "r": 2.0, "pow2": 2.0}
MEL_BUDGET_2048 = 113 * 1024      # mt3_logmel_f32, `launch`: the 2048 kernel stages its band up to this
SMEM_MAX = 227 * 1024             # mt3_logmel_f32, `launch` and `launch_r`: the shared-memory limit they check


# ------------------------------------------------------------------------------------------------
# the launchers' choices, restated
# ------------------------------------------------------------------------------------------------
def band(W):
    """The banded forms mt3_frontend_create builds (its "banded form" and "compact form"): per column the first and last non-zero FFT bin
    (-1 when the column is empty), the common tap count of the padded band, and the length of the compact CSR band."""
    nz = W != 0
    used = nz.any(axis=0)
    lo = np.where(used, nz.argmax(axis=0), -1)
    hi = np.where(used, W.shape[0] - 1 - nz[::-1].argmax(axis=0), -1)
    width = np.where(used, hi - lo + 1, 0)
    return lo, hi, max(1, int(width.max())), int(width.sum())


def smem_2048(hop, n_mel, taps, frames=12, warps=6):
    """logmel2048_kernel's shared memory (the `launch` lambda in mt3_logmel_f32): the audio span of 12 frames, window, twiddles, 6 warps'
    transpose tiles and the band offsets make up `base`; the padded band [taps][n_mel] is staged too iff
    base + band <= 113 KB, and is read from global memory otherwise.  Returns (base, band) in bytes."""
    chunk = (frames - 1) * hop + 2048
    base = (((chunk + 3) & ~3) + 2048) * 4 + 2 * 1024 * 8 + warps * 32 * 33 * 8 + ((n_mel + 3) & ~3) * 4
    return base, taps * n_mel * 4


def smem_r(fft, hop, n_mel, csr_len):
    """logmel_r_kernel's shared memory (the `launch_r` lambda in mt3_logmel_f32): 16 frames on 8 warps at FFT 1024, 8 frames on 4 warps at
    4096; the CSR band always lives in shared memory, and a launch needing more than 227 KB is MT3_ERR_UNSUPPORTED."""
    R, F, Wp = (16, 16, 8) if fft == 1024 else (64, 8, 4)
    NC = 32 * R
    chunk = (F - 1) * hop + fft
    return ((((chunk + 3) & ~3) + fft) * 4 + (R * 32 + NC) * 8 + Wp * (R * 33 + NC) * 8
            + (((n_mel + 3) & ~3) + ((n_mel + 4) & ~3)) * 4 + csr_len * 4)


def kernel_path(fft, hop, W):
    _, _, taps, csr = band(W)
    n_mel = W.shape[1]
    if fft in (1024, 4096):
        name = "r16" if fft == 1024 else "r64"
        return name if smem_r(fft, hop, n_mel, csr) <= SMEM_MAX else name + "/unsupported"
    if fft != 2048:
        return "pow2"
    base, mel = smem_2048(hop, n_mel, taps)
    return "2048/smem" if base + mel <= MEL_BUDGET_2048 else "2048/global"


# ------------------------------------------------------------------------------------------------
# matrices and signals
# ------------------------------------------------------------------------------------------------
def mat_identity(fft):
    """Every FFT bin is its own column: the output is log|X_k| for k = 0 .. N/2, DC and Nyquist included."""
    return np.eye(fft // 2 + 1, dtype=np.float32)


def mat_htk(fft, hi_hz=7600.0, n_mel=None):
    """The MT3 HTK filterbank (20 Hz - 7600 Hz; zero DC and Nyquist rows), or with hi_hz = 8000 one whose upper edge is
    the Nyquist frequency (its top triangle weighs the bins just below Nyquist; the Nyquist row itself stays zero, the
    crafted matrix puts a weight there)."""
    if n_mel is None:
        n_mel = 512 if fft >= 1024 else 128
    return O.linear_to_mel_weight_matrix(n_mel, fft // 2 + 1, SR, 20.0, hi_hz, np.float32)


def mat_crafted(fft, seed=5):
    """33 columns (not a multiple of 32) built to reach what the HTK matrices never do."""
    nb = fft // 2 + 1
    W = np.zeros((nb, 33), np.float32)
    W[0, 0] = 1.0                                            # only weight at DC
    W[nb - 1, 1] = 1.0                                       # only weight at Nyquist
    c = nb // 4
    W[[c, c + 3, c + 7], 2] = [0.5, 0.25, 0.125]             # interior zeros inside the column's span
    # column 3 stays empty
    W[[0, 1, 2], 4] = [-1.0, 0.5, 0.25]                      # negative weight on the loud DC bin: < 0 on a constant
    W[nb // 3, 5] = 0.7                                      # single bin
    wide = min(40, nb // 2)                                  # the widest column sets the padded tap count ...
    W[5:5 + wide, 6] = 1.0 - np.abs(np.arange(wide) - (wide - 1) / 2) / (wide / 2)
    W[nb - 3:nb - 1, 7] = [0.6, 0.3]                         # ... so this narrow top band's window start is clamped
    rng = np.random.default_rng(seed)
    for m in range(8, 33):
        lo = int(rng.integers(0, nb - 1))
        w = int(rng.integers(1, min(12, nb - lo) + 1))
        W[lo:lo + w, m] = rng.uniform(0.05, 1.0, w)
        W[lo, m] = max(W[lo, m], 0.05)
        if m % 8 == 0:
            W[lo + w - 1, m] = -W[lo + w - 1, m]             # negative weights in random places
    return W


def mat_wide(fft, n_mel=640, taps=40):
    """640 columns of 40 taps each, staggered across the spectrum: the padded band alone is 100 KB."""
    nb = fft // 2 + 1
    W = np.zeros((nb, n_mel), np.float32)
    lo = (np.arange(n_mel) * (nb - taps)) // (n_mel - 1)
    tri = 1.0 - np.abs(np.arange(taps) - (taps - 1) / 2) / (taps / 2)
    for m in range(n_mel):
        W[lo[m]:lo[m] + taps, m] = tri
    return W


MATRICES = {"identity": mat_identity, "htk": mat_htk, "htk_nyq": lambda f: mat_htk(f, 8000.0, 96),
            "crafted": mat_crafted, "wide": mat_wide}


def signals(n, fft, hop, seed=0):
    """One float32 row per signal: (names, [S, n])."""
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.float64)
    rows = {"noise": rng.uniform(-1, 1, n), "sines": O.sine_mix(n, seed=1234 + seed)}
    for name, off in (("impulse0", 0), ("impulse_mid", n // 2 + 1)):
        rows[name] = np.zeros(n)
        rows[name][min(off, n - 1)] = 1.0
    rows["impulse_comb"] = np.zeros(n)
    rows["impulse_comb"][::3 * hop + 1] = 1.0
    rows["dc"] = np.ones(n)
    rows["nyquist"] = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    for k, name in ((1, "cos1"), (fft // 4, "cos_quarter"), (fft // 2 - 1, "cos_top")):
        rows[name] = np.cos(2 * np.pi * k * i / fft)        # centred on FFT bin k
    rows["zeros"] = np.zeros(n)
    # amplitude sweep, inside the range where sqrtf(Xr^2 + Xi^2) is exact to rounding (logmel.cu header)
    for e in (-40, -20, 12):
        rows[f"noise*2^{e}"] = rng.uniform(-1, 1, n) * 2.0 ** e
    rows["cos_quarter*2^12"] = rows["cos_quarter"] * 2.0 ** 12
    names = list(rows)
    return names, np.stack([rows[k] for k in names]).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# the float64 restatement and the bars
# ------------------------------------------------------------------------------------------------
def window32(fft):
    """The periodic Hann window mt3_frontend_create uploads (`win`)."""
    return (0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(fft) / fft)).astype(np.float32)


def reference(audio, fft, hop, W, win=None, fft32=False):
    """audio [S, n] float32 -> (mel [S, T, M] float64 in the linear domain, A, B) with
      A = sum_b |W_bm| (log2 N |X_b| + sqrt(N) ||xw_t||)   (so the FFT part of the mel bar is tol u A)
      B = sum_b |W_bm X_b|                        (the FMA chain's part is n_fma u B).
    W None is the identity.  fft32: the magnitudes come from numpy's complex64 rfft of the float32 windowed frames
    (mel then stands for what such a kernel would sum), used by the CPU checks of the bar itself."""
    S, n = audio.shape
    T = -(-n // hop)
    nb = fft // 2 + 1
    w64 = (window32(fft) if win is None else win).astype(np.float64)
    M = nb if W is None else W.shape[1]
    Ws = None if W is None else scipy.sparse.csr_matrix(W.astype(np.float64))
    aWs = None if W is None else abs(Ws)
    mel, A, B = (np.empty((S, T, M)) for _ in range(3))
    per = max(1, (1 << 22) // max(1, T * fft))               # segments per block: bounded host memory
    for s0 in range(0, S, per):
        fr = O.frame_pad_end(audio[s0:s0 + per].astype(np.float64), fft, hop) * w64
        nrm = np.sqrt(np.einsum("...i,...i->...", fr, fr))
        if fft32:
            X = np.abs(np.fft.rfft(fr.astype(np.float32), axis=-1)).astype(np.float64)
        else:
            X = np.abs(np.fft.rfft(fr, axis=-1))
        a = np.log2(fft) * X + np.sqrt(fft) * nrm[..., None]
        k = X.shape[0]
        if W is None:
            mel[s0:s0 + k], A[s0:s0 + k], B[s0:s0 + k] = X, a, X
        else:
            flat = lambda v: v.reshape(-1, nb)
            mel[s0:s0 + k] = (flat(X) @ Ws).reshape(k, T, M)
            A[s0:s0 + k] = (flat(a) @ aWs).reshape(k, T, M)
            B[s0:s0 + k] = (flat(X) @ aWs).reshape(k, T, M)
    return mel, A, B


def n_fma(path, W, nb):
    """Length of each column's FMA chain: the padded tap count at 2048 / pow2, the CSR length at 1024 / 4096."""
    if W is None:
        return np.ones(nb)
    lo, hi, taps, _ = band(W)
    if path.startswith("r"):
        return np.where(lo >= 0, hi - lo + 1, 0).astype(np.float64)
    return np.full(W.shape[1], float(taps))


def check(name, got, mel, bar, n_valid=None, rows=None, zero=None, eps=EPS):
    """got [S, T, M] (the kernel's log-mel) against the linear mel and its bar.  `zero` marks the elements whose exact
    mel is 0 term by term: those must be logf(eps) to within 1 ulp.  Returns the worst err/bar."""
    S, T, M = got.shape
    l_eps = log_eps(eps)
    nv = np.full(S, T) if n_valid is None else np.asarray(n_valid)
    valid = np.arange(T)[None, :] < nv[:, None]
    pad = got[~valid]
    assert (pad == 0).all() and not np.signbit(pad).any(), f"{name}: rows past n_valid_frames are not +0.0"
    g = got.astype(np.float64)
    log_term = np.where(mel > 0, np.abs(mel) * (np.abs(np.log(np.where(mel > 0, mel, 1.0))) + 1.0) * 2 * U, 0.0)
    bound = bar + log_term + 1e-300
    err = np.abs(np.exp(g) - mel)
    at_eps = np.abs(got - l_eps) <= abs(np.spacing(l_eps))
    err = np.where(at_eps, np.minimum(err, np.maximum(mel, 0.0)), err)    # logf(eps): the sum may have been <= 0
    ratio = err / bound
    if zero is not None:
        ratio = np.where(zero, np.where(at_eps, 0.0, np.inf), ratio)
    ratio = np.where(np.isfinite(got), ratio, np.inf)
    ratio = np.where(valid[..., None], ratio, 0.0)
    ok = ratio <= 1.0                                                        # NaN fails
    worst = float(np.nanmax(ratio))
    print(f"{name}: worst err/bar {worst:.3f}")
    if not ok.all():
        s, t, m = np.unravel_index(np.argmax(np.where(ok, -1.0, np.nan_to_num(ratio, nan=np.inf))), ok.shape)
        row = rows[s] if rows is not None else s
        raise AssertionError(f"{name}: segment {s} ({row}) frame {t} mel {m}: got {got[s, t, m]!r} "
                             f"(exp {np.exp(g[s, t, m]):.9g}), exact mel {mel[s, t, m]:.9g}, bar {bound[s, t, m]:.3g}, "
                             f"{int((~ok).sum())} elements outside")
    return worst


def mel_bar(path, fft, W, A, B):
    family = "2048" if path.startswith("2048") else ("r" if path.startswith("r") else "pow2")
    wsum = 1.0 if W is None else np.abs(W.astype(np.float64)).sum(axis=0)
    return TOL_FFT[family] * U * A + n_fma(path, W, fft // 2 + 1) * U * B + SUBNORMAL * wsum


# ------------------------------------------------------------------------------------------------
# the library
# ------------------------------------------------------------------------------------------------
class Frontend:
    def __init__(self, fft, hop, W, eps=EPS):
        from mt3_b200 import _lib
        self.eps = eps
        self.lib, self.fft, self.hop = _lib.load(), fft, hop
        self.W = np.ascontiguousarray(W, np.float32)
        self.n_mel = self.W.shape[1]
        cfg = _lib.FrontendConfig(SR, hop, fft, self.n_mel, eps)
        self.h = C.c_void_p()
        _lib.check(self.lib.mt3_frontend_create(C.byref(cfg), self.W.ctypes.data_as(C.c_void_p), C.byref(self.h)))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.mt3_frontend_destroy(self.h)

    def launch(self, audio, stride, S, n, n_valid, out):
        return self.lib.mt3_logmel_f32(self.h, audio.data_ptr(), stride, S, n,
                                       None if n_valid is None else n_valid.data_ptr(), out, None)

    def run(self, audio, n_valid=None, gap=37, tail=64, guard=4096, expect=0):
        """Launches twice on NaN-poisoned buffers; returns the output (or None when `expect` is an error status, after
        checking that nothing was written)."""
        import torch
        S, n = audio.shape
        stride = n + gap
        buf = torch.full((S * stride + tail,), float("nan"), dtype=torch.float32, device=DEV)
        buf[:S * stride].view(S, stride)[:, :n] = torch.from_numpy(audio).to(DEV)
        nv = None if n_valid is None else torch.tensor(n_valid, dtype=torch.int32, device=DEV)
        T = -(-n // self.hop)
        size = S * T * self.n_mel
        outs = []
        for _ in range(2):
            o = torch.full((size + 2 * guard,), float("nan"), dtype=torch.float32, device=DEV)
            st = self.launch(buf, stride, S, n, nv, o.data_ptr() + 4 * guard)
            torch.cuda.synchronize()
            assert st == expect, f"mt3_logmel_f32 -> {st}, expected {expect}: {self.lib.mt3_last_error().decode()}"
            oc = o.cpu().numpy()
            if expect != 0:
                assert np.isnan(oc).all(), "a failed launch wrote to the output"
                return None
            assert np.isnan(oc[:guard]).all() and np.isnan(oc[guard + size:]).all(), "write outside the output"
            outs.append(oc[guard:guard + size].reshape(S, T, self.n_mel))
        assert outs[0].tobytes() == outs[1].tobytes(), "a second launch is not bit-identical to the first"
        return outs[0]


def run_case(name, path, fft, hop, W, audio, rows=None, n_valid=None, gap=37, eps=EPS):
    assert kernel_path(fft, hop, W) == path
    with Frontend(fft, hop, W, eps) as fe:
        got = fe.run(audio, n_valid=n_valid, gap=gap)
    Wr = None if _is_identity(W) else W
    mel, A, B = reference(audio, fft, hop, Wr)
    return check(name, got, mel, mel_bar(path, fft, Wr, A, B), n_valid, rows, zero=(A == 0) & (B == 0), eps=eps)


def _is_identity(W):
    return W.shape[0] == W.shape[1] and np.count_nonzero(W) == W.shape[0] and (np.diagonal(W) == 1).all()


# ------------------------------------------------------------------------------------------------
# the cases: (branch, FFT, hop, matrix, n_samples); worst err/bar on an H100 80GB HBM3 at 700 W in the comment
# ------------------------------------------------------------------------------------------------
CASES = [
    ("2048/smem", 2048, 128, "identity", 3000),           # 0.407
    ("2048/smem", 2048, 2, "identity", 600),              # 0.308
    ("2048/smem", 2048, 130, "crafted", 5000),            # 0.267
    ("2048/smem", 2048, 128, "htk", 3000),                # 0.182
    ("2048/smem", 2048, 130, "htk_nyq", 4000),            # 0.107
    ("2048/global", 2048, 128, "wide", 3000),             # 0.116
    ("2048/global", 2048, 256, "htk", 5000),              # 0.149
    ("2048/global", 2048, 2048, "identity", 9000),        # 0.249
    ("2048/global", 2048, 2048, "crafted", 9000),         # 0.244
    ("r16", 1024, 2, "identity", 700),                    # 0.482
    ("r16", 1024, 128, "htk", 4000),                      # 0.252
    ("r16", 1024, 130, "htk_nyq", 3000),                  # 0.225
    ("r16", 1024, 1024, "crafted", 6000),                 # 0.150
    ("r64", 4096, 128, "identity", 6000),                 # 0.432
    ("r64", 4096, 2, "crafted", 800),                     # 0.281
    ("r64", 4096, 256, "htk", 9000),                      # 0.182
    ("r64", 4096, 510, "htk_nyq", 12000),                 # 0.119
    ("pow2", 64, 2, "identity", 200),                     # 0.414
    ("pow2", 64, 64, "crafted", 300),                     # 0.359
    ("pow2", 256, 128, "htk", 2000),                      # 0.252
    ("pow2", 256, 256, "identity", 2000),                 # 0.252
    ("pow2", 512, 128, "htk", 3000),                      # 0.172
    ("pow2", 512, 130, "crafted", 3000),                  # 0.246
    ("pow2", 8192, 2048, "identity", 20000),              # 0.321
    ("pow2", 8192, 8192, "crafted", 30000),               # 0.151
    ("pow2", 16384, 4096, "htk_nyq", 40000),              # 0.038
    ("pow2", 16384, 2, "crafted", 40),                    # 0.128
]


def _case_id(c):
    return f"{c[0].replace('/', '-')}-fft{c[1]}-hop{c[2]}-{c[3]}-n{c[4]}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_logmel_kernel_vs_float64(case):
    """Every signal of `signals` as one segment, at a ragged length, through each kernel and branch (worst err/bar of
    each case in CASES)."""
    path, fft, hop, mat, n = case
    names, audio = signals(n, fft, hop, seed=fft + hop)
    run_case(_case_id(case), path, fft, hop, MATRICES[mat](fft), audio, rows=names)


@pytest.mark.gpu
def test_logmel2048_bench_shape_mt3_matrix():
    """bench.py's shape, 64 segments x 32 768 samples at hop 128 with the MT3 matrix (2048/smem), rows packed tightly
    as a [64, 32768] tensor is.  Worst err/bar on the H100: 0.176."""
    names, extra = signals(32768, 2048, 128, seed=11)
    mixes = np.stack([O.sine_mix(32768, seed=1234 + i) for i in range(64 - len(names))]).astype(np.float32)
    audio = np.concatenate([mixes, extra])
    rows = [f"sines{i}" for i in range(len(mixes))] + names
    run_case("2048/smem bench shape", "2048/smem", 2048, 128, mat_htk(2048), audio, rows=rows, gap=0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c[3] == "crafted"], ids=_case_id)
def test_logmel_configured_log_eps(case):
    """safe_log replaces with the configured log_eps, not the default: the crafted cases again with log_eps = 1e-3, where
    zero frames, the empty column and the negative sums must read logf(1e-3), and sums below 1e-3 keep their own log."""
    path, fft, hop, mat, n = case
    names, audio = signals(n, fft, hop, seed=fft + hop)
    run_case(_case_id(case) + " eps=1e-3", path, fft, hop, MATRICES[mat](fft), audio, rows=names, eps=1e-3)


LAYOUT = [("2048/smem", 2048, 128), ("2048/global", 2048, 256), ("r16", 1024, 130), ("r64", 4096, 128), ("pow2", 64, 6)]


@pytest.mark.gpu
@pytest.mark.parametrize("path,fft,hop", LAYOUT, ids=lambda v: str(v).replace("/", "-"))
def test_logmel_layout_edges(path, fft, hop):
    """n_samples in {1, hop - 1, hop + 1, N - 1, N + 1, ragged}, n_valid_frames in {0, 1, T - 1, T, T + 5}, S in {1, 3},
    tight and padded row strides, and 65 535 segments of one frame each (the grid.y limit).  Worst err/bar on the H100:
    0.42 (2048/smem), 0.14 (2048/global), 0.24 (r16), 0.30 (r64), 0.27 (pow2); one-sample segments are exact."""
    W = mat_htk(fft) if path == "2048/global" else mat_crafted(fft)
    names, base = signals(3 * fft + hop // 2 + 3, fft, hop, seed=3)
    pick = [names.index(k) for k in ("noise", "sines", "impulse_mid", "dc", "nyquist")]
    for n in sorted({1, hop - 1, hop + 1, fft - 1, fft + 1, 3 * fft + hop // 2 + 3} - {0}):
        T = -(-n // hop)
        audio = np.ascontiguousarray(base[pick, :n])
        nv = [0, 1, max(T - 1, 0), T, T + 5]
        run_case(f"{path} n={n} n_valid={nv}", path, fft, hop, W, audio, rows=[names[p] for p in pick], n_valid=nv)
    n = 3 * fft + hop // 2 + 3
    for S, gap in ((1, 0), (1, 5), (3, 0), (3, 1)):
        run_case(f"{path} S={S} gap={gap}", path, fft, hop, W, np.ascontiguousarray(base[pick[:S]]), gap=gap)
    # 65 535 segments of one frame (33 columns): segment s holds row s % 7, so seven reference rows cover them all
    Wc = mat_crafted(fft)
    small = np.ascontiguousarray(base[:7, :hop])
    audio = np.tile(small, (65535 // 7 + 1, 1))[:65535]
    with Frontend(fft, hop, Wc) as fe:
        got = fe.run(audio)
    mel, A, B = reference(small, fft, hop, Wc)
    idx = np.arange(65535) % 7
    wide_path = kernel_path(fft, hop, Wc)
    check(f"{wide_path} S=65535", got, mel[idx], mel_bar(wide_path, fft, Wc, A, B)[idx], zero=((A == 0) & (B == 0))[idx])


@pytest.mark.gpu
def test_logmel_error_paths_write_nothing():
    """65 536 segments is MT3_ERR_SHAPE; a CSR band too large for shared memory at FFT 1024 / 4096 is
    MT3_ERR_UNSUPPORTED.  Both return before any launch: the NaN output stays NaN."""
    hop = 128
    W = mat_crafted(2048)
    with Frontend(2048, hop, W) as fe:
        fe.run(np.zeros((65536, hop), np.float32), gap=0, expect=-2)
    for fft in (1024, 4096):
        dense = np.ones((fft // 2 + 1, 128), np.float32)
        assert kernel_path(fft, hop, dense).endswith("/unsupported")
        with Frontend(fft, hop, dense) as fe:
            fe.run(np.ones((2, 3000), np.float32), expect=-3)


# ------------------------------------------------------------------------------------------------
# CPU: the restatement, the bar and the branch choice
# ------------------------------------------------------------------------------------------------
def test_frontend_create_rejects_bad_configs():
    """Argument checks run before any CUDA call: odd hop, hop > FFT, FFT not a power of two, FFT 32 768."""
    from mt3_b200 import _lib
    lib = _lib.load()
    mel = np.ones((16385, 4), np.float32)
    h = C.c_void_p()
    for hop, fft, status in ((127, 2048, -1), (4096, 2048, -1), (128, 1000, -3), (128, 32768, -3), (0, 2048, -1)):
        cfg = _lib.FrontendConfig(SR, hop, fft, 4, EPS)
        assert lib.mt3_frontend_create(C.byref(cfg), mel.ctypes.data_as(C.c_void_p), C.byref(h)) == status, (hop, fft)


@pytest.mark.parametrize("fft,hop", [(2048, 128), (2048, 130), (1024, 2), (64, 64), (16384, 4096)])
def test_reference_matches_oracle_float64(fft, hop):
    """With a float64 window the restatement is the oracle's float64 pipeline."""
    n = 2 * fft + 77
    audio = np.stack([O.sine_mix(n, seed=5), np.random.default_rng(1).uniform(-1, 1, n)]).astype(np.float32)
    bins = 512 if fft >= 1024 else 128
    W = mat_htk(fft)
    mel, _, _ = reference(audio, fft, hop, W, win=O.hann_periodic(fft, np.float64))
    got = np.log(np.where(mel <= 0, EPS, mel))
    want = O.compute_logmel(audio.astype(np.float64), bins, 20.0, 7600.0, fft, hop, SR, np.float64)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


ALL_FFTS = [64, 256, 512, 1024, 2048, 4096, 8192, 16384]


def _complex64_logmel(audio, fft, hop):
    """What a kernel computing numpy's complex64 rfft would output with the identity matrix."""
    mel32, A, B = reference(audio, fft, hop, None, fft32=True)
    got = np.log(np.where(mel32 <= 0, EPS, mel32).astype(np.float32))
    return got, mel32


@pytest.mark.parametrize("fft", ALL_FFTS)
def test_bar_accepts_complex64_rfft(fft):
    """numpy's complex64 rfft of the float32 windowed frames (pocketfft: mixed radix, not the kernels' radix-2) passes
    the magnitude bar at tol = 1 within half of it, on every signal at every FFT size (measured: 0.34 at worst)."""
    hop = fft // 4
    names, audio = signals(2 * fft + hop + 5, fft, hop, seed=21)
    got, _ = _complex64_logmel(audio, fft, hop)
    mel, A, B = reference(audio, fft, hop, None)
    worst = check(f"complex64 rfft N={fft}", got, mel, U * A + U * B + SUBNORMAL, rows=names, zero=(A == 0) & (B == 0))
    assert worst <= 0.5


@pytest.mark.parametrize("fft", [64, 2048, 4096, 16384])
def test_bar_rejects_in_bounds_perturbations(fft):
    """The bar, at the loosest tol any kernel uses, rejects magnitudes scaled by 1 + 2^-14, one bin replaced by its
    neighbour, and the Nyquist bin computed as |Re Z_0 + Im Z_0| (which is the DC magnitude)."""
    hop = fft // 4
    audio = np.random.default_rng(4).uniform(-1, 1, (2, 2 * fft + 11)).astype(np.float32)
    _, mel32 = _complex64_logmel(audio, fft, hop)
    mel, A, B = reference(audio, fft, hop, None)
    bar = max(TOL_FFT.values()) * U * A + U * B + SUBNORMAL
    k = fft // 8
    bad = {"scaled": mel32 * (1 + 2.0 ** -14), "neighbour": mel32.copy(), "nyquist=|Re Z0 + Im Z0|": mel32.copy()}
    bad["neighbour"][..., k] = mel32[..., k + 1]
    bad["nyquist=|Re Z0 + Im Z0|"][..., -1] = mel32[..., 0]
    for what, m in bad.items():
        got = np.log(np.where(m <= 0, EPS, m).astype(np.float32))
        with pytest.raises(AssertionError):
            check(f"N={fft} {what}", got, mel, bar)


def test_check_pins_exact_zeros_to_log_eps():
    """Where the exact mel is 0 term by term, only logf(eps) passes: not logf(0) = -inf, not logf(FLT_MIN), not -60, and
    not logf of another eps.  A non-finite output fails anywhere."""
    mel = np.array([[[0.0, 1e-9, 0.5]]])
    bar = np.array([[[0.0, 1e-8, 1e-7]]])
    zero = np.array([[[True, False, False]]])
    for eps in (1e-5, 1e-3):
        good = np.array([[[log_eps(eps), log_eps(eps), np.log(0.5)]]], np.float32)
        assert check("exact zero", good, mel, bar, zero=zero, eps=eps) <= 1.0
        for bad0 in (-np.inf, np.log(np.finfo(np.float32).tiny), -60.0, log_eps(1e-5 if eps == 1e-3 else 1e-3)):
            got = good.copy()
            got[0, 0, 0] = bad0
            with pytest.raises(AssertionError):
                check(f"exact zero {bad0}", got, mel, bar, zero=zero, eps=eps)
        got = good.copy()
        got[0, 0, 1] = -np.inf                                  # within the bar of 0 in the linear domain, but not finite
        with pytest.raises(AssertionError):
            check("-inf", got, mel, bar, zero=zero, eps=eps)


def test_branch_margins():
    """Each case reaches the branch it names, and the two 2048 cases that guarantee a branch sit >= 16 KB from the
    113 KB threshold, so a retune of frames or warps per CTA cannot silently move them to the other branch."""
    for path, fft, hop, mat, n in CASES:
        assert kernel_path(fft, hop, MATRICES[mat](fft)) == path, (path, fft, hop, mat)
    for path, fft, hop in LAYOUT:
        assert kernel_path(fft, hop, mat_htk(fft) if path == "2048/global" else mat_crafted(fft)) == path
    _, _, taps, _ = band(mat_identity(2048))
    base, mel = smem_2048(128, 1025, taps)
    assert MEL_BUDGET_2048 - (base + mel) >= 16 * 1024                # identity, hop 128: band in shared memory
    W = mat_wide(2048)
    _, _, taps, _ = band(W)
    base, mel = smem_2048(128, W.shape[1], taps)
    assert taps >= 32 and W.shape[1] >= 600 and mel >= 77 * 1024
    assert (base + mel) - MEL_BUDGET_2048 >= 50 * 1024               # wide band, hop 128: band in global memory
    assert base <= SMEM_MAX
    # the realistic ways in, close to the threshold: the MT3 matrix has 10 taps (4 KB inside at hop 128, 1.5 KB
    # outside at hop 256)
    _, _, taps, _ = band(mat_htk(2048))
    assert taps == 10
    assert smem_2048(128, 512, taps) == (91136, 20480)
    assert sum(smem_2048(256, 512, taps)) - MEL_BUDGET_2048 == 1536
