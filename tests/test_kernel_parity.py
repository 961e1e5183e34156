"""Kernel-level parity (-m gpu): every hot-path CUDA kernel, launched alone through the test-only harness library
(mt3_b200/csrc/tools/kernel_harness.cu -> libmt3kernels.so), against a float64 numpy reference computed from the same
fp32 inputs -- at ragged shapes, in every epilogue and every K/V row format.

Error is judged per element against the condition of that element, not against max|ref|:
  GEMM       |got - ref| <= tol * cond,  cond = rs * sum_k |a_k b_k|  (+ |R| or |pe| for the additive epilogues; gated
             GELU propagates the two inputs' conditions through gelu'(c0) c1 and gelu(c0), plus |c0 c1| for tanhf)
  attention  |got - ref| <= tol_p * sum_k p_k |v_k|  +  tol_s * sum_k p_k |v_k - o| A_k,   A_k = sum_d |q_d k_kd|
             (tol_p: error of the weights p; tol_s: error of the scores, which moves p_k by a relative s-error)
Inputs have a positive mean, so a systematic error (a dropped correction term, a truncation) is not hidden by
random-sign cancellation in the condition.  Output buffers are larger than the logical output and start as NaN; after
the launch everything outside the written region must still be NaN.  Input rows a kernel must not read (cache rows
>= len, K/V rows past T inside cap) hold NaN.

The bars are derived from the arithmetic below (u = 2^-24) and sit within 10x of the worst err/bound measured on an
H100 80GB HBM3 (quoted in each test's docstring as a fraction of its bar).
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "mt3_b200", "csrc", "tools")
DEV = "cuda:0"
EPI_STORE, EPI_RESIDUAL, EPI_ADD_PE, EPI_GATED_GELU = 0, 1, 2, 3

# exact fp32 FMA chains: gamma_K = K u is the worst case, the per-element errors stay near sqrt(K) u.  SIMT GEMM: one
# chain of up to 1024 products (2^-17 = 128 u); decode GEMMs: chains of <= 128 products summed over 8 or 16 CTAs
# (2^-20 = 16 u)
TOL_FP32 = 2.0 ** -17
TOL_DEC = 2.0 ** -20
# attention in fp32 (attention_fp32_kernel, dec_attention_bulk_kernel): scores are 64-term dot products (tol_s), the
# weights carry expf's ulps and the row sum (tol_p)
TOL_ENC_ATT_P, TOL_ENC_ATT_S = 2.0 ** -18, 2.0 ** -20
TOL_DEC_ATT_P, TOL_DEC_ATT_S = 2.0 ** -20, 2.0 ** -22
# 3xTF32: the dropped lo.lo term and the lo operands read as tf32 (<= 2^-20 of each product) plus the tensor core's fp32
# accumulation
TOL_TF32X3 = 2.0 ** -16
# TF32: both operands truncated to 10 mantissa bits (<= 2^-10 each)
TOL_TF32 = 2.0 ** -9
# TC attention: P rounded to nearest tf32 (2^-11) in numerator and row sum
TOL_ATT_P = 2.0 ** -10


# ------------------------------------------------------------------------------------------------
# the harness library
# ------------------------------------------------------------------------------------------------
class TcGemmArgs(C.Structure):
    _fields_ = [("M", C.c_int), ("N", C.c_int), ("K", C.c_int), ("row_scale", C.c_void_p), ("epi", C.c_int),
                ("R_hi", C.c_void_p), ("R_lo", C.c_void_p), ("ldr", C.c_int), ("pe", C.c_void_p), ("pe_T", C.c_int),
                ("pe_ld", C.c_int), ("C_hi", C.c_void_p), ("C_lo", C.c_void_p), ("ldc", C.c_int), ("n_split", C.c_int),
                ("C1", C.c_void_p), ("kv_fmt", C.c_int), ("hm_rows_per_b", C.c_int), ("hm_cap", C.c_int), ("hm_H", C.c_int),
                ("hm_pos", C.c_void_p), ("VT_hi", C.c_void_p), ("VT_lo", C.c_void_p), ("vt_col0", C.c_int), ("vt_T", C.c_int),
                ("vt_H", C.c_int)]


class GemmArgs(C.Structure):
    _fields_ = [("A", C.c_void_p), ("lda", C.c_int), ("B", C.c_void_p), ("ldb", C.c_int), ("M", C.c_int), ("N", C.c_int),
                ("K", C.c_int), ("row_scale", C.c_void_p), ("epi", C.c_int), ("R", C.c_void_p), ("ldr", C.c_int),
                ("pe", C.c_void_p), ("pe_T", C.c_int), ("pe_ld", C.c_int), ("C", C.c_void_p), ("ldc", C.c_int),
                ("n_split", C.c_int), ("C1", C.c_void_p), ("kv_fmt", C.c_int), ("hm_rows_per_b", C.c_int), ("hm_cap", C.c_int),
                ("hm_H", C.c_int), ("hm_pos", C.c_void_p)]


class DecGemmArgs(C.Structure):
    _fields_ = [("A", C.c_void_p), ("lda", C.c_int), ("W", C.c_void_p), ("ldw", C.c_int), ("M", C.c_int), ("N", C.c_int),
                ("K", C.c_int), ("norm", C.c_int), ("eps", C.c_float), ("epi", C.c_int), ("R", C.c_void_p), ("ldr", C.c_int),
                ("C", C.c_void_p), ("ldc", C.c_int), ("n_split", C.c_int), ("C1", C.c_void_p), ("kv_fmt", C.c_int),
                ("hm_rows_per_b", C.c_int), ("hm_cap", C.c_int), ("hm_H", C.c_int), ("hm_pos", C.c_void_p),
                ("partial", C.c_void_p), ("counters", C.c_void_p), ("A2", C.c_void_p), ("lda2", C.c_int), ("K0", C.c_int),
                ("ssq_out", C.c_void_p), ("ssq_ld", C.c_int), ("trace", C.c_void_p)]


@pytest.fixture(scope="module")
def kh():
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, F, LL = C.c_void_p, C.c_int, C.c_float, C.c_longlong
    sig = {
        "kh_last_error": ([], C.c_char_p), "kh_sizeof": ([I], LL),
        "kh_tc_gemm": ([P, P, I, P, P, I, P, I], I), "kh_sgemm": ([P], I),
        "kh_enc_attention_tc": ([P, P, P, P, I, I, I, P, P, I, P], I), "kh_enc_attention_tc_scratch_floats": ([I, I, I], LL),
        "kh_enc_attention_tc_supported": ([I], I), "kh_enc_attention_fp32": ([P, I, I, I, P, P], I),
        "kh_dec_gemm_cluster": ([P], I), "kh_dec_gemm": ([P], I), "kh_dec_gemm_out_q": ([P, P], I),
        "kh_dec_attention": ([I, P, I, I, P, I, I, P, I, I, P, I, P, I, I, F, F, I, I], I),
        "kh_p24_roundtrip": ([P, P, P, LL, I], I),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    for i, s in enumerate((TcGemmArgs, GemmArgs, DecGemmArgs)):
        assert lib.kh_sizeof(i) == C.sizeof(s), f"ctypes mirror of {s.__name__} does not match the C layout"
    return lib


def _call(kh, fn, *args):
    r = getattr(kh, fn)(*args)
    assert r == 0, f"{fn} -> {r}: {kh.kh_last_error().decode()}"
    torch.cuda.synchronize()


def _p(t):
    return None if t is None else t.data_ptr()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def _split(x):
    """split_tf32: hi = x with the low 13 mantissa bits cleared, lo = x - hi (exact in fp32)."""
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, (x - hi).astype(np.float32)


def _check(name, got, ref, cond, tol, extra=None, tol_extra=0.0):
    """Per-element bar; prints the worst err / bound so the docstring numbers can be re-measured."""
    got = np.asarray(got, np.float64)
    bound = tol * cond + (tol_extra * extra if extra is not None else 0.0) + 1e-300
    err = np.abs(got - ref)
    ratio = err / bound
    ok = err <= bound                                     # NaN fails
    worst = float(np.nanmax(ratio)) if np.isfinite(ratio).any() else float("inf")
    print(f"{name}: worst err/bound {worst:.3f} (tol {tol:.2e})")
    if not ok.all():
        i = np.unravel_index(np.argmax(np.where(ok, -1, np.nan_to_num(ratio, nan=np.inf))), ok.shape)
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.size} elements out of bound; at {i}: got {got[i]!r} "
                             f"ref {ref[i]!r} bound {bound[i]:.3e}")
    return worst


def _assert_poison(name, buf, written):
    """Everything of `buf` (float tensor) outside the boolean mask `written` is still NaN."""
    b = buf.cpu().numpy()
    outside = ~written
    assert np.isnan(b[outside]).all(), f"{name}: {int((~np.isnan(b[outside])).sum())} elements written outside the output"


def _gelu(x):
    return 0.5 * x * (1.0 + np.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def _dgelu(x):
    u = 0.7978845608028654 * (x + 0.044715 * x ** 3)
    t = np.tanh(u)
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * 0.7978845608028654 * (1.0 + 3 * 0.044715 * x * x)


def _pos_mean(rng, shape, scale=1.0):
    """uniform on [-0.5, 1) * scale, as float32: a positive mean keeps sum |a b| close to |sum a b|"""
    return (rng.uniform(-0.5, 1.0, shape) * scale).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# host restatements of the storage formats
# ------------------------------------------------------------------------------------------------
ROWB = {0: 256, 1: 128, 2: 192}


def vt_key_slot(t):
    """Position of key t inside its group of 8 in the V^T operand: even keys of the group first, then odd ones."""
    t = np.asarray(t)
    g, i = t // 8 * 8, t % 8
    return g + np.where(i % 2 == 0, i // 2, 4 + i // 2)


def _p24_decode_bits(t):
    t = np.asarray(t).astype(np.uint64) & np.uint64(0xFFFFFF)
    return ((t << np.uint64(8)) | (t & np.uint64(255))).astype(np.uint32)


def p24_encode_ref(x):
    """The 24 stored bits of the p24 value NEAREST to finite fp32 x: the candidates are the values whose low byte repeats
    the third byte next to x (codes t = bits >> 8 and t +- 1 of the same sign); ties keep the truncated code t, and t + 1
    beats t - 1 (encoder order, gemm_simt.cuh)."""
    x = np.asarray(x, np.float32)
    t = (x.view(np.uint32) >> np.uint32(8)).astype(np.int64)
    xv = x.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        def dist(c):
            return np.abs(_p24_decode_bits(c).view(np.float32).astype(np.float64) - xv)
        best, berr = t.copy(), dist(t)
        for c, allowed in ((t + 1, np.ones(t.shape, bool)), (t - 1, (t & 0x7FFFFF) != 0)):
            e = np.where(allowed, dist(c), np.inf)
            take = e < berr
            best, berr = np.where(take, c, best), np.where(take, e, berr)
    return best.astype(np.uint32)


def encode_rows(v, fmt):
    """[..., 64] fp32 -> [..., ROWB] bytes of the K/V row format (kv_dest() in gemm_simt.cuh)"""
    v = np.ascontiguousarray(v, np.float32)
    if fmt == 0:
        return v.view(np.uint8).reshape(v.shape[:-1] + (256,))
    if fmt == 1:
        return v.astype(np.float16).view(np.uint8).reshape(v.shape[:-1] + (128,))
    t = p24_encode_ref(v)
    hi = (t >> np.uint32(8)).astype(np.uint16).view(np.uint8).reshape(v.shape[:-1] + (128,))
    lo = (t & np.uint32(255)).astype(np.uint8)
    return np.concatenate([hi, lo], axis=-1)


def decode_rows(u8, fmt):
    """[..., ROWB] bytes -> [..., 64] float64 values as stored"""
    u8 = np.ascontiguousarray(u8)
    if fmt == 0:
        return u8.view(np.float32).astype(np.float64)
    if fmt == 1:
        return u8.view(np.float16).astype(np.float64)
    hi = np.ascontiguousarray(u8[..., :128]).view(np.uint16).astype(np.uint32)
    lo = u8[..., 128:].astype(np.uint32)
    return ((hi << 16) | (lo << 8) | lo).astype(np.uint32).view(np.float32).astype(np.float64)


def test_host_restatements_self_consistent():
    """The numpy restatements the kernel tests rely on: vt_key_slot is a permutation of every group of 8, and the p24
    encoder picks a value whose decoded form is within 2^-16 of x."""
    s = vt_key_slot(np.arange(64))
    assert sorted(s.tolist()) == list(range(64)) and (s // 8 == np.arange(64) // 8).all()
    x = np.random.default_rng(0).standard_normal(4096).astype(np.float32)
    y = decode_rows(encode_rows(x.reshape(-1, 64), 2), 2).ravel()
    assert (np.abs(y - x) <= 2.0 ** -16 * np.abs(x)).all()


# ------------------------------------------------------------------------------------------------
# GEMMs: gemm_tf32_kernel (TF32, TF32X3) and sgemm_kernel
# ------------------------------------------------------------------------------------------------
def _gemm_ref(A, W, rs, epi, R=None, pe=None, pe_T=None):
    A64, W64 = A.astype(np.float64), W.astype(np.float64)
    acc, cond = A64 @ W64, np.abs(A64) @ np.abs(W64)
    if rs is not None:
        acc, cond = acc * rs[:, None], cond * rs[:, None]
    if epi == EPI_GATED_GELU:
        c0, c1, k0, k1 = acc[:, 0::2], acc[:, 1::2], cond[:, 0::2], cond[:, 1::2]
        ref = _gelu(c0) * c1
        return ref, np.abs(_dgelu(c0)) * np.abs(c1) * k0 + np.abs(_gelu(c0)) * k1 + np.abs(c0 * c1)
    if epi == EPI_RESIDUAL:
        return acc + R, cond + np.abs(R)
    if epi == EPI_ADD_PE:
        p = pe.astype(np.float64)[np.arange(A.shape[0]) % pe_T]
        return acc + p, cond + np.abs(p)
    return acc, cond


def _run_gemm(kh, mode, M, N, K, epi, rs=False, pe_T=None, c_lo=False, inplace=False, seed=0, kv=None, AW=None):
    """One GEMM launch (mode "tf32" | "tf32x3" | "simt") into NaN-poisoned, padded buffers.  Returns (C [M, Nout] as
    float64 hi + lo, the C_hi / C_lo device buffers, ref, cond).  kv = (n_split, fmt, T, cap, H, C1 buffer) routes columns
    >= n_split to the head-major K/V store; AW = (A, W) replaces the random operands."""
    rng = np.random.default_rng(seed)
    A = _pos_mean(rng, (M, K))
    W = _pos_mean(rng, (K, N), 2.0 / K)
    if AW is not None:
        A, W = AW
    rsv = rng.uniform(0.5, 2.0, M).astype(np.float32) if rs else None
    Nout = N // 2 if epi == EPI_GATED_GELU else N
    n_split = kv[0] if kv else N
    ncols = min(Nout, n_split)
    ldc = ncols + 4 + (4 if mode == "simt" else 0)
    R = _pos_mean(rng, (M, N)) if epi == EPI_RESIDUAL else None
    pe = _pos_mean(rng, (pe_T, N)) if epi == EPI_ADD_PE else None
    ref, cond = _gemm_ref(A, W, rsv, epi, R, pe, pe_T)
    split3 = mode == "tf32x3"
    Ch, Cl = _nan(M + 3, ldc), (_nan(M + 3, ldc) if c_lo else None)
    Rh = Rl = None
    if R is not None:
        rh, rl = _split(R) if split3 else (R, None)
        if inplace:                                            # R == C, as the model's residual GEMMs run
            Ch[:M, :N] = _dev(rh)
            Rh, ldr = Ch, ldc
            if rl is not None and Cl is not None:
                Cl[:M, :N] = _dev(rl)
                Rl = Cl
            elif rl is not None:
                Rl = _dev(np.pad(rl, ((0, 0), (0, ldc - N))))
        else:
            Rh, Rl, ldr = _dev(rh), (_dev(rl) if rl is not None else None), N
    else:
        ldr = 0
    d_rs = _dev(rsv) if rs else None
    d_pe = _dev(pe) if pe is not None else None
    kv_fields = dict(n_split=n_split)
    if kv:
        _, fmt, T, cap, H, C1 = kv
        kv_fields.update(C1=_p(C1), kv_fmt=fmt, hm_rows_per_b=T, hm_cap=cap, hm_H=H, hm_pos=None)
    if mode == "simt":
        dA, dW = _dev(A), _dev(W)
        a = GemmArgs(A=_p(dA), lda=K, B=_p(dW), ldb=N, M=M, N=N, K=K, row_scale=_p(d_rs), epi=epi, R=_p(Rh), ldr=ldr,
                     pe=_p(d_pe), pe_T=pe_T or 0, pe_ld=N, C=_p(Ch), ldc=ldc, **kv_fields)
        keep = (dA, dW)
        _call(kh, "kh_sgemm", C.byref(a))
    else:
        Wt = np.ascontiguousarray(W.T)
        if split3:
            (ah, al), (wh, wl) = _split(A), _split(Wt)
            dA, dAl, dW, dWl = _dev(ah), _dev(al), _dev(wh), _dev(wl)
        else:
            dA, dAl, dW, dWl = _dev(A), None, _dev(Wt), None
        a = TcGemmArgs(M=M, N=N, K=K, row_scale=_p(d_rs), epi=epi, R_hi=_p(Rh), R_lo=_p(Rl), ldr=ldr, pe=_p(d_pe), pe_T=pe_T or 0,
                       pe_ld=N, C_hi=_p(Ch), C_lo=_p(Cl), ldc=ldc, **kv_fields)
        keep = (dA, dAl, dW, dWl, Rl)
        _call(kh, "kh_tc_gemm", _p(dA), _p(dAl), K, _p(dW), _p(dWl), K, C.byref(a), int(split3))
    del keep
    got = Ch[:M, :ncols].double().cpu().numpy()
    if Cl is not None:
        got = got + Cl[:M, :ncols].double().cpu().numpy()
    return got, Ch, Cl, ref, cond


GEMM_TOL = {"tf32": TOL_TF32, "tf32x3": TOL_TF32X3, "simt": TOL_FP32}
# (M, N, K, epilogue, row scale, pe_T, C_lo, in place): every M / N / K of the list appears at least once
TC_CASES = [
    (1, 32, 32, EPI_STORE, False, None, False, False),
    (64, 96, 64, EPI_RESIDUAL, True, None, True, False),
    (127, 160, 384, EPI_GATED_GELU, True, None, True, False),
    (128, 1152, 384, EPI_STORE, True, None, True, False),
    (129, 2048, 1024, EPI_GATED_GELU, True, None, False, False),
    (200, 160, 1024, EPI_ADD_PE, False, 37, True, False),
    (200, 96, 384, EPI_RESIDUAL, True, None, True, True),
    (129, 32, 64, EPI_ADD_PE, True, 129, False, False),
    (16448, 160, 384, EPI_RESIDUAL, False, None, True, True),
]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
@pytest.mark.parametrize("case", TC_CASES, ids=lambda c: f"M{c[0]}-N{c[1]}-K{c[2]}-epi{c[3]}" + ("-inplace" if c[7] else ""))
def test_tc_gemm_epilogues(kh, mode, case):
    """gemm_tf32_kernel: ragged M (1, 127, 129, 200, 16448), N not a multiple of the 128-column tile, every epilogue,
    sinusoid rows wrapping at pe_T != M, hi/lo output, residual read from the buffer being written.
    Measured worst err/bound: TF32X3 0.31, TF32 0.23."""
    M, N, K, epi, rs, pe_T, c_lo, inplace = case
    c_lo = c_lo and mode == "tf32x3"
    got, Ch, Cl, ref, cond = _run_gemm(kh, mode, M, N, K, epi, rs, pe_T, c_lo, inplace, seed=M + N + K)
    _check(f"tc gemm {mode} {case}", got, ref, cond, GEMM_TOL[mode])
    w = np.zeros(Ch.shape, bool)
    w[:M, :got.shape[1]] = True
    _assert_poison("C_hi", Ch, w)
    if Cl is not None:
        _assert_poison("C_lo", Cl, w)


@pytest.mark.parametrize("case", [(100, 96, 64, EPI_STORE, True, None), (100, 160, 384, EPI_GATED_GELU, True, None),
                                  (129, 96, 384, EPI_RESIDUAL, False, None), (200, 1152, 1024, EPI_ADD_PE, True, 37),
                                  (1, 36, 16, EPI_STORE, False, None), (300, 2048, 512, EPI_GATED_GELU, False, None)],
                         ids=lambda c: f"M{c[0]}-N{c[1]}-K{c[2]}-epi{c[3]}")
def test_sgemm_epilogues(kh, case):
    """sgemm_kernel, the exact-fp32 parity anchor, on both tile shapes (M <= 128: 64 x 32 tiles; M > 128: 128 x 128).
    Measured worst err/bound: 0.10."""
    M, N, K, epi, rs, pe_T = case
    got, Ch, _, ref, cond = _run_gemm(kh, "simt", M, N, K, epi, rs, pe_T, seed=7 + M)
    _check(f"sgemm {case}", got, ref, cond, TOL_FP32)
    w = np.zeros(Ch.shape, bool)
    w[:M, :got.shape[1]] = True
    _assert_poison("C", Ch, w)


@pytest.mark.parametrize("epi", [EPI_STORE, EPI_RESIDUAL, EPI_GATED_GELU])
def test_tc_gemm_hi_lo_split_is_exact(kh, epi):
    """The hi/lo output split: hi is exactly tf32 (low 13 bits zero) and hi + lo is bit-for-bit the unsplit result."""
    M, N, K = 200, 160, 384
    _, Ch, Cl, _, _ = _run_gemm(kh, "tf32x3", M, N, K, epi, True, None, True, seed=5)
    _, Cu, _, _, _ = _run_gemm(kh, "tf32x3", M, N, K, epi, True, None, False, seed=5)
    n = N // 2 if epi == EPI_GATED_GELU else N
    hi, lo, un = (x[:M, :n].cpu().numpy() for x in (Ch, Cl, Cu))
    assert (hi.view(np.uint32) & 0x1FFF == 0).all()
    np.testing.assert_array_equal((hi + lo).view(np.uint32), un.view(np.uint32))


@pytest.mark.parametrize("vt_T,B", [(8, 3), (200, 2), (256, 1)])
def test_tc_gemm_vt_store(kh, vt_T, B):
    """The transposed per-head V^T store of the fused QKV projection: vt[((b H + h) 64 + d) T + vt_key_slot(t)] (numpy
    restatement of the slot order), hi exactly tf32, hi + lo within the 3xTF32 bar; the V third of C is not written."""
    H, K = 2, 512
    Q = H * 64
    N, M = 3 * Q, B * vt_T
    rng = np.random.default_rng(vt_T)
    A, W = _pos_mean(rng, (M, K)), _pos_mean(rng, (K, N), 2.0 / K)
    ref, cond = _gemm_ref(A, W, None, EPI_STORE)
    (ah, al), (wh, wl) = _split(A), _split(np.ascontiguousarray(W.T))
    dA, dAl, dW, dWl = _dev(ah), _dev(al), _dev(wh), _dev(wl)
    Ch, Cl = _nan(M + 2, N + 4), _nan(M + 2, N + 4)
    n_vt = B * H * 64 * vt_T
    VTh, VTl = _nan(n_vt + 64), _nan(n_vt + 64)
    a = TcGemmArgs(M=M, N=N, K=K, epi=EPI_STORE, C_hi=_p(Ch), C_lo=_p(Cl), ldc=N + 4, n_split=N, VT_hi=_p(VTh), VT_lo=_p(VTl),
                   vt_col0=2 * Q, vt_T=vt_T, vt_H=H)
    _call(kh, "kh_tc_gemm", _p(dA), _p(dAl), K, _p(dW), _p(dWl), K, C.byref(a), 1)
    got = Ch[:M, :2 * Q].double().cpu().numpy() + Cl[:M, :2 * Q].double().cpu().numpy()
    _check("qk part", got, ref[:, :2 * Q], cond[:, :2 * Q], TOL_TF32X3)
    w = np.zeros(Ch.shape, bool)
    w[:M, :2 * Q] = True
    _assert_poison("C_hi", Ch, w)
    _assert_poison("C_lo", Cl, w)
    # expected V^T: [B, H, 64, T] with the key axis permuted by vt_key_slot
    slot = vt_key_slot(np.arange(vt_T))
    exp_ref = np.empty((B, H, 64, vt_T))
    exp_cond = np.empty((B, H, 64, vt_T))
    exp_ref[..., slot] = ref[:, 2 * Q:].reshape(B, vt_T, H, 64).transpose(0, 2, 3, 1)
    exp_cond[..., slot] = cond[:, 2 * Q:].reshape(B, vt_T, H, 64).transpose(0, 2, 3, 1)
    vh, vl = VTh.cpu().numpy(), VTl.cpu().numpy()
    assert np.isnan(vh[n_vt:]).all() and np.isnan(vl[n_vt:]).all()
    assert (vh[:n_vt].view(np.uint32) & 0x1FFF == 0).all()
    _check(f"V^T T={vt_T}", (vh[:n_vt].astype(np.float64) + vl[:n_vt]).reshape(exp_ref.shape), exp_ref, exp_cond, TOL_TF32X3)


@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("mode", ["tf32x3", "simt"])
def test_gemm_head_major_kv_store(kh, fmt, mode):
    """Columns >= n_split go to the head-major K/V rows kv[b][K|V][h][t][64] (the hoisted cross K/V: rows_per_b = T), in
    fp32, fp16 and p24 rows; byte-for-byte what the host encoders make of the same GEMM's plain fp32 output, rows >= T of
    each (b, K|V, h) inside cap untouched."""
    B, T, cap, H, K, n_split = 2, 200, 208, 2, 384, 64
    N, M = n_split + 2 * H * 64, B * T
    full, _, _, ref, cond = _run_gemm(kh, mode, M, N, K, EPI_STORE, True, seed=11)
    _check("unsplit", full, ref, cond, GEMM_TOL[mode])
    C1 = torch.full((B * 2 * H * cap * ROWB[fmt],), 255, dtype=torch.uint8, device=DEV)
    got, Ch, _, _, _ = _run_gemm(kh, mode, M, N, K, EPI_STORE, True, seed=11, kv=(n_split, fmt, T, cap, H, C1))
    np.testing.assert_array_equal(got, full[:, :n_split])
    w = np.zeros(Ch.shape, bool)
    w[:M, :n_split] = True
    _assert_poison("C", Ch, w)
    kvb = C1.cpu().numpy().reshape(B, 2, H, cap, ROWB[fmt])
    want = encode_rows(full[:, n_split:].astype(np.float32).reshape(B, T, 2, H, 64).transpose(0, 2, 3, 1, 4), fmt)
    np.testing.assert_array_equal(kvb[:, :, :, :T], want)
    assert (kvb[:, :, :, T:] == 255).all(), "rows past T were written"


# ------------------------------------------------------------------------------------------------
# encoder attention: attention_tc_kernel (+ combine) and the exact-fp32 attention_fp32_kernel in the encoder's form
# ------------------------------------------------------------------------------------------------
def _attn_inputs(rng, B, T, H, sharp):
    """qkv [B*T, 3*H*64] exactly as the QKV GEMM leaves it.  Diffuse: |S| ~ 1.  Sharp: S = r_i s_j along a shared
    direction plus noise, row maxima 90..120 (above the 88.7 where e^S overflows fp32); key scales alternate between
    sequences (so a key that is masked for one sequence would dominate it) and shrink across the key parts of T > 256
    (part row maxima far apart)."""
    Q = H * 64
    qkv = np.empty((B, T, 3, H, 64), np.float32)
    if not sharp:
        qkv[:, :, :2] = rng.standard_normal((B, T, 2, H, 64)) * 0.35
    else:
        u = rng.standard_normal(64)
        u /= np.linalg.norm(u)
        r = rng.uniform(8.0, 11.0, (B, T, H, 1))
        part = np.arange(T) // 256
        top = np.array([11.0, 4.0, 1.0, 8.0])[part % 4][None, :, None, None]
        s = rng.uniform(-0.1, 1.0, (B, T, H, 1)) * top
        if B > 1:                                              # even sequences: small keys, |S| <= 6
            s[0::2] = rng.uniform(-0.5, 0.5, s[0::2].shape)
        noise = rng.standard_normal((B, T, 2, H, 64)) * 0.05
        qkv[:, :, 0] = r * u + noise[:, :, 0]
        qkv[:, :, 1] = s * u + noise[:, :, 1]
    qkv[:, :, 2] = rng.uniform(-0.5, 1.0, (B, T, H, 64))
    return qkv.reshape(B * T, 3 * Q)


def _attn_ref(qkv, B, T, H):
    """float64 softmax(Q K^T) V per (b, h) and the two condition terms"""
    x = qkv.astype(np.float64).reshape(B, T, 3, H, 64).transpose(2, 0, 3, 1, 4)    # [3, B, H, T, 64]
    q, k, v = x
    S = q @ k.transpose(0, 1, 3, 2)
    p = np.exp(S - S.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    o = p @ v
    cond_p = p @ np.abs(v)
    pA = p * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2))                       # p_k A_k  [B, H, Tq, Tk]
    cond_s = pA @ np.abs(v) + np.abs(o) * pA.sum(-1, keepdims=True)                # >= sum_k p_k A_k |v_k - o|
    tr = lambda a: a.transpose(0, 2, 1, 3).reshape(B * T, H * 64)                   # noqa: E731
    return tr(o), tr(cond_p), tr(cond_s)


def _vt_host(qkv, B, T, H):
    Q = H * 64
    v = qkv.reshape(B, T, 3, H, 64)[:, :, 2].transpose(0, 2, 3, 1)                 # [B, H, 64, T]
    vt = np.empty_like(v)
    vt[..., vt_key_slot(np.arange(T))] = v
    return np.ascontiguousarray(vt.reshape(B * H * 64, T))


# TC attention: P rounded to tf32 -> TOL_ATT_P on cond_p; scores in 3xTF32 (TF32): error of S relative to A_k
TOL_ATT_S = {True: 2.0 ** -16, False: 2.0 ** -10}
TOL_ATT_PV = {True: TOL_ATT_P, False: TOL_ATT_P}


@pytest.mark.parametrize("T,B,H,sharp,split3,lo", [
    (8, 3, 2, False, True, True), (24, 2, 2, True, True, False), (72, 2, 3, False, False, False), (128, 1, 2, True, True, True),
    (136, 2, 2, False, True, True), (200, 3, 2, True, True, True), (200, 2, 2, False, False, True), (256, 2, 2, True, False, False),
    (512, 2, 2, True, True, True), (768, 2, 2, True, True, True), (1024, 2, 1, True, True, False), (1024, 1, 2, False, False, True),
    (256, 32, 6, False, True, True)])
def test_enc_attention_tc(kh, T, B, H, sharp, split3, lo):
    """attention_tc_kernel in the encoder's form: partial query tiles and masked keys (T = 8, 24, 72, 136, 200), one and two key chunks,
    the key-split form with KS = 2, 3, 4 (T = 512, 768, 1024) and its combine kernel, 2 .. 768 work items (below and far
    above the SM count: the persistent loop's barrier parity over many items per CTA), both precisions, out_lo null and
    not.  Measured worst err/bound: 3xTF32 0.21, TF32 0.18."""
    assert kh.kh_enc_attention_tc_supported(T), f"T={T} is documented as supported"
    rng = np.random.default_rng(T * 7 + B)
    enc_attention_tc_check(kh, _attn_inputs(rng, B, T, H, sharp), B, T, H, split3, lo,
                           f"tc attention T={T} B={B} H={H} sharp={sharp} split3={split3}")


def enc_attention_tc_check(kh, qkv, B, T, H, split3, lo, name):
    """attention_tc_kernel (encoder form) on qkv [B*T, 3*H*64] against _attn_ref, per-element bars, NaN-poisoned outputs."""
    Q = H * 64
    vt = _vt_host(qkv, B, T, H)
    o_ref, cond_p, cond_s = _attn_ref(qkv, B, T, H)
    if split3:
        (qh, ql), (vh, vl) = _split(qkv), _split(vt)
        d = [_dev(qh), _dev(ql), _dev(vh), _dev(vl)]
    else:
        d = [_dev(qkv), None, _dev(vt), None]
    n_scr = kh.kh_enc_attention_tc_scratch_floats(B, T, H)
    scratch = _nan(n_scr) if n_scr else None
    oh, ol = _nan(B * T + 5, Q), (_nan(B * T + 5, Q) if lo else None)
    _call(kh, "kh_enc_attention_tc", *[_p(x) for x in d], B, T, H, _p(oh), _p(ol), int(split3), _p(scratch))
    got = oh[:B * T].double().cpu().numpy()
    if lo:
        got += ol[:B * T].double().cpu().numpy()
        assert (oh[:B * T].cpu().numpy().view(np.uint32) & 0x1FFF == 0).all()
    worst = _check(name, got, o_ref, cond_p, TOL_ATT_PV[split3], cond_s, TOL_ATT_S[split3])
    w = np.zeros(oh.shape, bool)
    w[:B * T] = True
    _assert_poison("out_hi", oh, w)
    if lo:
        _assert_poison("out_lo", ol, w)
    return worst


@pytest.mark.parametrize("T", [1, 37, 100, 300, 768])
def test_enc_attention_fp32(kh, T):
    """attention_fp32_kernel in the encoder's form (exact fp32; every T, the path of T % 8 != 0 and of T > 256 that is not a multiple of 256).
    Measured worst err/bound: 0.22."""
    B, H = 2, 2
    rng = np.random.default_rng(T)
    enc_attention_fp32_check(kh, _attn_inputs(rng, B, T, H, sharp=T % 2 == 0), B, T, H, f"fp32 attention T={T}")


def enc_attention_fp32_check(kh, qkv, B, T, H, name):
    """attention_fp32_kernel (encoder form) on qkv [B*T, 3*H*64] (rows past B*T NaN), with and without out_lo, against _attn_ref."""
    Q = H * 64
    o_ref, cond_p, cond_s = _attn_ref(qkv, B, T, H)
    buf = _nan(B * T + 8, 3 * Q)                               # rows past B*T: NaN the kernel must not read
    buf[:B * T] = _dev(qkv)
    worst = 0.0
    for lo in (False, True):
        oh, ol = _nan(B * T + 5, Q), (_nan(B * T + 5, Q) if lo else None)
        _call(kh, "kh_enc_attention_fp32", _p(buf), B, T, H, _p(oh), _p(ol))
        got = oh[:B * T].double().cpu().numpy() + (ol[:B * T].double().cpu().numpy() if lo else 0)
        worst = max(worst, _check(f"{name} lo={lo}", got, o_ref, cond_p, TOL_ENC_ATT_P, cond_s, TOL_ENC_ATT_S))
        w = np.zeros(oh.shape, bool)
        w[:B * T] = True
        _assert_poison("out", oh, w)
    return worst


# ------------------------------------------------------------------------------------------------
# decode GEMMs: sgemm_dec_cluster_kernel, sgemm_dec_kernel, sgemm_dec_cluster2_kernel
# ------------------------------------------------------------------------------------------------
def _dec_setup(M, N, K, epi, norm, seed, AW=None):
    rng = np.random.default_rng(seed)
    A = _pos_mean(rng, (M, K), 2.0)
    W = _pos_mean(rng, (K, N), 2.0 / K)
    if AW is not None:
        A, W = AW
    R = _pos_mean(rng, (M, N)) if epi == EPI_RESIDUAL else None
    rs = 1.0 / np.sqrt((A.astype(np.float64) ** 2).mean(1) + 1e-6) if norm else None
    ref, cond = _gemm_ref(A, W, rs, epi, R)
    return A, W, R, ref, cond


def _dec_run(kh, kernel, M, N, K, epi, norm, inplace, seed, kv=None, ssq=False, AW=None):
    A, W, R, ref, cond = _dec_setup(M, N, K, epi, norm, seed, AW)
    Nout = N // 2 if epi == EPI_GATED_GELU else N
    n_split = kv[0] if kv else N
    ncols = min(Nout, n_split)
    ldc = ncols + 4
    Cb = _nan(M + 3, ldc)
    ldr = 0
    Rd = None
    if R is not None:
        if inplace:
            Cb[:M, :N] = _dev(R)
            Rd, ldr = Cb, ldc
        else:
            Rd, ldr = _dev(R), N
    n_tiles = -(-N // 32)
    ssq_buf = _nan(M + 1, n_tiles + 1) if ssq else None
    dA, dW = _dev(A), _dev(W)
    partial = torch.empty((K // 64) * n_tiles * (64 * 32 + 64), dtype=torch.float32, device=DEV)
    counters = torch.zeros(n_tiles, dtype=torch.int32, device=DEV)
    f = dict(n_split=n_split)
    if kv:
        _, fmt, cap, H, C1, pos = kv
        f.update(C1=_p(C1), kv_fmt=fmt, hm_rows_per_b=1, hm_cap=cap, hm_H=H, hm_pos=_p(pos))
    a = DecGemmArgs(A=_p(dA), lda=K, W=_p(dW), ldw=N, M=M, N=N, K=K, norm=int(norm), eps=1e-6, epi=epi, R=_p(Rd), ldr=ldr,
                    C=_p(Cb), ldc=ldc, partial=_p(partial), counters=_p(counters), ssq_out=_p(ssq_buf), ssq_ld=n_tiles + 1, **f)
    _call(kh, kernel, C.byref(a))
    assert (counters.cpu().numpy() == 0).all()
    got = Cb[:M, :ncols].double().cpu().numpy()
    w = np.zeros(Cb.shape, bool)
    w[:M, :ncols] = True
    _assert_poison("C", Cb, w)
    return got, ref, cond, ssq_buf


DEC_CASES = [  # (M, N, K, epilogue, norm, in place): every cluster instantiation (K = 384 / 512 / 1024 -> KC 48 / 64 / 128,
    # K = 1024 with N <= 512 -> 16 CTAs of 64)
    (1, 36, 384, EPI_STORE, True, False), (5, 1516, 384, EPI_RESIDUAL, False, True), (63, 1536, 512, EPI_GATED_GELU, True, False),
    (64, 36, 1024, EPI_RESIDUAL, True, True), (64, 1536, 1024, EPI_GATED_GELU, False, False), (5, 1516, 1024, EPI_STORE, True, False),
    (63, 36, 512, EPI_GATED_GELU, False, False), (1, 1536, 512, EPI_RESIDUAL, True, True)]


@pytest.mark.parametrize("kernel", ["kh_dec_gemm_cluster", "kh_dec_gemm"])
@pytest.mark.parametrize("case", DEC_CASES, ids=lambda c: f"M{c[0]}-N{c[1]}-K{c[2]}-epi{c[3]}-norm{int(c[4])}")
def test_dec_gemm(kh, kernel, case):
    """The decode-step GEMMs (exact fp32): the cluster kernel and the split-K fallback, RMSNorm statistic from the A tiles,
    in-place residual, gated GELU, N not a multiple of 32; two launches are bit-identical.  Measured worst err/bound: 0.13."""
    M, N, K, epi, norm, inplace = case
    got, ref, cond, _ = _dec_run(kh, kernel, M, N, K, epi, norm, inplace, seed=M * 3 + K)
    _check(f"{kernel} {case}", got, ref, cond, TOL_DEC)
    again, _, _, _ = _dec_run(kh, kernel, M, N, K, epi, norm, inplace, seed=M * 3 + K)
    np.testing.assert_array_equal(again, got)


def test_dec_gemm_ssq_out(kh):
    """ssq_out: per (row, 32-column tile) sum of squares of the output row slice, against float64 sums of the output."""
    M, N, K = 63, 512, 384
    got, ref, cond, ssq = _dec_run(kh, "kh_dec_gemm_cluster", M, N, K, EPI_RESIDUAL, True, True, seed=3, ssq=True)
    _check("ssq gemm", got, ref, cond, TOL_DEC)
    s = ssq.cpu().numpy()
    want = (got.reshape(M, N // 32, 32) ** 2).sum(-1)
    _check("ssq_out", s[:M, :N // 32], want, want, TOL_DEC)
    w = np.zeros(s.shape, bool)
    w[:M, :N // 32] = True
    assert np.isnan(s[~w]).all()


@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("kernel", ["kh_dec_gemm_cluster", "kh_dec_gemm"])
def test_dec_gemm_kv_append(kh, kernel, fmt):
    """The fused K/V-cache append of the decode QKV projection (q to C, k and v to row `pos` of every (b, K|V, h)): at
    pos = 0, 31, 32, cap - 1 only that row changes, byte-for-byte the host encoding of the same kernel's fp32 output."""
    H, cap, K = 6, 48, 512
    Q = H * 64
    N = 3 * Q
    for M, pos in ((1, 0), (5, 31), (63, 32), (64, cap - 1)):
        full, ref, cond, _ = _dec_run(kh, kernel, M, N, K, EPI_STORE, True, False, seed=M)
        _check("unsplit", full, ref, cond, TOL_DEC)
        C1 = torch.full((M * 2 * H * cap * ROWB[fmt],), 255, dtype=torch.uint8, device=DEV)
        dpos = torch.tensor([pos], dtype=torch.int32, device=DEV)
        got, _, _, _ = _dec_run(kh, kernel, M, N, K, EPI_STORE, True, False, seed=M, kv=(Q, fmt, cap, H, C1, dpos))
        np.testing.assert_array_equal(got, full[:, :Q])
        kvb = C1.cpu().numpy().reshape(M, 2, H, cap, ROWB[fmt])
        want = encode_rows(full[:, Q:].astype(np.float32).reshape(M, 2, H, 64), fmt)
        np.testing.assert_array_equal(kvb[:, :, :, pos], want)
        others = np.ones(cap, bool)
        others[pos] = False
        assert (kvb[:, :, :, others] == 255).all(), f"rows other than pos={pos} changed"


def test_dec_gemm_out_q(kh):
    """sgemm_dec_cluster2_kernel: y' = y + o.Wo (with ssq_out) and q = [o | y].Wq' (two-source A, K0 = 384) in one launch."""
    rng = np.random.default_rng(9)
    M, Q, D = 37, 384, 512
    o, y = _pos_mean(rng, (M, Q)), _pos_mean(rng, (M, D))
    W0, W1 = _pos_mean(rng, (Q, D), 2.0 / Q), _pos_mean(rng, (Q + D, Q), 2.0 / (Q + D))
    ref0, cond0 = _gemm_ref(o, W0, None, EPI_RESIDUAL, y.astype(np.float64))
    ref1, cond1 = _gemm_ref(np.concatenate([o, y], 1), W1, None, EPI_STORE)
    do, dy, dW0, dW1 = _dev(o), _dev(y), _dev(W0), _dev(W1)
    C0, C1 = _nan(M + 2, D + 4), _nan(M + 2, Q + 4)
    ssq = _nan(M + 1, D // 32 + 1)
    a0 = DecGemmArgs(A=_p(do), lda=Q, W=_p(dW0), ldw=D, M=M, N=D, K=Q, epi=EPI_RESIDUAL, R=_p(dy), ldr=D, C=_p(C0), ldc=D + 4,
                     n_split=D, ssq_out=_p(ssq), ssq_ld=D // 32 + 1)
    a1 = DecGemmArgs(A=_p(do), lda=Q, W=_p(dW1), ldw=Q, M=M, N=Q, K=Q + D, epi=EPI_STORE, C=_p(C1), ldc=Q + 4, n_split=Q,
                     A2=_p(dy), lda2=D, K0=Q)
    _call(kh, "kh_dec_gemm_out_q", C.byref(a0), C.byref(a1))
    g0, g1 = C0[:M, :D].double().cpu().numpy(), C1[:M, :Q].double().cpu().numpy()
    _check("out", g0, ref0, cond0, TOL_DEC)
    _check("q", g1, ref1, cond1, TOL_DEC)
    want = (g0.reshape(M, D // 32, 32) ** 2).sum(-1)
    _check("ssq_out", ssq[:M, :D // 32].double().cpu().numpy(), want, want, TOL_DEC)
    for name, buf, n in (("C0", C0, D), ("C1", C1, Q)):
        w = np.zeros(buf.shape, bool)
        w[:M, :n] = True
        _assert_poison(name, buf, w)


# ------------------------------------------------------------------------------------------------
# decode attention: dec_attention_bulk_kernel<FMT>
# ------------------------------------------------------------------------------------------------
KT = {0: 32, 1: 64, 2: 64}
STAGES = {0: 6, 1: 6, 2: 4}


def _dec_attn_cases():
    out = []
    for fmt in (0, 1, 2):
        kt, st = KT[fmt], STAGES[fmt]
        for i, L in enumerate((1, kt - 1, kt, kt + 1, st * kt - 1, st * kt + 1, 1023, 1024)):
            out.append((fmt, L, 2, 2, 16 * (i % 2), i % 3 != 0, i % 2 == 0))
        out.append((fmt, 1024, 96, 2, 16, True, True))
    return out


@pytest.mark.parametrize("fmt,L,B,H,pf,ssq,len_ptr", _dec_attn_cases(),
                         ids=lambda v: str(v))
def test_dec_attention(kh, fmt, L, B, H, pf, ssq, len_ptr):
    """One query per (sequence, head) over L head-major K/V rows of format fmt; rows >= L inside cap are NaN and must not
    be read.  The reference is float64 over the DECODED stored rows, so every format meets the fp32 bar (the formats'
    own rounding is the codec test's).  len = *len_ptr + len_add, q scaled by rsqrt(sum q_ssq / q_dim + eps).
    Measured worst err/bound: 0.10."""
    H_ldq = H * 64 + 8
    rng = np.random.default_rng(L * 3 + fmt)
    rows = rng.standard_normal((B, 2, H, L, 64)).astype(np.float32) * np.float32(0.4)
    rows[:, 1] = rng.uniform(-0.5, 1.0, (B, H, L, 64))
    q = _pos_mean(rng, (B, H_ldq), 1.0)
    part = rng.uniform(100.0, 200.0, (B, 17)).astype(np.float32)
    dec_attention_check(kh, fmt, rows, q, part if ssq else None, pf, len_ptr, f"decode attention fmt={fmt} L={L} B={B}")


def dec_attention_check(kh, fmt, rows, q, part, pf, len_ptr, name, q_off=4, qd=512.0, eps=1e-6):
    """dec_attention_bulk_kernel<fmt> on K/V rows [B, 2, H, L, 64] (fp32 values, stored in format fmt; rows past L inside
    cap NaN) and queries q [B, ldq] (head h at columns q_off + 64 h), scaled by rsqrt(sum part[:, :-1] / qd + eps) when
    part [B, n + 1] is given, against float64 over the DECODED stored rows."""
    B, _, H, L, _ = rows.shape
    cap, ldq, ldo = L + 9, q.shape[1], H * 64 + 4
    kvb = np.full((B, 2, H, cap, ROWB[fmt]), 255, np.uint8)
    kvb[:, :, :, :L] = encode_rows(rows, fmt)
    kv_vals = decode_rows(kvb[:, :, :, :L], fmt)                   # what is stored
    n_ssq = 0 if part is None else part.shape[1] - 1
    rs = np.ones(B) if part is None else 1.0 / np.sqrt(part[:, :n_ssq].astype(np.float64).sum(1) / qd + eps)
    qh = q[:, q_off:q_off + H * 64].astype(np.float64).reshape(B, H, 64) * rs[:, None, None]
    k, v = kv_vals[:, 0], kv_vals[:, 1]
    S = np.einsum("bhd,bhkd->bhk", qh, k)
    p = np.exp(S - S.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    o = np.einsum("bhk,bhkd->bhd", p, v)
    cond_p = np.einsum("bhk,bhkd->bhd", p, np.abs(v))
    pA = p * np.einsum("bhd,bhkd->bhk", np.abs(qh), np.abs(k))
    cond_s = np.einsum("bhk,bhkd->bhd", pA, np.abs(v)) + np.abs(o) * pA.sum(-1, keepdims=True)
    d_kv = _dev(kvb.reshape(-1))
    d_q, d_ssq = _dev(q), (_dev(part) if part is not None else None)
    lenp = torch.tensor([L - 1], dtype=torch.int32, device=DEV) if len_ptr else None
    out = _nan(B + 1, ldo)
    _call(kh, "kh_dec_attention", fmt, _p(d_q), ldq, q_off, _p(d_kv), H, cap, _p(lenp), 1 if len_ptr else L, L, _p(out), ldo,
          _p(d_ssq), n_ssq, n_ssq + 1, qd, eps, pf, B)
    got = out[:B, :H * 64].double().cpu().numpy()
    worst = _check(name, got, o.reshape(B, H * 64), cond_p.reshape(B, H * 64), TOL_DEC_ATT_P, cond_s.reshape(B, H * 64),
                   TOL_DEC_ATT_S)
    w = np.zeros(out.shape, bool)
    w[:B, :H * 64] = True
    _assert_poison("out", out, w)
    return S, worst


# ------------------------------------------------------------------------------------------------
# p24 codec: kv_store<N> -> p24_elt
# ------------------------------------------------------------------------------------------------
def _p24_test_set():
    rng = np.random.default_rng(24)
    bits = [rng.integers(0, 2 ** 32, 2 ** 24, dtype=np.uint64).astype(np.uint32)]
    e = np.arange(256, dtype=np.uint32) << np.uint32(23)
    special = [np.array([0, 0x80000000, 1, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000],
                        np.uint32),
               e, e | np.uint32(0x7FFFFF), e | np.uint32(0x80000000), e | np.uint32(0x807FFFFF)]
    # halfway between neighbouring p24 values (and one bit either side)
    t = rng.integers(0, 2 ** 24, 4096, dtype=np.uint64)
    lo, hi = _p24_decode_bits(t).astype(np.uint64), _p24_decode_bits(t + 1).astype(np.uint64)
    mid = (lo + hi) // 2
    special += [(x & 0xFFFFFFFF).astype(np.uint32) for x in (mid, mid + 1, mid - 1)]
    x = np.concatenate(bits + special)
    x = x[: len(x) // 8 * 8]
    return x.view(np.float32)


@pytest.fixture(scope="module")
def p24_set():
    x = _p24_test_set()
    fin = np.isfinite(x)
    return x, fin, p24_encode_ref(np.where(fin, x, 0).astype(np.float32))


@pytest.mark.parametrize("N", [1, 2, 4])
def test_p24_codec(kh, p24_set, N):
    """kv_store<N> (p24 rows) -> p24_elt over >= 2^24 random bit patterns plus +-0, denormals, the first and last mantissa
    of every exponent, +-max finite, +-inf and values halfway between neighbours: the code is bit-exactly the nearest
    p24 value (numpy restatement), |rel err| < 2^-16 for normals (measured 1.526e-5 = 2^-16 (1 - 2^-15)), finite never
    becomes inf or NaN, inf stays inf."""
    x, fin, want = p24_set
    dx = _dev(x)
    y = torch.empty_like(dx)
    code = torch.empty(x.shape, dtype=torch.int32, device=DEV)
    _call(kh, "kh_p24_roundtrip", _p(dx), _p(y), _p(code), x.size, N)
    yc, cc = y.cpu().numpy(), code.cpu().numpy().view(np.uint32)
    np.testing.assert_array_equal(cc[fin], want[fin])
    np.testing.assert_array_equal(yc.view(np.uint32), _p24_decode_bits(cc))
    assert np.isfinite(yc[fin]).all()
    inf = np.isinf(x)
    np.testing.assert_array_equal(yc[inf], x[inf])
    normal = fin & (np.abs(x) >= np.finfo(np.float32).tiny)
    rel = np.abs(yc[normal].astype(np.float64) - x[normal]) / np.abs(x[normal].astype(np.float64))
    print(f"p24 N={N}: max rel err {rel.max():.3e}")
    assert rel.max() < 2.0 ** -16


# ------------------------------------------------------------------------------------------------
# ragged shapes through the model (network.Transformer against the float64 oracle)
# ------------------------------------------------------------------------------------------------
LOGIT_TOL = 5e-4


def _ragged_model_check(T, B, gm, vocab, steps=4, seed=0, emb_dim=512, num_heads=6, mlp_dim=1024):
    from mt3_b200 import network
    from oracle import mt3_oracle as O
    ocfg = O.T5Config(vocab_size=vocab, num_encoder_layers=1, num_decoder_layers=2, emb_dim=emb_dim, num_heads=num_heads,
                      mlp_dim=mlp_dim)
    params = O.init_params(ocfg, seed=seed, norm_scale_jitter=0.05)
    cfg = network.T5Config(vocab_size=vocab, emb_dim=emb_dim, num_heads=num_heads, num_encoder_layers=1, num_decoder_layers=2,
                           head_dim=64, mlp_dim=mlp_dim, mlp_activations=('gelu', 'linear'))
    m = network.Transformer(cfg, params, device=DEV, max_batch=B, max_input_length=T, max_decode_length=steps + 4, gemm_mode=gm)
    audio = np.stack([O.sine_mix(T * 128, seed=500 + seed + i) for i in range(B)])
    x = O.compute_spectrogram(audio, np.float32)[:, :T]
    assert x.shape[1] == T
    pick = sorted({0, B // 2, B - 1})
    enc = m.encode(torch.from_numpy(x).to(DEV))
    enc64 = O.encode(params, ocfg, x[pick], np.float64)
    e_enc = np.abs(enc.cpu().numpy()[pick] - enc64).max() / np.abs(enc64).max()
    toks64, l64 = O.greedy_decode(params, ocfg, enc64, steps, np.float64, stop_at_eos=False, return_logits=True)
    dec_in = np.zeros((B, steps), np.int64)
    dec_in[pick, 1:] = toks64[:, :steps - 1]
    lg = m.teacher_forced_logits(enc, torch.from_numpy(dec_in).to(DEV).to(torch.int32)).cpu().numpy()[pick]
    scale = np.abs(l64).max()
    e = np.abs(lg - l64).max() / scale
    print(f"model T={T} B={B} gemm={gm} vocab={vocab} D={emb_dim} H={num_heads} F={mlp_dim}: encoder {e_enc:.2e} logits {e:.2e} (of max)")
    assert e_enc <= LOGIT_TOL and e <= LOGIT_TOL
    out = m.generate(torch.from_numpy(x).to(DEV), num_steps=steps, stop_at_eos=False, use_graph=False).cpu().numpy()[pick]
    srt = np.sort(l64, axis=-1)
    safe = np.cumprod((srt[..., -1] - srt[..., -2]) > 2 * e * scale, axis=1).astype(bool)
    np.testing.assert_array_equal(out[:, :steps][safe], toks64[:, :steps][safe])


@pytest.mark.parametrize("gm", ["tf32x3", "simt"])
@pytest.mark.parametrize("T", [1, 37, 100, 200, 300, 768])
def test_model_ragged_input_length(T, gm):
    """Input lengths that pick different encoder attention paths: T = 1, 37 (exact fp32: T % 8 != 0, no V^T operand),
    100 (T % 8 != 0, T % 4 == 0), 200 (TC, partial query tile and masked keys), 300 (exact fp32: T > 256 and not a multiple
    of 256), 768 (TC key-split with 3 parts); 1 encoder and 2 decoder layers against the float64 oracle."""
    from mt3_b200 import _lib
    _ragged_model_check(T, 2, {"tf32x3": _lib.GEMM_TF32X3, "simt": _lib.GEMM_FP32_SIMT}[gm], 1536, seed=T)


@pytest.mark.parametrize("B,vocab", [(65, 1516), (96, 1536)])
def test_model_batch_above_64(B, vocab):
    """B > 64: the decode GEMMs run in 64-row blocks and the fused out+query GEMM declines; vocab 1516 leaves the logits
    GEMM a partial 32-column tile (and the argmax / vocabulary decode a ragged row)."""
    from mt3_b200 import _lib
    _ragged_model_check(32, B, _lib.GEMM_TF32X3, vocab, seed=B)


@pytest.mark.parametrize("B", [5, 65])
def test_model_width_off_cluster_tiling(B):
    """4 heads (Q = 256): the self- and cross-attention out-projections (K = 256 does not split into 8 chunks of 48, 64 or
    128) run on the non-cluster split-K decode GEMM, the other decode GEMMs on clusters, and the fused out+query GEMM
    declines (it is built for Q = 384, D = 512)."""
    from mt3_b200 import _lib
    _ragged_model_check(32, B, _lib.GEMM_TF32X3, 1536, seed=B, emb_dim=512, num_heads=4, mlp_dim=1024)
