"""Decode GEMMs with the tensor-core multiply (-m gpu): sgemm_dec_cluster_kernel and sgemm_dec_cluster2_kernel with the
3xTF32 wgmma multiply (decode.cuh, dec_mma_3xtf32), the decoder's path in gemm modes TF32X3 and TF32, launched alone
through the harness library (kh_dec_gemm_cluster_tc, kh_dec_gemm_out_q_tc) against the float64 reference, per-element
condition bars, positive-mean inputs and NaN-poisoned outputs of test_kernel_parity.py.

Bar: 2^-17 of cond = rs * sum_k |a_k b_k|.  Per product the dropped lo.lo term and the lo operands read as tf32 cost
<= 3 * 2^-22; the fp32 sums -- the tensor core's over the KC / 8 k-steps of a CTA (its adds may truncate: 2^-23 each),
hi.hi + (lo.hi + hi.lo), and the rank-ordered sum over the 8 or 16 CTAs -- add <= 32 * 2^-23; together < 2^-17.
Worst err/bound measured on an H100 80GB HBM3 (700 W): 0.31 (GEMM outputs), 0.12 of TOL_DEC for ssq_out.

Row independence: a row's output depends on that row's inputs only, bit for bit, wherever it sits in the 64-row tile
and whatever the other rows hold -- the decode loop's batch invariance rests on it.
"""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

import test_kernel_parity as kp

pytestmark = pytest.mark.gpu

DEV = kp.DEV
EPI_STORE, EPI_RESIDUAL, EPI_GATED_GELU = kp.EPI_STORE, kp.EPI_RESIDUAL, kp.EPI_GATED_GELU
TOL = 2.0 ** -17


@pytest.fixture(scope="module")
def kh():
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(kp.TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I = C.c_void_p, C.c_int
    sig = {"kh_last_error": ([], C.c_char_p), "kh_sizeof": ([I], C.c_longlong), "kh_dec_gemm_cluster_tc": ([P], I),
           "kh_dec_gemm_out_q_tc": ([P, P], I)}
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    assert lib.kh_sizeof(2) == C.sizeof(kp.DecGemmArgs), "ctypes mirror of DecGemmArgs does not match the C layout"
    return lib


@pytest.mark.parametrize("case", kp.DEC_CASES, ids=lambda c: f"M{c[0]}-N{c[1]}-K{c[2]}-epi{c[3]}-norm{int(c[4])}")
def test_dec_gemm_tc(kh, case):
    """Every cluster instantiation (KC 48 / 64 / 128, clusters of 16 for K = 1024 narrow), every epilogue, N not a
    multiple of 32, M = 1 / 5 / 63 / 64, in-place residual; a repeat launch is bit-identical."""
    M, N, K, epi, norm, inplace = case
    got, ref, cond, _ = kp._dec_run(kh, "kh_dec_gemm_cluster_tc", M, N, K, epi, norm, inplace, seed=M * 3 + K)
    kp._check(f"tc {case}", got, ref, cond, TOL)
    again, _, _, _ = kp._dec_run(kh, "kh_dec_gemm_cluster_tc", M, N, K, epi, norm, inplace, seed=M * 3 + K)
    np.testing.assert_array_equal(again, got)


def test_dec_gemm_tc_ssq_out(kh):
    """ssq_out of the tensor-core path: per (row, 32-column tile) sums of squares of the output it wrote."""
    M, N, K = 63, 512, 384
    got, ref, cond, ssq = kp._dec_run(kh, "kh_dec_gemm_cluster_tc", M, N, K, EPI_RESIDUAL, True, True, seed=3, ssq=True)
    kp._check("tc ssq gemm", got, ref, cond, TOL)
    s = ssq.cpu().numpy()
    want = (got.reshape(M, N // 32, 32) ** 2).sum(-1)
    kp._check("tc ssq_out", s[:M, :N // 32], want, want, kp.TOL_DEC)
    w = np.zeros(s.shape, bool)
    w[:M, :N // 32] = True
    assert np.isnan(s[~w]).all()


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_dec_gemm_tc_kv_append(kh, fmt):
    """The fused K/V-cache append in the fp32 / fp16 / p24 row formats: at pos = 0, 31, 32, cap - 1 only that row
    changes, byte-for-byte the host encoding of the same kernel's unsplit output."""
    H, cap, K = 6, 48, 512
    Q = H * 64
    N = 3 * Q
    for M, pos in ((1, 0), (5, 31), (63, 32), (64, cap - 1)):
        full, ref, cond, _ = kp._dec_run(kh, "kh_dec_gemm_cluster_tc", M, N, K, EPI_STORE, True, False, seed=M)
        kp._check("tc unsplit", full, ref, cond, TOL)
        C1 = torch.full((M * 2 * H * cap * kp.ROWB[fmt],), 255, dtype=torch.uint8, device=DEV)
        dpos = torch.tensor([pos], dtype=torch.int32, device=DEV)
        got, _, _, _ = kp._dec_run(kh, "kh_dec_gemm_cluster_tc", M, N, K, EPI_STORE, True, False, seed=M,
                                   kv=(Q, fmt, cap, H, C1, dpos))
        np.testing.assert_array_equal(got, full[:, :Q])
        kvb = C1.cpu().numpy().reshape(M, 2, H, cap, kp.ROWB[fmt])
        want = kp.encode_rows(full[:, Q:].astype(np.float32).reshape(M, 2, H, 64), fmt)
        np.testing.assert_array_equal(kvb[:, :, :, pos], want)
        others = np.ones(cap, bool)
        others[pos] = False
        assert (kvb[:, :, :, others] == 255).all(), f"rows other than pos={pos} changed"


def _out_q(kh, o, y, W0, W1):
    M, Q = o.shape
    D = y.shape[1]
    do, dy, dW0, dW1 = kp._dev(o), kp._dev(y), kp._dev(W0), kp._dev(W1)
    C0, C1 = kp._nan(M + 2, D + 4), kp._nan(M + 2, Q + 4)
    ssq = kp._nan(M + 1, D // 32 + 1)
    P = kp._p
    a0 = kp.DecGemmArgs(A=P(do), lda=Q, W=P(dW0), ldw=D, M=M, N=D, K=Q, epi=EPI_RESIDUAL, R=P(dy), ldr=D, C=P(C0), ldc=D + 4,
                        n_split=D, ssq_out=P(ssq), ssq_ld=D // 32 + 1)
    a1 = kp.DecGemmArgs(A=P(do), lda=Q, W=P(dW1), ldw=Q, M=M, N=Q, K=Q + D, epi=EPI_STORE, C=P(C1), ldc=Q + 4, n_split=Q,
                        A2=P(dy), lda2=D, K0=Q)
    kp._call(kh, "kh_dec_gemm_out_q_tc", C.byref(a0), C.byref(a1))
    return C0, C1, ssq


def test_dec_gemm_out_q_tc(kh):
    """sgemm_dec_cluster2_kernel (KC 48 and 112): y' = y + o.Wo with ssq_out and q = [o | y].Wq' (two-source A) in one
    launch; a repeat launch is bit-identical."""
    rng = np.random.default_rng(9)
    M, Q, D = 37, 384, 512
    o, y = kp._pos_mean(rng, (M, Q)), kp._pos_mean(rng, (M, D))
    W0, W1 = kp._pos_mean(rng, (Q, D), 2.0 / Q), kp._pos_mean(rng, (Q + D, Q), 2.0 / (Q + D))
    ref0, cond0 = kp._gemm_ref(o, W0, None, EPI_RESIDUAL, y.astype(np.float64))
    ref1, cond1 = kp._gemm_ref(np.concatenate([o, y], 1), W1, None, EPI_STORE)
    C0, C1, ssq = _out_q(kh, o, y, W0, W1)
    g0, g1 = C0[:M, :D].double().cpu().numpy(), C1[:M, :Q].double().cpu().numpy()
    kp._check("tc out", g0, ref0, cond0, TOL)
    kp._check("tc q", g1, ref1, cond1, TOL)
    want = (g0.reshape(M, D // 32, 32) ** 2).sum(-1)
    kp._check("tc ssq_out", ssq[:M, :D // 32].double().cpu().numpy(), want, want, kp.TOL_DEC)
    for name, buf, n in (("C0", C0, D), ("C1", C1, Q)):
        w = np.zeros(buf.shape, bool)
        w[:M, :n] = True
        kp._assert_poison(name, buf, w)
    D0, D1, _ = _out_q(kh, o, y, W0, W1)
    assert torch.equal(D0[:M, :D], C0[:M, :D]) and torch.equal(D1[:M, :Q], C1[:M, :Q])


def _cluster(kh, A, W, epi, norm):
    M, K = A.shape
    N = W.shape[1]
    Nout = N // 2 if epi == EPI_GATED_GELU else N
    dA, dW = kp._dev(A), kp._dev(W)
    Cb = kp._nan(M, Nout)
    a = kp.DecGemmArgs(A=kp._p(dA), lda=K, W=kp._p(dW), ldw=N, M=M, N=N, K=K, norm=int(norm), eps=1e-6, epi=epi, C=kp._p(Cb),
                       ldc=Nout, n_split=N)
    kp._call(kh, "kh_dec_gemm_cluster_tc", C.byref(a))
    return Cb.cpu().numpy()


@pytest.mark.parametrize("N,K,epi", [(1152, 384, EPI_STORE), (1536, 512, EPI_GATED_GELU), (512, 1024, EPI_STORE),
                                     (1536, 1024, EPI_STORE)], ids=["KC48", "KC64", "KC64-S16", "KC128"])
def test_dec_gemm_tc_rows_independent(kh, N, K, epi):
    """Row x gives the same bits at row 0 of M = 1, row 39 of M = 40 and row 63 of M = 64, with different rows around it
    (the RMSNorm statistic included)."""
    rng = np.random.default_rng(K + N)
    W = kp._pos_mean(rng, (K, N), 2.0 / K)
    x = kp._pos_mean(rng, (1, K), 2.0)
    outs = []
    for M in (1, 40, 64):
        A = kp._pos_mean(rng, (M, K), 2.0)
        A[M - 1] = x[0]
        outs.append(_cluster(kh, A, W, epi, True)[M - 1])
    assert np.isfinite(outs[0]).all()
    np.testing.assert_array_equal(outs[1], outs[0])
    np.testing.assert_array_equal(outs[2], outs[0])


def test_dec_gemm_out_q_tc_rows_independent(kh):
    """The same for both halves of the out+q launch."""
    rng = np.random.default_rng(5)
    Q, D = 384, 512
    W0, W1 = kp._pos_mean(rng, (Q, D), 2.0 / Q), kp._pos_mean(rng, (Q + D, Q), 2.0 / (Q + D))
    xo, xy = kp._pos_mean(rng, (Q,)), kp._pos_mean(rng, (D,))
    outs = []
    for M in (1, 40, 64):
        o, y = kp._pos_mean(rng, (M, Q)), kp._pos_mean(rng, (M, D))
        o[M - 1], y[M - 1] = xo, xy
        C0, C1, ssq = _out_q(kh, o, y, W0, W1)
        outs.append((C0[M - 1, :D].cpu().numpy(), C1[M - 1, :Q].cpu().numpy(), ssq[M - 1, :D // 32].cpu().numpy()))
    for got in outs[1:]:
        for g, want in zip(got, outs[0]):
            np.testing.assert_array_equal(g, want)
