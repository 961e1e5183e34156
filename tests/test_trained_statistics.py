"""The model and its decode kernels at the value statistics of a trained checkpoint, against float64.

Every other model test runs random-init weights: norm scales 1 +- 0.05, no outlier channels in the residual stream, diffuse
attention (scores of order 1).  A trained checkpoint need not be that mild (DESIGN.md section 4), and none can be loaded
here, so `trained_params` makes synthetic weights with trained statistics from the random-init ones by documented,
deterministic transforms:

  norm scales    exp(N(0, 1)) clipped to [0.05, 20]
  outliers       three residual-stream channels made 30-300x the median by scaling those output columns of every
                 attention-out and MLP-out kernel
  heads          per layer two diffuse, two sharp and two sink heads (the kind rotates with the layer), made by rank-1
                 additions to the query and key kernels of the encoder, the decoder self- and the cross-attention:
                 sharp  q and k along one direction, S_ij ~ c z_i z_j: row maxima 30-300, many above 88.7 (where e^S
                        overflows fp32 without the max subtraction)
                 sink   q along the mean of the normalised inputs (the same sign for every query), k along the
                        regularised Fisher discriminant of position 0 against the others: most of the mass on key 0
  MLP gates      wi_0 scaled so that the gate pre-activations span about +-10
  logits         the EOS column scaled so that EOS is the argmax at EOS_RATE of the calibration positions: reachable,
                 and sequences end at scattered steps

The directions and scales are calibrated layer by layer on the float64 oracle's activations for sine-mix audio and random
tokens (CAL_SEEDS); the tests measure on other inputs.  test_generator_statistics (no GPU) asserts that the weights really
are in that regime.  The GPU tests hold the decode attention, the decode GEMMs, the gated-GELU epilogues and the encoder
attention to the per-element bars of test_kernel_parity.py at such values, and the full model to the bars of DESIGN.md
section 4 wherever the float32 oracle is well-conditioned: these weights make the late decoder positions chaotic, the
float32 oracle itself far from float64 there, and no float32 implementation can be held to a bar at them.
"""
import functools
import os

import numpy as np
import pytest

import test_kernel_parity as kp
from oracle import mt3_oracle as O

CFG = O.T5Config()
D, NH, DH = CFG.emb_dim, CFG.num_heads, CFG.head_dim
KINDS = ("diffuse", "sharp", "sink")
OUT_CH = (37, 211, 400)              # the outlier channels of the residual stream
OUT_F = (40.0, 100.0, 250.0)         # their out-kernel column scales
GATE_SPAN = 10.0                     # largest |gate pre-activation| per layer on the calibration inputs
SHARP_C = (20.0, 45.0)               # sharp heads: S ~ c z_i z_j, z of unit variance
SINK_C = 24.0                        # sink heads: score per standard deviation of the key feature
FISHER_LAM = 1e-2                    # ridge of the position-0 discriminant, relative to the mean variance
EOS_RATE = 0.02
CAL_SEEDS = (9100, 9101, 9102, 9103)
OVERFLOW = 88.72                     # ln(FLT_MAX)


def head_kind(layer, h):
    return KINDS[(h + layer) % 3]


def spectrogram(seeds, t=256):
    audio = np.stack([O.sine_mix(t * 128, seed=s) for s in seeds])
    return O.compute_spectrogram(audio, np.float32)[:, :t]


def _unit(v):
    return v / np.linalg.norm(v)


def _add_heads(p, prefix, layer, Uq, Uk, rng):
    """Rank-1 additions to the query / key kernels of the sharp and sink heads of one attention.  Uq [N, D]: the rows the
    query kernel sees; Uk [B, T, D]: the rows the key kernel sees, position axis kept (key 0 is the sink)."""
    Wq, Wk = p[prefix + "query/kernel"], p[prefix + "key/kernel"]
    kf = Uk.reshape(-1, D)
    for h in range(NH):
        kind = head_kind(layer, h)
        e = _unit(rng.standard_normal(DH))
        cols = slice(h * DH, (h + 1) * DH)
        if kind == "sharp":
            a = rng.standard_normal(D)
            m = _unit(kf.mean(0))
            a = _unit(a - (a @ m) * m)                   # no common part: the sign of z varies over the keys
            c = rng.uniform(*SHARP_C)
            Wq[:, cols] += np.sqrt(c) / (Uq @ a).std() * np.outer(a, e)
            Wk[:, cols] += np.sqrt(c) / (kf @ a).std() * np.outer(a, e)
        elif kind == "sink":
            a = _unit(Uq.mean(0))
            zq = (Uq @ a).mean()
            rest = Uk[:, 1:].reshape(-1, D)
            mu = rest.mean(0)
            cov = np.cov(rest.T)
            v = np.linalg.solve(cov + FISHER_LAM * np.trace(cov) / D * np.eye(D), Uk[:, 0].mean(0) - mu)
            sd = ((rest - mu) @ v).std()
            Wq[:, cols] += (1.0 / zq) * np.outer(a, e)
            Wk[:, cols] += (SINK_C / sd) * np.outer(v, e)


def _scale_gate(p, prefix, M):
    g = M.reshape(-1, D) @ p[prefix + "mlp/wi_0/kernel"]
    p[prefix + "mlp/wi_0/kernel"] *= GATE_SPAN / np.abs(g).max()


def _attn(p, prefix, xq, xkv, mask):
    return O.mha(p, prefix, xq, xkv, NH, DH, mask=mask)


def _mlp(p, prefix, m):
    return O.mlp_block(m, [p[prefix + "mlp/wi_0/kernel"], p[prefix + "mlp/wi_1/kernel"]], p[prefix + "mlp/wo/kernel"],
                       CFG.mlp_activations)


@functools.lru_cache(maxsize=None)
def trained_params(seed=0):
    """float32 weights with trained statistics (module docstring), deterministic in `seed`."""
    p = {k: v.astype(np.float64) for k, v in O.init_params(CFG, seed).items()}
    rng = np.random.default_rng(seed + 7919)
    for k in sorted(p):
        if k.endswith("/scale"):
            p[k] = np.clip(np.exp(rng.standard_normal(p[k].shape)), 0.05, 20.0)
    for k in sorted(p):
        if k.endswith("out/kernel") or k.endswith("mlp/wo/kernel"):
            for c, f in zip(OUT_CH, OUT_F):
                p[k][:, c] *= f
    # encoder, layer by layer on the calibration inputs
    x = spectrogram(CAL_SEEDS).astype(np.float64)
    B, T = x.shape[:2]
    pe = O.sinusoidal_table(2048, D).astype(np.float64)
    h = x @ p["encoder/continuous_inputs_projection/kernel"] + pe[None, :T]
    ones = np.ones((B, 1, T, T))
    for i in range(CFG.num_encoder_layers):
        pre = f"encoder/layers_{i}/"
        u = O.rms_norm(h, p[pre + "pre_attention_layer_norm/scale"])
        _add_heads(p, pre + "attention/", i, u.reshape(-1, D), u, rng)
        h = h + _attn(p, pre + "attention/", u, u, ones)
        m = O.rms_norm(h, p[pre + "pre_mlp_layer_norm/scale"])
        _scale_gate(p, pre, m)
        h = h + _mlp(p, pre, m)
    enc = O.rms_norm(h, p["encoder/encoder_norm/scale"])
    # decoder, teacher-forced on random tokens
    L = 64
    toks = np.random.default_rng(seed + 31).integers(3, 1500, size=(B, L))
    toks[:, 0] = 0
    y = p["decoder/token_embedder/embedding"][toks] + pe[None, :L]
    causal = np.tril(np.ones((L, L)))[None, None]
    for i in range(CFG.num_decoder_layers):
        pre = f"decoder/layers_{i}/"
        a = O.rms_norm(y, p[pre + "pre_self_attention_layer_norm/scale"])
        _add_heads(p, pre + "self_attention/", i, a.reshape(-1, D), a, rng)
        y = y + _attn(p, pre + "self_attention/", a, a, causal)
        c = O.rms_norm(y, p[pre + "pre_cross_attention_layer_norm/scale"])
        _add_heads(p, pre + "encoder_decoder_attention/", i, c.reshape(-1, D), enc, rng)
        y = y + _attn(p, pre + "encoder_decoder_attention/", c, enc, None)
        m = O.rms_norm(y, p[pre + "pre_mlp_layer_norm/scale"])
        _scale_gate(p, pre, m)
        y = y + _mlp(p, pre, m)
    lg = O.rms_norm(y, p["decoder/decoder_norm/scale"]) @ p["decoder/logits_dense/kernel"]
    e = lg[..., O.EOS_ID]
    others = np.delete(lg, O.EOS_ID, axis=-1).max(-1)
    # EOS wins where boost * e > others, i.e. where others / e < boost (e > 0)
    boost = np.quantile(np.where(e > 0, others / np.where(e > 0, e, 1.0), np.inf), EOS_RATE)
    p["decoder/logits_dense/kernel"][:, O.EOS_ID] *= boost
    return {k: np.ascontiguousarray(v, np.float32) for k, v in p.items()}


# ------------------------------------------------------------------------------------------------
# the statistics of the generated weights (float64 oracle, no GPU)
# ------------------------------------------------------------------------------------------------
def _scores(q, k, mask=None):
    """[B, Tq, H*64] x [B, Tk, H*64] -> [B, H, Tq, Tk] float64 scores, -inf where masked"""
    B, Tq, Tk = q.shape[0], q.shape[1], k.shape[1]
    S = np.einsum("bqhd,bkhd->bhqk", q.reshape(B, Tq, NH, DH), k.reshape(B, Tk, NH, DH))
    return S if mask is None else np.where(mask, S, -np.inf)


def layer0_scores(params, x, toks):
    """Layer-0 scores of the encoder, the decoder self- and the cross-attention (float64)."""
    p = {k: v.astype(np.float64) for k, v in params.items()}
    B, T = x.shape[:2]
    L = toks.shape[1]
    pe = O.sinusoidal_table(2048, D).astype(np.float64)
    h = x.astype(np.float64) @ p["encoder/continuous_inputs_projection/kernel"] + pe[None, :T]
    pre = "encoder/layers_0/"
    u = O.rms_norm(h, p[pre + "pre_attention_layer_norm/scale"])
    s_enc = _scores(u @ p[pre + "attention/query/kernel"], u @ p[pre + "attention/key/kernel"])
    enc = O.encode(params, CFG, x, np.float64)
    pre = "decoder/layers_0/"
    y = p["decoder/token_embedder/embedding"][toks] + pe[None, :L]
    a = O.rms_norm(y, p[pre + "pre_self_attention_layer_norm/scale"])
    causal = np.tril(np.ones((L, L), bool))[None, None]
    s_self = _scores(a @ p[pre + "self_attention/query/kernel"], a @ p[pre + "self_attention/key/kernel"], causal)
    y = y + _attn(p, pre + "self_attention/", a, a, causal.astype(np.float64))
    c = O.rms_norm(y, p[pre + "pre_cross_attention_layer_norm/scale"])
    s_cross = _scores(c @ p[pre + "encoder_decoder_attention/query/kernel"], enc @ p[pre + "encoder_decoder_attention/key/kernel"])
    return {"encoder": s_enc, "decoder self": s_self, "cross": s_cross}


def _softmax(S):
    e = np.exp(S - S.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def encoder_activations(params, x):
    """Per encoder layer: the residual stream after it [B, T, D] and the gate pre-activations of its MLP."""
    p = {k: v.astype(np.float64) for k, v in params.items()}
    _, layers = O.encode(params, CFG, x, np.float64, return_layers=True)
    T = x.shape[1]
    ones = np.ones((x.shape[0], 1, T, T))
    gates = []
    for i, h in enumerate(layers[:-1]):
        pre = f"encoder/layers_{i}/"
        u = O.rms_norm(h, p[pre + "pre_attention_layer_norm/scale"])
        hm = h + _attn(p, pre + "attention/", u, u, ones)
        gates.append(O.rms_norm(hm, p[pre + "pre_mlp_layer_norm/scale"]) @ p[pre + "mlp/wi_0/kernel"])
    return layers[1:], gates


def test_generator_statistics():
    """The generated weights are in the trained regime on inputs other than the calibration ones (sine mixes 1234, 1235;
    random tokens), and stay there.  Sharp heads of every layer-0 attention: at least 10 % of the score rows peak above
    88.7, the median row maximum lies in 30 .. 300, at least 30 % of the rows peak in 30 .. 300 and none above 1500.
    Sink heads: key 0 takes the larger part of the mass.  Diffuse heads: row maxima below 50.  After every encoder
    layer the largest residual channel is 30 .. 300x the median one, and the 99.9th percentile of |gate pre-activation|
    lies in 5 .. 15.  EOS is the float64 argmax at 0.5 .. 8 % of the teacher-forced positions."""
    params = trained_params()
    x = spectrogram((1234, 1235))
    toks = np.random.default_rng(12).integers(3, 1500, size=(2, 128))
    toks[:, 0] = 0
    S = layer0_scores(params, x, toks)
    bad = []
    for name, s in S.items():
        kinds = np.array([head_kind(0, h) for h in range(NH)])
        mx = s.max(-1)                                                    # [B, H, Tq]
        sharp, sink, diffuse = mx[:, kinds == "sharp"], s[:, kinds == "sink"], mx[:, kinds == "diffuse"]
        over = float((sharp > OVERFLOW).mean())
        med = float(np.median(sharp))
        q95 = float(np.quantile(sharp, 0.95))
        inside = float(((sharp >= 30) & (sharp <= 300)).mean())
        key0 = float(_softmax(sink)[..., 0].mean())
        print(f"{name:12s}: sharp heads: row max median {med:6.1f}, 95th percentile {q95:6.1f}, max {sharp.max():6.1f}, in 30 .. 300 {inside:5.1%}, rows above 88.7 {over:5.1%};  "
              f"sink heads: mass on key 0 {key0:.3f};  diffuse heads: row max {diffuse.max():5.1f}")
        ok = over >= 0.1 and 30 <= med <= 300 and inside >= 0.3 and sharp.max() <= 1500
        bad += [] if ok else [(name, "sharp", over, med, inside, float(sharp.max()))]
        bad += [] if key0 >= 0.5 else [(name, "sink", key0)]
        bad += [] if diffuse.max() < 50 else [(name, "diffuse", float(diffuse.max()))]
    res, gates = encoder_activations(params, x)
    for i, (h, g) in enumerate(zip(res, gates)):
        ch = np.abs(h).mean((0, 1))
        ratio = ch.max() / np.median(ch)
        print(f"encoder layer {i}: largest / median |h| channel {ratio:6.1f} (channel {int(ch.argmax())});  "
              f"gate pre-activations {g.min():6.2f} .. {g.max():6.2f}, 99.9th percentile of |g| {np.quantile(np.abs(g), 0.999):5.2f}")
        bad += [] if 30 <= ratio <= 300 else [(i, "outlier ratio", float(ratio))]
        g999 = float(np.quantile(np.abs(g), 0.999))
        bad += [] if 5 <= g999 <= 15 else [(i, "gates", float(g.min()), float(g.max()), g999)]
    for k, v in params.items():
        if k.endswith("/scale"):
            assert v.min() >= 0.05 and v.max() <= 20
    sc = np.concatenate([v for k, v in params.items() if k.endswith("/scale")])
    print(f"norm scales: {sc.min():.3f} .. {sc.max():.2f}, log std {np.log(sc).std():.2f}")
    assert 0.8 <= np.log(sc).std() <= 1.2
    lg = O.decode_teacher_forced(params, CFG, O.encode(params, CFG, x, np.float64), toks, np.float64)
    eos = float((lg.argmax(-1) == O.EOS_ID).mean())
    print(f"EOS is the argmax at {eos:.1%} of {toks.size} teacher-forced positions")
    bad += [] if 0.005 <= eos <= 0.08 else [("EOS rate", eos)]
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# kernel-level value edges (-m gpu): the harness library and the per-element bars of test_kernel_parity.py
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    import ctypes as C
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(kp.TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, F, LL = C.c_void_p, C.c_int, C.c_float, C.c_longlong
    sig = {"kh_last_error": ([], C.c_char_p), "kh_sizeof": ([I], LL), "kh_tc_gemm": ([P, P, I, P, P, I, P, I], I),
           "kh_sgemm": ([P], I), "kh_enc_attention_tc": ([P, P, P, P, I, I, I, P, P, I, P], I),
           "kh_enc_attention_tc_scratch_floats": ([I, I, I], LL), "kh_enc_attention_fp32": ([P, I, I, I, P, P], I),
           "kh_dec_gemm_cluster": ([P], I), "kh_dec_gemm": ([P], I), "kh_dec_gemm_out_q": ([P, P], I),
           "kh_dec_gemm_cluster_tc": ([P], I), "kh_dec_gemm_out_q_tc": ([P, P], I),
           "kh_dec_attention": ([I, P, I, I, P, I, I, P, I, I, P, I, P, I, I, F, F, I, I], I)}
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    for i, st in enumerate((kp.TcGemmArgs, kp.GemmArgs, kp.DecGemmArgs)):
        assert lib.kh_sizeof(i) == C.sizeof(st), f"ctypes mirror of {st.__name__} does not match the C layout"
    return lib


KT = {0: 32, 1: 64, 2: 64}
DEC_ATT_KINDS = ("sharp", "sink0", "sinkL", "equal", "bigv", "ssq")


def dec_attention_values(kind, fmt, L, seed, B=2, H=2):
    """(rows [B, 2, H, L, 64], q [B, ldq], part or None) for one value edge of the decode attention (q_off = 4):
    sharp  scores along one direction, the first K tile's far below the rest: row maxima 90 .. 300, and more than 88.7
           between the first tile's maximum and the row's
    sink0 / sinkL   one key (0 or L - 1) scores 150 .. 250, the others |S| of order 1
    equal  every key row the same (scores all equal, above 88.7): the result is the mean of V
    bigv   diffuse scores, V rows scaled by up to 1e4
    ssq    the q_ssq scaling with the statistic dominated by one of 16 partials (1e6 against <= 1e-3), on sharp rows"""
    rng = np.random.default_rng(seed)
    ldq = H * 64 + 8
    k = rng.standard_normal((B, H, L, 64)) * 0.4
    v = rng.uniform(-0.5, 1.0, (B, H, L, 64))
    q = rng.uniform(-0.5, 1.0, (B, H, 64))
    part = None
    u = q / np.linalg.norm(q, axis=-1, keepdims=True)
    qn = np.linalg.norm(q, axis=-1)[..., None]                      # [B, H, 1]
    if kind in ("sharp", "ssq"):
        top = rng.uniform(90.0, 300.0, (B, H, 1))
        s = rng.uniform(-1.0, 1.0, (B, H, L)) * top
        s[..., :KT[fmt]] = rng.uniform(-1.0, 1.0, (B, H, min(L, KT[fmt])))
        s[..., -1] = top[..., 0]                                    # the maximum in the last tile
        k = k * 0.05 + (s / qn)[..., None] * u[:, :, None, :]
    elif kind in ("sink0", "sinkL"):
        j = 0 if kind == "sink0" else L - 1
        k[:, :, j] = u * (rng.uniform(150.0, 250.0, (B, H, 1)) / qn)
    elif kind == "equal":
        k[:] = u[:, :, None, :] * (rng.uniform(120.0, 200.0, (B, H, 1, 1)) / qn[..., None])
    elif kind == "bigv":
        v = v * 10.0 ** rng.uniform(0.0, 4.0, (B, H, L, 1))
    rows = np.stack([k, v], 1).astype(np.float32)
    qq = rng.uniform(-0.5, 1.0, (B, ldq))
    qq[:, 4:4 + H * 64] = q.reshape(B, H * 64)
    if kind == "ssq":
        part = np.concatenate([np.full((B, 1), 1e6), rng.uniform(0.0, 1e-3, (B, 16))], 1)
        rs = 1.0 / np.sqrt(part[:, :16].sum(1) / 512.0 + 1e-6)
        qq = qq / rs[:, None]                                      # the kernel's scaling brings q back
    return rows, qq.astype(np.float32), (None if part is None else part.astype(np.float32))


def _dec_att_cases():
    return [(fmt, L, kind) for fmt in (0, 1, 2) for L in sorted({1, KT[fmt], 257, 1023, 1024}) for kind in DEC_ATT_KINDS]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,L,kind", _dec_att_cases(), ids=lambda v: str(v))
def test_dec_attention_value_edges(kh, fmt, L, kind):
    """dec_attention_bulk_kernel<fmt> at the values the trained regime brings (dec_attention_values), every row format,
    L = 1, one K tile, 257, 1023, 1024, against float64 over the stored rows with the bars of test_dec_attention; rows past
    L stay NaN and unread, the output outside its rows stays NaN."""
    rows, q, part = dec_attention_values(kind, fmt, L, seed=1000 * fmt + L + DEC_ATT_KINDS.index(kind))
    S, _ = kp.dec_attention_check(kh, fmt, rows, q, part, 16 * (L % 2), L % 2 == 0, f"decode attention {kind} fmt={fmt} L={L}")
    mx = S.max(-1)
    if kind in ("sharp", "ssq", "sink0", "sinkL", "equal"):
        assert (mx > OVERFLOW).all(), f"{kind}: row maxima {mx.ravel()} do not reach past 88.7"
    if kind in ("sharp", "ssq") and L > KT[fmt]:
        assert (mx - S[..., :KT[fmt]].max(-1) > OVERFLOW).all()


def _outlier_A(rng, M, K, cols=(3, 100, 257)):
    A = kp._pos_mean(rng, (M, K), 2.0)
    for c in cols[:2 + (K > 300)]:
        A[:, c % K] *= 300.0
    return A


def _lognormal_W(rng, K, N):
    return (kp._pos_mean(rng, (K, N), 2.0 / K) * np.exp(rng.standard_normal(N))).astype(np.float32)


DEC_OUTLIER_CASES = [(64, 1152, 512, 0, False), (37, 512, 384, 1, True), (5, 1536, 512, 3, False), (64, 512, 1024, 1, True),
                     (63, 36, 1024, 0, False), (1, 1516, 384, 0, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["kh_dec_gemm_cluster", "kh_dec_gemm", "kh_dec_gemm_cluster_tc"])
@pytest.mark.parametrize("case", DEC_OUTLIER_CASES, ids=lambda c: f"M{c[0]}-N{c[1]}-K{c[2]}-epi{c[3]}")
def test_dec_gemm_outlier_columns(kh, kernel, case):
    """The decode GEMMs with the fused RMSNorm statistic (norm=1) on rows whose sum of squares 2-3 outlier columns at 300x
    dominate, and W with log-normal column scales: the FMA cluster kernel and the split-K fallback within TOL_DEC, the
    3xTF32 cluster kernel within 2^-17 (test_dec_gemm_tc.py)."""
    M, N, K, epi, inplace = case
    rng = np.random.default_rng(M + N + K)
    A, W = _outlier_A(rng, M, K), _lognormal_W(rng, K, N)
    got, ref, cond, _ = kp._dec_run(kh, kernel, M, N, K, epi, True, inplace, seed=M, AW=(A, W))
    kp._check(f"{kernel} outliers {case}", got, ref, cond, 2.0 ** -17 if kernel.endswith("_tc") else kp.TOL_DEC)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [False, True])
def test_dec_gemm_out_q_outliers(kh, tc):
    """The fused out+query launch with outlier columns in o and y and log-normal column scales in both weights."""
    import ctypes as C
    rng = np.random.default_rng(77 + tc)
    M, Q, D_ = 64, 384, 512
    o, y = _outlier_A(rng, M, Q), _outlier_A(rng, M, D_, cols=(5, 400, 511))
    W0, W1 = _lognormal_W(rng, Q, D_), _lognormal_W(rng, Q + D_, Q)
    ref0, cond0 = kp._gemm_ref(o, W0, None, kp.EPI_RESIDUAL, y.astype(np.float64))
    ref1, cond1 = kp._gemm_ref(np.concatenate([o, y], 1), W1, None, kp.EPI_STORE)
    do, dy, dW0, dW1 = kp._dev(o), kp._dev(y), kp._dev(W0), kp._dev(W1)
    C0, C1 = kp._nan(M + 2, D_ + 4), kp._nan(M + 2, Q + 4)
    ssq = kp._nan(M + 1, D_ // 32 + 1)
    P = kp._p
    a0 = kp.DecGemmArgs(A=P(do), lda=Q, W=P(dW0), ldw=D_, M=M, N=D_, K=Q, epi=kp.EPI_RESIDUAL, R=P(dy), ldr=D_, C=P(C0),
                        ldc=D_ + 4, n_split=D_, ssq_out=P(ssq), ssq_ld=D_ // 32 + 1)
    a1 = kp.DecGemmArgs(A=P(do), lda=Q, W=P(dW1), ldw=Q, M=M, N=Q, K=Q + D_, epi=kp.EPI_STORE, C=P(C1), ldc=Q + 4, n_split=Q,
                        A2=P(dy), lda2=D_, K0=Q)
    kp._call(kh, "kh_dec_gemm_out_q_tc" if tc else "kh_dec_gemm_out_q", C.byref(a0), C.byref(a1))
    tol = 2.0 ** -17 if tc else kp.TOL_DEC
    g0, g1 = C0[:M, :D_].double().cpu().numpy(), C1[:M, :Q].double().cpu().numpy()
    kp._check(f"out tc={tc}", g0, ref0, cond0, tol)
    kp._check(f"q tc={tc}", g1, ref1, cond1, tol)
    want = (g0.reshape(M, D_ // 32, 32) ** 2).sum(-1)
    kp._check(f"ssq_out tc={tc}", ssq[:M, :D_ // 32].double().cpu().numpy(), want, want, kp.TOL_DEC)


def _gate_operands(rng, M, N, K):
    """A, W with gate columns (even) whose pre-activations spread over about [-12, 12], linear columns (odd) of order 1"""
    A = kp._pos_mean(rng, (M, K))
    W = kp._pos_mean(rng, (K, N), 2.0 / K)
    rms = np.sqrt((A.astype(np.float64) ** 2).mean())
    W[:, 0::2] = rng.standard_normal((K, N // 2)) * (4.0 / (rms * np.sqrt(K)))
    return A, W.astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tf32x3", "tf32", "simt", "kh_dec_gemm_cluster", "kh_dec_gemm", "kh_dec_gemm_cluster_tc"])
def test_gated_gelu_gate_tails(kh, path):
    """The gated-GELU epilogue (wgmma in both precisions, the SIMT GEMM, the decode GEMMs) with gate pre-activations spread
    over about [-12, 12]: gelu's negative tail (tanh -> -1, the product 0.5 x (1 + tanh) cancels) and its linear tail."""
    M, N, K = (200, 2048, 512) if path in ("tf32x3", "tf32", "simt") else (64, 2048, 512)
    rng = np.random.default_rng(len(path))
    A, W = _gate_operands(rng, M, N, K)
    g = A.astype(np.float64) @ W[:, 0::2].astype(np.float64)
    assert g.min() < -10 and g.max() > 10
    if path in ("tf32x3", "tf32", "simt"):
        got, _, _, ref, cond = kp._run_gemm(kh, path, M, N, K, kp.EPI_GATED_GELU, False, None, path == "tf32x3", seed=1, AW=(A, W))
        tol = kp.GEMM_TOL[path]
    else:
        got, ref, cond, _ = kp._dec_run(kh, path, M, N, K, kp.EPI_GATED_GELU, False, False, seed=1, AW=(A, W))
        tol = 2.0 ** -17 if path.endswith("_tc") else kp.TOL_DEC
    kp._check(f"gated gelu {path} gates {g.min():.1f} .. {g.max():.1f}", got, ref, cond, tol)


def enc_attention_values(kind, B, T, H, seed):
    """qkv [B*T, 3*H*64] for the encoder attention: 'sink' -- every query along one direction (|q| 8 .. 11) and key 0 along
    it at 15x, scores on key 0 of 120 .. 165 (above 88.7), the other keys |S| of order 1; 'uniform' -- every key row the
    same, so every score row is constant (the result is the mean of V)."""
    rng = np.random.default_rng(seed)
    qkv = np.empty((B, T, 3, H, 64))
    qkv[:, :, :2] = rng.standard_normal((B, T, 2, H, 64)) * 0.1
    u = rng.standard_normal(64)
    u /= np.linalg.norm(u)
    if kind == "sink":
        qkv[:, :, 0] += rng.uniform(8.0, 11.0, (B, T, H, 1)) * u
        qkv[:, 0, 1] = 15.0 * u
    else:
        qkv[:, :, 0] += rng.uniform(-3.0, 3.0, (B, T, H, 1)) * u
        qkv[:, :, 1] = qkv[:, :1, 1]
    qkv[:, :, 2] = rng.uniform(-0.5, 1.0, (B, T, H, 64))
    return qkv.reshape(B * T, 3 * H * 64).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sink", "uniform"])
@pytest.mark.parametrize("path", ["tc3", "tc1", "fp32"])
@pytest.mark.parametrize("T", [200, 256, 512])
def test_enc_attention_sink_and_uniform(kh, path, kind, T):
    """The encoder attention (wgmma 3xTF32 and TF32, exact fp32) with a sink key and with constant score rows, at one
    partial query tile (T = 200), one full pass (256) and the key-split form (512), with the bars of test_kernel_parity.py."""
    B, H = 2, 2
    qkv = enc_attention_values(kind, B, T, H, seed=T + len(kind))
    if path == "fp32":
        kp.enc_attention_fp32_check(kh, qkv, B, T, H, f"fp32 attention {kind} T={T}")
    else:
        kp.enc_attention_tc_check(kh, qkv, B, T, H, path == "tc3", True, f"tc attention {kind} T={T} {path}")



# ------------------------------------------------------------------------------------------------
# the full model against float64 (-m gpu)
# ------------------------------------------------------------------------------------------------
LOGIT_TOL = 5e-4
LONG_PROBE = [0, 1, 31, 32, 63, 64, 65, 191, 192, 257, 383, 511, 512, 767, 1022, 1023]
PICK = [0, 17, 63]
STEPS = 1024
GREEDY_STEPS = 512                   # steps the float64 greedy reference runs (the comparison horizon's upper end)
# a probe is well-conditioned where the float32 oracle's own logit error is small enough that 4x it is inside LOGIT_TOL
COND = LOGIT_TOL / 4
# (gemm mode, K/V rows, tensor-core encoder attention)
MODEL_CONFIGS = [("simt", "f32", True), ("tf32x3", "f32", True), ("tf32x3", "p24", True), ("tf32x3", "f16", True),
                 ("tf32x3", "p24", False)]


def _cfg_id(c):
    return f"{c[0]}-kv{c[1]}" + ("" if c[2] else "-fp32attn")


def _rel(a, ref):
    return float(np.abs(a - ref).max() / np.abs(ref).max())


def run_oracle():
    """float64 / float32 oracle runs on the generated weights: the encoder at B = 2 (the inputs of test_gpu_parity's
    long-cache test) and on sequences PICK of a B = 64 batch; teacher-forced logits at LONG_PROBE over 1024 random tokens
    on the float64 encoder output, in float64 and float32, and the float32 oracle's error per probe; the float64 greedy
    decode of the PICK sequences over GREEDY_STEPS steps with its logits."""
    params = trained_params()
    x2 = spectrogram((1274, 1275))
    x64 = spectrogram(range(5000, 5064))
    r = dict(params=params, x2=x2, x64=x64)
    r["enc64"], r["enc32"] = (O.encode(params, CFG, x2, dt) for dt in (np.float64, np.float32))
    r["pick64"], r["pick32"] = (O.encode(params, CFG, x64[PICK], dt) for dt in (np.float64, np.float32))
    toks = np.random.default_rng(12).integers(3, 1500, size=(2, STEPS))
    toks[:, 0] = 0
    r["toks"] = toks
    l64 = O.decode_teacher_forced(params, CFG, r["enc64"], toks, np.float64)[:, LONG_PROBE]
    l32 = O.decode_teacher_forced(params, CFG, r["enc64"].astype(np.float32), toks, np.float32)[:, LONG_PROBE]
    r["l64"], r["scale"] = l64, float(np.abs(l64).max())
    r["e32"] = np.abs(l32 - l64).max(axis=(0, 2)) / r["scale"]
    r["g64"], r["gl64"] = O.greedy_decode(params, CFG, r["pick64"], GREEDY_STEPS, np.float64, stop_at_eos=False,
                                          return_logits=True)
    return r


@pytest.fixture(scope="module")
def oracle_runs():
    r = run_oracle()
    print("\nfloat32 oracle vs float64: encoder B=2 %.2e, B=64 picks %.2e; logits per probe: %s" % (
        _rel(r["enc32"], r["enc64"]), _rel(r["pick32"], r["pick64"]),
        " ".join(f"{p}:{e:.1e}" for p, e in zip(LONG_PROBE, r["e32"]))))
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODEL_CONFIGS, ids=_cfg_id)
def test_model_trained_statistics_vs_float64(oracle_runs, mode, monkeypatch):
    """The mt3 model (8 + 8 layers, T = 256, L = 1024) on the generated weights -- SIMT with fp32 rows, TF32X3 with fp32,
    24-bit and fp16 rows, and TF32X3 with 24-bit rows and the exact-fp32 encoder attention (MT3_TC_ATTENTION=0, without
    the tf32-rounded P) -- against the float64 oracle.
      encoder   B = 2 and sequences 0, 17, 63 of B = 64: within max(5e-4, 4 e_f32) of max |enc|, SIMT within
                4 e_f32 + 1e-5 (e_f32: the float32 oracle's own deviation on the same input).
      logits    the decoder teacher-forced over 1024 positions on the float64 encoder output (the input the float32
                oracle gets), at LONG_PROBE.  These weights make late positions chaotic: there the float32 oracle is
                itself far from float64, and no float32 implementation can be held to a bar.  So the bars are asserted
                at the probes where the float32 oracle's error e_f32(p) is at most 5e-4 / 4: fp32 rows within
                max(4 e_f32(p), 2e-5), hence within 5e-4.  24-bit and fp16 rows leave that bar at these statistics
                (24-bit rows by about 20 e_f32, 1.9e-3; DESIGN.md section 4) and are reported only.
      tokens    1024 graph-replayed greedy steps at B = 64 (bench's path): sequences 0, 17, 63 equal the float64
                oracle's greedy tokens up to the first of: their first EOS, the first step whose float64 top-2 margin is
                not above twice the worst logit error at the well-conditioned probes, the first ill-conditioned probe."""
    import torch
    from mt3_b200 import _lib, network
    gm, kv, tc_attn = mode
    name = _cfg_id(mode)
    if not tc_attn:
        monkeypatch.setenv("MT3_TC_ATTENTION", "0")
    r = oracle_runs
    ncfg = network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=8, num_decoder_layers=8, head_dim=64,
                            mlp_dim=1024, mlp_activations=('gelu', 'linear'))
    gmode = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3}[gm]
    kvf = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[kv]
    m = network.Transformer(ncfg, r["params"], device="cuda:0", max_batch=64, max_input_length=256, max_decode_length=STEPS,
                            gemm_mode=gmode, kv_format=kvf)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")      # noqa: E731
    # encoder
    x64 = dev(r["x64"])
    e_enc = (_rel(m.encode(dev(r["x2"])).cpu().numpy(), r["enc64"]), _rel(m.encode(x64).cpu().numpy()[PICK], r["pick64"]))
    f_enc = (_rel(r["enc32"], r["enc64"]), _rel(r["pick32"], r["pick64"]))
    # teacher-forced logits at the probes, on the float64 encoder output
    enc = dev(r["enc64"].astype(np.float32))
    m.init_cache(enc)
    t = dev(r["toks"].astype(np.int32))
    got = np.empty(r["l64"].shape, np.float32)
    j = 0
    for i in range(STEPS):
        lg = m.decode(enc, None, t[:, i:i + 1])
        if i == LONG_PROBE[j]:
            got[:, j] = lg[:, 0].cpu().numpy()
            j = min(j + 1, len(LONG_PROBE) - 1)
    errs = np.abs(got - r["l64"]).max(axis=(0, 2)) / r["scale"]
    e32 = r["e32"]
    cond = e32 <= COND
    assert cond.sum() >= 5, f"only {int(cond.sum())} well-conditioned probes: the generator has drifted"
    e_log = float(errs[cond].max())
    horizon = min([p for p, c in zip(LONG_PROBE, cond) if not c] + [GREEDY_STEPS])
    # greedy tokens, bench's path
    toks = m.generate(x64, num_steps=STEPS, stop_at_eos=False, use_graph=True).cpu().numpy()[PICK, :GREEDY_STEPS]
    del m
    torch.cuda.empty_cache()
    g64, gl64 = r["g64"], r["gl64"]
    srt = np.sort(gl64, axis=-1)
    safe = np.cumprod((srt[..., -1] - srt[..., -2]) > 2 * e_log * np.abs(gl64).max(), axis=1).astype(bool)
    eos = g64 == O.EOS_ID
    alive = np.cumsum(eos, axis=1) - eos == 0
    cmp = safe & alive & (np.arange(GREEDY_STEPS) < horizon)
    ends = [int(np.argmax(e)) if e.any() else -1 for e in eos]
    print(f"[{name}] encoder vs fp64: B=2 {e_enc[0]:.2e}, B=64 {e_enc[1]:.2e} (fp32 oracle {f_enc[0]:.2e}, {f_enc[1]:.2e});  "
          f"logits at the {int(cond.sum())} well-conditioned probes worst {e_log:.2e} (fp32 oracle {e32[cond].max():.2e});  "
          f"greedy tokens compared {int(cmp.sum())} (horizon {horizon}, fp64 first EOS {ends}), differing "
          f"{int((toks[cmp] != g64[cmp]).sum())}")
    print(f"[{name}] logits vs fp64 per probe (gpu / fp32 oracle): " +
          " ".join(f"{p}:{e:.1e}/{f:.1e}" for p, e, f in zip(LONG_PROBE, errs, e32)))
    np.testing.assert_array_equal(toks[cmp], g64[cmp], err_msg=f"{name}: greedy tokens")
    for e, f in zip(e_enc, f_enc):
        assert e <= max(LOGIT_TOL, 4 * f), (name, "encoder", e, f)
        if gm == "simt":
            assert e <= 4 * f + 1e-5, (name, "SIMT encoder", e, f)
    if kv == "f32":
        bar = np.maximum(4 * e32, 2e-5)
        assert (errs[cond] <= bar[cond]).all(), (name, errs, e32)
