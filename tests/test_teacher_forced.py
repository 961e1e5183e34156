"""The teacher-forced decoder pass: Transformer.decode(decode=False) / __call__, Transformer.score, score_batch and
InferenceModel.score, and the kernels under them (causal self-attention and cross-attention on wgmma and in exact fp32,
the token-score kernel).

CPU: the float64 oracle of the pass with the reference's masks (make_decoder_mask / make_attention_mask), its score
restatement, the host-side target building of InferenceModel.score, and the argument checks of the C ABI.
GPU: every kernel alone against float64 with test_kernel_parity.py's per-element bars, the model against the float64
oracle at the positions whose target is not padding with DESIGN.md section 4's bar, scores, isolation from the decode
state, errors, and InferenceModel.score end to end."""
import ctypes as C
import functools
import importlib.util
import os

import numpy as np
import pytest
import scipy.special

from mt3_b200 import layers as L_
from oracle import mt3_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
LOGIT_TOL = 5e-4


# ------------------------------------------------------------------------------------------------
# float64 oracle of the pass (host)
# ------------------------------------------------------------------------------------------------
def decode_full(params, cfg, encoded, decoder_input_tokens, decoder_target_tokens, dtype=np.float64):
    """network.py:196-262 with decode=False and the reference's masks: self-attention make_decoder_mask(targets),
    encoder-decoder make_attention_mask(targets > 0, ones(T)) (network.py:320-335).  [B,L] ints -> logits [B,L,V]."""
    p = O._cast(params, dtype)
    enc = np.asarray(encoded, dtype)
    tgt = np.asarray(decoder_target_tokens)
    b, length = decoder_input_tokens.shape
    pe = O.sinusoidal_table(2048, cfg.emb_dim).astype(dtype)
    y = p["decoder/token_embedder/embedding"][decoder_input_tokens] + pe[None, :length]
    self_mask = L_.make_decoder_mask(tgt, dtype=dtype)
    cross_mask = L_.make_attention_mask(tgt > 0, np.ones(enc.shape[:2]), dtype=dtype)
    for i in range(cfg.num_decoder_layers):
        pre = f"decoder/layers_{i}/"
        a = O.rms_norm(y, p[pre + "pre_self_attention_layer_norm/scale"])
        y = y + O.mha(p, pre + "self_attention/", a, a, cfg.num_heads, cfg.head_dim, mask=self_mask)
        c = O.rms_norm(y, p[pre + "pre_cross_attention_layer_norm/scale"])
        y = y + O.mha(p, pre + "encoder_decoder_attention/", c, enc, cfg.num_heads, cfg.head_dim, mask=cross_mask)
        m = O.rms_norm(y, p[pre + "pre_mlp_layer_norm/scale"])
        y = y + O.mlp_block(m, [p[pre + "mlp/wi_0/kernel"], p[pre + "mlp/wi_1/kernel"]], p[pre + "mlp/wo/kernel"],
                            cfg.mlp_activations)
    y = O.rms_norm(y, p["decoder/decoder_norm/scale"])
    return O.dense(y, p["decoder/logits_dense/kernel"])


def token_scores_ref(logits, targets, weights=None):
    """T5X score_batch's per-token term with z_loss = 0: (logits[target] - logsumexp(logits)) * weight, weight = target > 0
    unless given."""
    x = np.asarray(logits, np.float64)
    m = x.max(-1, keepdims=True)
    lse = (m + np.log(np.exp(x - m).sum(-1, keepdims=True)))[..., 0]
    picked = np.take_along_axis(x, np.asarray(targets)[..., None], -1)[..., 0]
    w = (np.asarray(targets) > 0) if weights is None else np.asarray(weights)
    return (picked - lse) * w


def _tokens(rng, B, L, V, pad_tail=True, inner_zero=True, all_pad_row=True):
    """targets in [3, V): row 0 has a 0 inside the sequence, row 1 a padding tail, row 2 (if any) is all padding;
    decoder inputs are the targets shifted right behind a 0 (models.py:77-98)."""
    tgt = rng.integers(3, V, size=(B, L)).astype(np.int32)
    if inner_zero and L > 4:
        tgt[0, L // 3] = 0
    if pad_tail and B > 1 and L > 1:
        tgt[1, (2 * L) // 3:] = 0
    if all_pad_row and B > 2:
        tgt[2] = 0
    din = np.concatenate([np.zeros((B, 1), np.int32), tgt[:, :-1]], axis=1)
    return din, tgt


def test_decode_full_equals_decode_teacher_forced_without_padding():
    """With no target equal to 0 the masks are the causal mask and all ones: the same logits, bit for bit."""
    cfg = O.T5Config(vocab_size=64, emb_dim=64, num_heads=2, num_decoder_layers=2, num_encoder_layers=1, mlp_dim=128)
    params = O.init_params(cfg, seed=3, norm_scale_jitter=0.05)
    rng = np.random.default_rng(0)
    enc = rng.standard_normal((2, 24, 64))
    din, tgt = _tokens(rng, 2, 17, 64, pad_tail=False, inner_zero=False, all_pad_row=False)
    for dt in (np.float64, np.float32):
        a = decode_full(params, cfg, enc, din, tgt, dt)
        b = O.decode_teacher_forced(params, cfg, enc, din, dt)
        assert a.dtype == b.dtype and np.array_equal(a, b)


def test_score_restatement_equals_scipy_log_softmax():
    rng = np.random.default_rng(1)
    x = rng.standard_normal((3, 11, 40)) * 7
    tgt = rng.integers(0, 40, size=(3, 11))
    w = rng.integers(0, 3, size=(3, 11))
    ref = np.take_along_axis(scipy.special.log_softmax(x, -1), tgt[..., None], -1)[..., 0]
    np.testing.assert_allclose(token_scores_ref(x, tgt, w), ref * w, rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(token_scores_ref(x, tgt), ref * (tgt > 0), rtol=1e-13, atol=1e-13)


def _dense_note_sequence():
    """Notes over 5 s; the first 2.048 s (one mt3 segment) so dense that its tokens run past 1024."""
    from mt3_b200 import note_decoding as nd
    rng = np.random.default_rng(5)
    ns = nd.NoteSequence()
    for k in range(700):
        t0 = float(rng.integers(0, 200)) / 100.0
        ns.add(t0, t0 + 0.01 * float(rng.integers(1, 5)), int(rng.integers(21, 109)), 100, program=int(rng.integers(0, 3)) * 8)
    for k in range(12):
        ns.add(2.3 + 0.2 * k, 2.35 + 0.2 * k, 60 + k, 100)
    return ns


@pytest.mark.parametrize("model_type", ["mt3", "ismir2021"])
def test_segment_score_targets(model_type):
    """Per-segment ids +3, EOS, the feature converter's trim / pad to 1024, shifted inputs and weights; a short last
    segment, and a first segment of more than 1024 tokens (trimmed, so it loses its EOS)."""
    from mt3_b200 import inference, models, note_encoding as ne, vocabularies
    spec, T, ties = {"mt3": ("NoteEncodingWithTiesSpec", 256, True), "ismir2021": ("NoteEncodingSpec", 512, False)}[model_type]
    codec = vocabularies.build_codec(vocabularies.VocabularyConfig(num_velocity_bins=1 if model_type == "mt3" else 127))
    vocab = vocabularies.vocabulary_from_codec(codec)
    ns = _dense_note_sequence()
    n_frames = 5 * 16000 // 128 + 1
    frame_times = np.arange(n_frames) / 125.0
    got = inference.segment_score_targets(ns, codec, vocab, frame_times, T, spec, 1024)
    raw = ne.note_sequence_to_segment_targets(ns, codec, frame_times, T, include_ties=ties)
    S = -(-n_frames // T)
    assert len(raw) == S and got["decoder_target_tokens"].shape == (S, 1024) and n_frames % T != 0
    assert max(len(r) for r in raw) > 1024, "the dense segment should need trimming"
    assert any(0 < len(r) < 1000 for r in raw)
    conv = models.ContinuousInputsEncDecFeatureConverter()
    for i, r in enumerate(raw):
        t = got["decoder_target_tokens"][i]
        n = min(len(r) + 1, 1024)
        np.testing.assert_array_equal(t[:min(len(r), 1024)], np.asarray(r[:1024]) + 3)
        if len(r) < 1024:
            assert t[len(r)] == 1 and (t[len(r) + 1:] == 0).all()
        np.testing.assert_array_equal(got["decoder_input_tokens"][i], np.concatenate([[0], t[:-1]]))
        np.testing.assert_array_equal(got["decoder_loss_weights"][i], (t != 0).astype(np.int32))
        assert got["decoder_loss_weights"][i].sum() == n
        feats = conv.convert_example({'inputs': np.zeros((T, 512), np.float32),
                                      'targets': np.asarray(list(vocab.encode(r)) + [1], np.int32)},
                                     {'inputs': T, 'targets': 1024})
        for k in ("decoder_input_tokens", "decoder_target_tokens", "decoder_loss_weights"):
            np.testing.assert_array_equal(got[k][i], feats[k])


def test_abi_null_handle():
    from mt3_b200 import _lib
    lib = _lib.load()
    assert lib.mt3_teacher_forced_workspace_bytes(None, 1, 1, 1) == -1
    assert lib.mt3_decode_teacher_forced(None, None, 1, 1, None, None, None, 1, None, None, None, 0, None) == -1


# ------------------------------------------------------------------------------------------------
# kernels alone (-m gpu)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    import test_kernel_parity as kp
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(kp.TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, LL = C.c_void_p, C.c_int, C.c_longlong
    sig = {
        "kh_last_error": ([], C.c_char_p),
        "kh_attention_tc": ([P, P, I, I, I, P, P, I, I, I, P, P, I, I, P, P, I, I, P, I, P], I),
        "kh_attention_tc_scratch_floats": ([I, I, I, I, I], LL),
        "kh_attention_fp32": ([P, I, I, P, I, I, I, I, I, I, I, P, P, P, I], I),
        "kh_token_score": ([P, I, I, I, I, I, P, P, P, P], I),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    return lib


def _attn_ref_masked(q, k, v, mask):
    """float64 softmax over the visible keys (mask [B, Tq, Tk] bool), 0 for a row with none; the condition terms of
    test_kernel_parity._attn_ref.  q [B, H, Tq, 64], k / v [B, H, Tk, 64]."""
    S = q @ k.transpose(0, 1, 3, 2)
    m = mask[:, None]
    Sm = np.where(m, S, -np.inf)
    mx = Sm.max(-1, keepdims=True)
    mx = np.where(np.isfinite(mx), mx, 0.0)
    p = np.where(m, np.exp(Sm - mx), 0.0)
    den = p.sum(-1, keepdims=True)
    p = np.divide(p, den, out=np.zeros_like(p), where=den > 0)
    o = p @ v
    cond_p = p @ np.abs(v)
    pA = p * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2))
    cond_s = pA @ np.abs(v) + np.abs(o) * pA.sum(-1, keepdims=True)
    return o, cond_p, cond_s


def _rows(a):      # [B, H, T, 64] -> [B, T, H*64]
    return a.transpose(0, 2, 1, 3).reshape(a.shape[0], a.shape[2], -1)


def _key_valid(rng, B, L):
    kv = (rng.random((B, L)) > 0.15).astype(np.int32)
    kv[0, :min(L, 5)] = 0                      # rows 0..4 of sequence 0 see no key at all
    return kv


ATT_PATHS = ["tc3", "tc1", "fp32"]
LS = [1, 8, 127, 128, 129, 256, 257, 511, 512, 1000, 1024]


def _run_attention(kh, path, q_rows, kv_rows, vt, B, H, Tq, Tk, ldq, q_col0, ldk, k_col0, v_col0, causal, key_valid, n_valid):
    """launch one attention form; returns the output [B*Tq, H*64] (hi + lo) as float64 and the NaN-poisoned buffers."""
    import torch
    import test_kernel_parity as kp
    Q = H * 64
    kvd = None if key_valid is None else kp._dev(key_valid.astype(np.int32))
    oh = kp._nan(B * Tq + 3, Q)
    ol = kp._nan(B * Tq + 3, Q) if path != "tc1" else None
    if path == "fp32":
        qd, kd = kp._dev(q_rows), kp._dev(kv_rows)
        kp._call(kh, "kh_attention_fp32", kp._p(qd), ldq, q_col0, kp._p(kd), ldk, k_col0, v_col0, Tq, Tk, H, B, kp._p(oh), kp._p(ol),
                 kp._p(kvd), n_valid)
    else:
        s3 = path == "tc3"
        if s3:
            (qh, ql), (kh_, kl), (vh, vl) = kp._split(q_rows), kp._split(kv_rows), kp._split(vt)
            d = [kp._dev(x) for x in (qh, ql, kh_, kl, vh, vl)]
        else:
            d = [kp._dev(q_rows), None, kp._dev(kv_rows), None, kp._dev(vt), None]
        n_scr = kh.kh_attention_tc_scratch_floats(B, Tq, Tk, H, int(causal))
        scratch = kp._nan(n_scr) if n_scr else None
        kp._call(kh, "kh_attention_tc", kp._p(d[0]), kp._p(d[1]), ldq, q_col0, Tq, kp._p(d[2]), kp._p(d[3]), ldk, k_col0, Tk, kp._p(d[4]),
                 kp._p(d[5]), B, H, kp._p(oh), kp._p(ol), int(s3), int(causal), kp._p(kvd), n_valid, kp._p(scratch))
    got = oh[:B * Tq].double().cpu().numpy() + (ol[:B * Tq].double().cpu().numpy() if ol is not None else 0)
    w = np.zeros(oh.shape, bool)
    w[:B * Tq] = True
    kp._assert_poison("out_hi", oh, w)
    torch.cuda.synchronize()
    return got


def _bars(path):
    import test_kernel_parity as kp
    if path == "fp32":
        return kp.TOL_ENC_ATT_P, kp.TOL_ENC_ATT_S
    return kp.TOL_ATT_P, kp.TOL_ATT_S[path == "tc3"]


def _causal_check(kh, path, qkv, B, L, H, key_valid, name):
    """qkv [B*Lp, 3Q] (rows past L are padding); compares rows < L against the masked float64 softmax."""
    import test_kernel_parity as kp
    Q = H * 64
    Lp = -(-L // 128) * 128
    x = qkv.astype(np.float64).reshape(B, Lp, 3, H, 64).transpose(2, 0, 3, 1, 4)
    i = np.arange(Lp)
    ok = np.zeros((B, Lp), bool)
    ok[:, :L] = key_valid > 0
    mask = (i[None, :, None] >= i[None, None, :]) & ok[:, None, :]
    o, cp, cs = (_rows(a)[:, :L] for a in _attn_ref_masked(x[0], x[1], x[2], mask))
    vt = kp._vt_host(qkv, B, Lp, H) if path != "fp32" else None
    got = _run_attention(kh, path, qkv, qkv, vt, B, H, Lp, Lp, 3 * Q, 0, 3 * Q, Q, 2 * Q, True, key_valid, L)
    got = got.reshape(B, Lp, Q)[:, :L]
    tp, ts = _bars(path)
    kp._check(name, got, o, cp, tp, cs, ts)
    assert np.isfinite(got).all()
    none = ~(mask[:, :L].any(-1))
    assert (got[none] == 0).all(), "a row with no visible key must write 0"


@pytest.mark.gpu
@pytest.mark.parametrize("path", ATT_PATHS)
@pytest.mark.parametrize("L", LS)
def test_causal_self_attention(kh, path, L):
    """Causal self-attention with per-key masking (zeros inside the sequence, rows with no visible key), one and two key
    chunks, the key-split form over parts of 256 keys with the parts above the diagonal skipped, padded L."""
    import test_kernel_parity as kp
    B, H = 2, 2
    Lp = -(-L // 128) * 128
    rng = np.random.default_rng(L)
    qkv = kp._attn_inputs(rng, B, Lp, H, sharp=L % 2 == 1)
    _causal_check(kh, path, qkv, B, L, H, _key_valid(rng, B, L), f"causal attention {path} L={L}")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ATT_PATHS)
@pytest.mark.parametrize("L", [129, 512, 1000])
def test_causal_self_attention_sink(kh, path, L):
    """test_trained_statistics' sink values (scores on key 0 of 120 .. 165, above exp's overflow) under the causal mask;
    key 0 is visible to every query here, except in the rows of sequence 0 that see no key."""
    import test_trained_statistics as tsx
    B, H = 2, 2
    Lp = -(-L // 128) * 128
    qkv = tsx.enc_attention_values("sink", B, Lp, H, seed=L)
    rng = np.random.default_rng(L + 1)
    kv = _key_valid(rng, B, L)
    kv[1, 0] = 1
    _causal_check(kh, path, qkv, B, L, H, kv, f"causal attention sink {path} L={L}")


@pytest.mark.gpu
@pytest.mark.parametrize("path", ATT_PATHS)
@pytest.mark.parametrize("Tk", [256, 512])
@pytest.mark.parametrize("L", LS)
def test_cross_attention(kh, path, Tk, L):
    """Cross-attention: queries [B*Lp, Q] of their own, keys / values from a [B*Tk, 2Q] projection (V^T for the wgmma
    form); single pass at Tk = 256, key split at Tk = 512.  Sharp values (row maxima above 88.7) at odd L."""
    import test_kernel_parity as kp
    B, H = 2, 2
    Q = H * 64
    Lp = -(-L // 128) * 128
    rng = np.random.default_rng(L * 3 + Tk)
    a = kp._attn_inputs(rng, B, max(Lp, Tk), H, sharp=L % 2 == 1).reshape(B, max(Lp, Tk), 3, H, 64)
    q = np.ascontiguousarray(a[:, :Lp, 0].reshape(B * Lp, Q))
    kv = np.ascontiguousarray(a[:, :Tk, 1:].reshape(B * Tk, 2 * Q))
    xq = a[:, :Lp, 0].astype(np.float64).transpose(0, 2, 1, 3)
    xk, xv = (a[:, :Tk, j].astype(np.float64).transpose(0, 2, 1, 3) for j in (1, 2))
    o, cp, cs = (_rows(t)[:, :L] for t in _attn_ref_masked(xq, xk, xv, np.ones((B, Lp, Tk), bool)))
    vt = None
    if path != "fp32":
        qkv_like = np.concatenate([np.zeros((B, Tk, 1, H, 64), np.float32), a[:, :Tk, 1:]], axis=2).reshape(B * Tk, 3 * Q)
        vt = kp._vt_host(qkv_like, B, Tk, H)
    got = _run_attention(kh, path, q, kv, vt, B, H, Lp, Tk, Q, 0, 2 * Q, 0, Q, False, None, 0).reshape(B, Lp, Q)[:, :L]
    tp, ts = _bars(path)
    kp._check(f"cross attention {path} L={L} Tk={Tk}", got, o, cp, tp, cs, ts)


@pytest.mark.gpu
@pytest.mark.parametrize("weights", [False, True])
def test_token_score_kernel(kh, weights):
    """token_score_kernel on a chunk of padded rows: float64 log-softmax at the target times the weight, padding rows
    skipped, the logits copy exact, rows past L untouched."""
    import torch
    import test_kernel_parity as kp
    B, L, Lp, V = 3, 200, 256, 1536
    rng = np.random.default_rng(7)
    x = (rng.standard_normal((B * Lp, V)) * 6).astype(np.float32)
    x[5, 17] = 90.0                                          # a row whose exp would overflow without the max
    tgt = rng.integers(0, V, size=(B, L)).astype(np.int32)
    tgt[1, 50:] = 0
    w = rng.integers(0, 3, size=(B, L)).astype(np.int32) if weights else None
    row0, n = 128, B * Lp - 128 - 40                          # a chunk that starts and ends inside sequences
    xd = kp._dev(x[row0:row0 + n])
    td, wd = kp._dev(tgt), (None if w is None else kp._dev(w))      # held: the launch reads them
    scores = kp._nan(B * L)
    out = kp._nan(B * L * V)
    kp._call(kh, "kh_token_score", kp._p(xd), V, row0, n, Lp, L, kp._p(td), kp._p(wd), kp._p(scores), kp._p(out))
    rows = np.arange(row0, row0 + n)
    b, i = rows // Lp, rows % Lp
    keep = i < L
    pos = b[keep] * L + i[keep]
    ref = token_scores_ref(x[rows[keep]], tgt.reshape(-1)[pos], None if w is None else w.reshape(-1)[pos])
    s = scores.cpu().numpy()
    written = np.zeros(B * L, bool)
    written[pos] = True
    assert np.isnan(s[~written]).all()
    np.testing.assert_allclose(s[pos], ref, rtol=0, atol=2e-6 * (1 + np.abs(x).max()))
    o = out.cpu().numpy().reshape(B * L, V)
    np.testing.assert_array_equal(o[pos], x[rows[keep]])
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# the model (-m gpu)
# ------------------------------------------------------------------------------------------------
CONFIGS = {"mt3": (256, 1536), "ismir2021": (512, 1664)}


def _net_cfg(V, enc_layers=1):
    from mt3_b200 import network
    return network.T5Config(vocab_size=V, emb_dim=512, num_heads=6, num_encoder_layers=enc_layers, num_decoder_layers=8, head_dim=64,
                            mlp_dim=1024, mlp_activations=('gelu', 'linear'))


@functools.lru_cache(maxsize=None)
def _params(V):
    return O.init_params(O.T5Config(vocab_size=V, num_encoder_layers=1), seed=0, norm_scale_jitter=0.05)


@functools.lru_cache(maxsize=None)
def _case(config, L):
    """B = 3 inputs for a config and length, float64 and float32 oracle logits; B = 1 runs use sequence 0."""
    T, V = CONFIGS[config]
    rng = np.random.default_rng(L + T)
    enc = rng.standard_normal((3, T, 512)).astype(np.float32)
    din, tgt = _tokens(rng, 3, L, V)
    params = _params(V)
    l64 = decode_full(params, O.T5Config(vocab_size=V), enc, din, tgt, np.float64)
    l32 = decode_full(params, O.T5Config(vocab_size=V), enc, din, tgt, np.float32)
    return enc, din, tgt, l64, l32


_MODELS = {}


def _model(config, mode, kv=None):
    import torch
    from mt3_b200 import _lib, network
    key = (config, mode, kv)
    if key not in _MODELS:
        for k in list(_MODELS):
            del _MODELS[k]
        torch.cuda.empty_cache()
        T, V = CONFIGS[config]
        gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3, "tf32": _lib.GEMM_TF32}[mode]
        _MODELS[key] = network.Transformer(_net_cfg(V), _params(V), device=DEV, max_batch=64, max_input_length=T, max_decode_length=1024,
                                           gemm_mode=gm, kv_format=_lib.KV_P24 if kv is None else kv)
    return _MODELS[key]


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["mt3", "ismir2021"])
@pytest.mark.parametrize("mode", ["simt", "tf32x3", "tf32"])
@pytest.mark.parametrize("L", [1, 37, 300, 1024])
@pytest.mark.parametrize("B", [1, 3])
def test_model_logits_vs_float64(config, mode, L, B):
    """decode(decode=False) logits against the float64 oracle at the positions with target > 0: within 5e-4 of max |l64|
    and within max(4 e_f32, 2e-5), e_f32 the float32 oracle's own deviation (DESIGN.md section 4).  A padding tail, a 0
    inside sequence 0, an all-padding sequence 2 (finite logits, score 0).  TF32 (documented outside the bar): shape and
    finiteness only."""
    enc, din, tgt, l64, l32 = _case(config, L)
    enc, din, tgt, l64, l32 = enc[:B], din[:B], tgt[:B], l64[:B], l32[:B]
    m = _model(config, mode)
    e = _dev(enc)
    lg = m.decode(e, None, _dev(din), _dev(tgt), decode=False).cpu().numpy()
    sc = m.score(e, _dev(din), _dev(tgt)).cpu().numpy()
    assert lg.shape == l64.shape and lg.dtype == np.float32 and np.isfinite(lg).all() and np.isfinite(sc).all()
    assert (sc[tgt == 0] == 0).all()
    real = tgt > 0
    if mode == "tf32" or not real.any():
        return
    scale = np.abs(l64[real]).max()
    e_gpu = np.abs(lg[real] - l64[real]).max() / scale
    e_f32 = np.abs(l32[real] - l64[real]).max() / scale
    print(f"[{config} {mode} B={B} L={L}] logits vs fp64 {e_gpu:.2e} (fp32 oracle {e_f32:.2e})")
    assert e_gpu <= LOGIT_TOL and e_gpu <= max(4 * e_f32, 2e-5), (e_gpu, e_f32)


@pytest.mark.gpu
def test_model_full_size_tf32x3():
    """B = 64, T = 256, L = 1024 in TF32X3 (M = 65536 rows, 1536 self-attention work items per layer): sequences 0, 17, 63
    against float64 over all 1024 positions."""
    V = 1536
    rng = np.random.default_rng(64)
    enc = rng.standard_normal((64, 256, 512)).astype(np.float32)
    tgt = rng.integers(3, V, size=(64, 1024)).astype(np.int32)
    din = np.concatenate([np.zeros((64, 1), np.int32), tgt[:, :-1]], axis=1)
    pick = [0, 17, 63]
    l64 = decode_full(_params(V), O.T5Config(), enc[pick], din[pick], tgt[pick], np.float64)
    l32 = decode_full(_params(V), O.T5Config(), enc[pick], din[pick], tgt[pick], np.float32)
    m = _model("mt3", "tf32x3")
    lg = m.decode(_dev(enc), None, _dev(din), _dev(tgt), decode=False)[pick].cpu().numpy()
    scale = np.abs(l64).max()
    e_gpu, e_f32 = np.abs(lg - l64).max() / scale, np.abs(l32 - l64).max() / scale
    print(f"full size: logits vs fp64 {e_gpu:.2e} (fp32 oracle {e_f32:.2e})")
    assert e_gpu <= LOGIT_TOL and e_gpu <= max(4 * e_f32, 2e-5)


@pytest.mark.gpu
def test_trained_statistics_probes(monkeypatch):
    """test_trained_statistics' generated trained-regime weights, the decoder fed the float64 encoder output over 1024
    tokens, at the well-conditioned probes 0, 1, 31, 32, 65, 191.  SIMT: within max(4 e_f32, 2e-5), where 24-bit K/V rows
    of the step path are not.  TF32X3, with the wgmma and with the exact-fp32 attention (MT3_TC_ATTENTION=0), leaves that
    bar at these statistics, as 24-bit rows do, and is reported only (DESIGN.md section 4).  Prints the measured ratios."""
    import torch
    import test_trained_statistics as tsx
    from mt3_b200 import _lib, network
    params = tsx.trained_params()
    enc64 = O.encode(params, tsx.CFG, tsx.spectrogram((1274, 1275)), np.float64)
    toks = np.random.default_rng(12).integers(3, 1500, size=(2, 1024)).astype(np.int32)
    toks[:, 0] = 0
    tgt = np.concatenate([toks[:, 1:], np.full((2, 1), 5, np.int32)], axis=1)    # every position scored
    probe = [0, 1, 31, 32, 65, 191]
    l64 = O.decode_teacher_forced(params, tsx.CFG, enc64, toks, np.float64)[:, probe]
    l32 = O.decode_teacher_forced(params, tsx.CFG, enc64.astype(np.float32), toks, np.float32)[:, probe]
    scale = np.abs(l64).max()
    e32 = np.abs(l32 - l64).max(axis=(0, 2)) / scale
    for gm, tc_attn in ((_lib.GEMM_FP32_SIMT, True), (_lib.GEMM_TF32X3, False), (_lib.GEMM_TF32X3, True)):
        monkeypatch.setenv("MT3_TC_ATTENTION", "1" if tc_attn else "0")
        m = network.Transformer(_net_cfg(1536, enc_layers=8), params, device=DEV, max_batch=2, max_input_length=256,
                                max_decode_length=1024, gemm_mode=gm, kv_format=_lib.KV_P24)
        lg = m.decode(_dev(enc64.astype(np.float32)), None, _dev(toks), _dev(tgt), decode=False).cpu().numpy()[:, probe]
        del m
        torch.cuda.empty_cache()
        errs = np.abs(lg - l64).max(axis=(0, 2)) / scale
        bar = np.maximum(4 * e32, 2e-5)
        print(f"trained statistics gemm_mode={gm} tc_attention={tc_attn}: per probe err / e_f32 " +
              " ".join(f"{p}:{e:.1e}/{f:.1e}" for p, e, f in zip(probe, errs, e32)) + f"  worst err/bar {float((errs / bar).max()):.2f}")
        if gm == _lib.GEMM_FP32_SIMT:
            assert (errs <= bar).all(), (gm, errs, e32)


@pytest.mark.gpu
def test_agrees_with_step_path():
    """teacher_forced_logits (one decode step per position) of an MT3_KV_F32 model against the pass on the same tokens
    (B = 3, L = 300), at positions with target > 0: both are float32 implementations of the same logits."""
    from mt3_b200 import _lib
    enc, din, tgt, l64, l32 = _case("mt3", 300)
    tgt = np.where(tgt == 0, 7, tgt)             # the step path knows no padding: compare with every key visible
    m = _model("mt3", "tf32x3", _lib.KV_F32)
    e = _dev(enc)
    a = m.decode(e, None, _dev(din), _dev(tgt), decode=False).cpu().numpy()
    b = m.teacher_forced_logits(e, _dev(din)).cpu().numpy()
    d = np.abs(a - b).max() / np.abs(b).max()
    real = _case("mt3", 300)[2] > 0
    e_f32 = np.abs(l32[real] - l64[real]).max() / np.abs(l64[real]).max()
    print(f"pass vs step path: max |dlogit| / max |logit| {d:.2e} (fp32 oracle vs fp64 {e_f32:.2e})")
    assert d <= 2 * max(4 * e_f32, 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["simt", "tf32x3"])
def test_scores(mode):
    """score_batch equals a float64 log-softmax of the pass's own logits at the targets; it is within the summed
    per-token bar of the oracle's scores; the logits == NULL path gives bit-identical scores."""
    import torch
    from mt3_b200 import models
    enc, din, tgt, l64, l32 = _case("mt3", 300)
    m = _model("mt3", mode)
    e = _dev(enc)
    lg, sc_both = m._teacher_forced(e, _dev(din), _dev(tgt), None, True, True)
    sc = m.score(e, _dev(din), _dev(tgt))
    assert torch.equal(sc, sc_both)
    lg, sc = lg.cpu().numpy(), sc.cpu().numpy()
    own = token_scores_ref(lg, tgt)
    np.testing.assert_allclose(sc, own, rtol=0, atol=4e-6 * (1 + np.abs(lg).max()))
    wrapper = models.ContinuousInputsEncoderDecoderModel(m)
    # score_batch from the encoder input: compare with Transformer.score on the encoder's own output
    xin = np.random.default_rng(3).standard_normal((3, 256, 512)).astype(np.float32)
    batch = {"encoder_input_tokens": xin, "decoder_input_tokens": din, "decoder_target_tokens": tgt,
             "decoder_loss_weights": (tgt > 0).astype(np.int32)}
    sb = wrapper.score_batch(None, batch).cpu().numpy()
    own_b = token_scores_ref(m.decode(m.encode(_dev(xin)), None, _dev(din), _dev(tgt), decode=False).cpu().numpy(), tgt).sum(-1)
    assert sb.dtype == np.float32 and sb.shape == (3,)
    np.testing.assert_allclose(sb, own_b, rtol=1e-5, atol=1e-3)
    with pytest.raises(ValueError):
        wrapper.score_batch(None, batch, return_intermediates=True)
    # against the oracle: each token's error is at most that of its logit and of the log-sum-exp
    ref = token_scores_ref(l64, tgt)
    scale = np.abs(l64[tgt > 0]).max()
    bar = 2 * LOGIT_TOL * scale * (tgt > 0).sum(-1)
    assert (np.abs(sc.astype(np.float64).sum(-1) - ref.sum(-1)) <= bar).all()


@pytest.mark.gpu
def test_isolation_from_decode_state():
    """Greedy and beam-1 generate, with graphs, give bit-identical tokens before and after a teacher-forced call on the
    same handle."""
    m = _model("mt3", "tf32x3")
    x = _dev(np.random.default_rng(11).standard_normal((4, 256, 512)).astype(np.float32))
    before = [m.generate(x, num_steps=48, stop_at_eos=False, use_graph=True, decode=d).clone() for d in ("greedy", "beam1")]
    enc, din, tgt, _, _ = _case("mt3", 37)
    m.decode(_dev(enc), None, _dev(din), _dev(tgt), decode=False)
    m.score(_dev(enc), _dev(din), _dev(tgt))
    after = [m.generate(x, num_steps=48, stop_at_eos=False, use_graph=True, decode=d) for d in ("greedy", "beam1")]
    for a, b in zip(before, after):
        assert (a == b).all()


@pytest.mark.gpu
def test_errors():
    import torch
    from mt3_b200 import _lib
    m = _model("mt3", "simt")
    enc, din, tgt, _, _ = _case("mt3", 37)
    e, d, t = _dev(enc), _dev(din), _dev(tgt)
    with pytest.raises(ValueError):
        m.decode(e, None, torch.zeros((3, 1025), dtype=torch.int32, device=DEV), torch.ones((3, 1025), dtype=torch.int32, device=DEV),
                 decode=False)
    with pytest.raises(ValueError):
        m.decode(_dev(np.zeros((65, 256, 512), np.float32)), None, torch.zeros((65, 4), dtype=torch.int32, device=DEV),
                 torch.ones((65, 4), dtype=torch.int32, device=DEV), decode=False)
    bad = tgt.copy()
    bad[0, 3] = 1536
    with pytest.raises(ValueError):
        m.decode(e, None, d, _dev(bad), decode=False)
    with pytest.raises(ValueError):
        m.decode(e, None, d, None, decode=False)
    with pytest.raises(ValueError):
        m.decode(e, None, d, t, decoder_segment_ids=t, decode=False)
    with pytest.raises(ValueError):
        m.decode(e, None, d, t, enable_dropout=True, decode=False)
    lib = _lib.load()
    need = int(lib.mt3_teacher_forced_workspace_bytes(m._h, 3, 256, 37))
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.empty((3, 37), dtype=torch.float32, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    args = lambda ws_ptr, nb: (m._h, e.data_ptr(), 3, 256, d.data_ptr(), t.data_ptr(), None, 37, None, out.data_ptr(), ws_ptr, nb, s)  # noqa: E731
    assert lib.mt3_decode_teacher_forced(*args(ws.data_ptr(), need - 256)) == -4
    assert lib.mt3_decode_teacher_forced(*args(ws.data_ptr() + 16, need)) == -4
    assert lib.mt3_decode_teacher_forced(m._h, e.data_ptr(), 3, 256, d.data_ptr(), t.data_ptr(), None, 37, None, None, ws.data_ptr(),
                                         need, s) == -1
    assert lib.mt3_decode_teacher_forced(m._h, e.data_ptr(), 65, 256, d.data_ptr(), t.data_ptr(), None, 37, None, out.data_ptr(),
                                         ws.data_ptr(), need, s) == -2
    assert lib.mt3_decode_teacher_forced(*args(ws.data_ptr(), need)) == 0


@pytest.mark.gpu
def test_inference_model_score_end_to_end():
    """InferenceModel.score on synthetic weights: a 5 s clip (3 segments, a short tail) and a NoteSequence; equals
    score_batch on the same batches built by hand, every value finite."""
    import torch
    from mt3_b200 import inference, models, spectrograms
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=2)
    audio = O.sine_mix(5 * 16000, 77).astype(np.float32)
    ns = _dense_note_sequence()
    res = im.score(audio, ns)
    assert len(res) == 3
    assert all(np.isfinite(r['score']) and np.isfinite(r['token_scores']).all() for r in res)
    assert all(r['num_tokens'] > 0 for r in res)
    frames, times = im._audio_to_frames(audio)
    ds = im.preprocess(im.audio_to_dataset(audio))
    tg = inference.segment_score_targets(ns, im.codec, im.vocabulary, times, im.inputs_length, im.encoding_spec, 1024)
    wrapper = models.ContinuousInputsEncoderDecoderModel(im.model)
    hop = im.spectrogram_config.hop_width
    for s0 in range(0, 3, 2):
        s1 = min(3, s0 + 2)
        segs = np.zeros((s1 - s0, 256 * hop), np.float32)
        nv = np.zeros((s1 - s0,), np.int32)
        for j, ex in enumerate(ds[s0:s1]):
            flat = np.asarray(ex['inputs'], np.float32).reshape(-1)
            segs[j, :flat.size] = flat
            nv[j] = flat.size // hop
        spec = im._pad_inputs(spectrograms.compute_spectrogram(_dev(segs), im.spectrogram_config, n_valid_frames=_dev(nv)))
        batch = {"encoder_input_tokens": spec, **{k: v[s0:s1] for k, v in tg.items()}}
        sb = wrapper.score_batch(None, batch).cpu().numpy()
        np.testing.assert_allclose(sb, [np.float32(r['score']) for r in res[s0:s1]], rtol=1e-6, atol=1e-4)
    torch.cuda.synchronize()
