"""Logit bias in the decode loop (mt3_generate_biased, Transformer.generate(logit_bias=...), InferenceModel(programs=...,
drums=...), `python -m mt3_b200.transcribe --programs ... --no-drums`).

The rule, restated here in numpy: with bias [B, V] every token picker behaves exactly as if the model had produced
    l'[b, i] = -inf where bias[b, i] == -inf, else logits[b, i] + bias[b, i] (one float32 add)
so the existing restatements -- greedy (test_decode_loop_kernels.argmax_ref, test_decode_scores' log_softmax64), beam-size-1
(beam1_scored_trace, tied to oracle/beam_search.py) and sampling (test_sampling.sample_step_ref) -- are fed l'.  Forced
prompt positions are the caller's tokens even where suppressed; a zero bias is bit-identical to an unbiased call.
"""
import ctypes as C
import os

import numpy as np
import pytest

import test_decode_loop_kernels as DK
import test_decode_scores as DS
import test_sampling as TS

DEV = "cuda:0"
EOS, PAD = 1, 0
ALPHA = DK.ALPHA
_call, _p, _dev, _np, _same_bits = DK._call, DK._p, DK._dev, DK._np, DK._same_bits


def biased(l, bias):
    """l' of the rule, float32"""
    l, bias = np.asarray(l, np.float32), np.asarray(bias, np.float32)
    with np.errstate(invalid="ignore"):
        return np.where(np.isneginf(bias), np.float32(-np.inf), l + bias).astype(np.float32)


def _finite_floor(lp):
    """l' for test_sampling's restatement, whose ambiguity bar is infinite at -inf entries: -1e30 stands in for -inf (never
    drawn, zero mass, the same top-k / top-p cuts)"""
    return np.where(np.isneginf(lp), np.float32(-1e30), lp).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# CPU: the bias row, the host checks, the CLI
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nvb", [1, 127], ids=["mt3", "ismir2021"])
def test_program_logit_bias(nvb):
    """-inf exactly at the program ids outside `programs` and, with drums=False, at the drum range (codec index + 3); 0
    elsewhere; the defaults give all zeros; programs outside 0..127 and a vocabulary smaller than the codec are refused"""
    from mt3_b200 import event_codec, vocabularies as VOC
    codec = VOC.build_codec(VOC.VocabularyConfig(num_velocity_bins=nvb))
    V = VOC.num_embeddings(VOC.vocabulary_from_codec(codec))
    assert (VOC.program_logit_bias(codec, V) == 0).all() and VOC.program_logit_bias(codec, V).dtype == np.float32
    plo, phi = codec.event_type_range('program')
    dlo, dhi = codec.event_type_range('drum')
    for programs, drums in (([0], False), ([0, 1, 40, 127], True), ([], True), (None, False), (range(128), True)):
        b = VOC.program_logit_bias(codec, V, programs, drums)
        assert b.shape == (V,) and b.dtype == np.float32
        want = np.zeros(V, bool)
        for p in range(128):
            if programs is not None and p not in list(programs):
                want[codec.encode_event(event_codec.Event('program', p)) + 3] = True
        if not drums:
            want[dlo + 3:dhi + 4] = True
        np.testing.assert_array_equal(np.isneginf(b), want)
        assert (b[~want] == 0).all()
        assert not np.isneginf(b[:plo + 3]).any() and not np.isneginf(b[dhi + 4:]).any()
    for bad in ([128], [-1], [0, 200]):
        with pytest.raises(ValueError):
            VOC.program_logit_bias(codec, V, bad)
    with pytest.raises(ValueError):
        VOC.program_logit_bias(codec, codec.num_classes + 2)


def test_host_logit_bias_check():
    """float32 [V] or [B, V], numpy or torch; no NaN / +inf; every row keeps a finite id"""
    import torch
    from mt3_b200 import network
    t = object.__new__(network.Transformer)
    t.config, t.device = network.T5Config(vocab_size=16), torch.device("cpu")
    row = np.zeros(16, np.float32)
    row[3:9] = -np.inf
    assert t._check_logit_bias(row, 4).shape == (16,)
    assert t._check_logit_bias(torch.from_numpy(np.tile(row, (4, 1))), 4).shape == (4, 16)
    bad_rows = [row.astype(np.float64), row[:15], np.tile(row, (3, 1)), np.tile(row, (4, 2)), [0.0] * 16]
    for v in (np.nan, np.inf):
        r = np.tile(row, (4, 1))
        r[2, 5 if v == np.inf else 12] = v
        bad_rows.append(r)
    r = np.tile(row, (4, 1))
    r[1] = -np.inf
    bad_rows.append(r)
    for b in bad_rows:
        with pytest.raises(ValueError):
            t._check_logit_bias(b, 4)


def test_cli_program_flags():
    """--programs 0,1 --no-drums parse to InferenceModel's programs / drums; the defaults leave both off"""
    from mt3_b200 import transcribe
    ap = transcribe._parser()
    a = ap.parse_args(['in.wav', 'out.mid', '--checkpoint', 'synthetic'])
    assert a.programs is None and a.drums is True
    a = ap.parse_args(['in.wav', 'out.mid', '--checkpoint', 'synthetic', '--programs', '0,1,33', '--no-drums'])
    assert a.programs == [0, 1, 33] and a.drums is False
    for bad in ('128', 'piano', '0,,1', '-1'):
        with pytest.raises(SystemExit):
            ap.parse_args(['in.wav', 'out.mid', '--checkpoint', 'synthetic', '--programs', bad])


def test_inference_model_passes_the_bias(monkeypatch):
    """InferenceModel gives generate its bias row only when programs / drums restrict the instruments; bad programs are
    refused before any model is built"""
    import torch
    from mt3_b200 import inference
    im = object.__new__(inference.InferenceModel)
    assert im.logit_bias is None and im._bias_kw() == {}
    seen = []

    class _M:
        def generate(self, x, **kw):
            seen.append(kw)
            return torch.full((x.shape[0], 3), 5, dtype=torch.int32)

    class _Voc:
        def decode_tf(self, t):
            return t
    im.model, im.vocabulary, im.use_graph, im.device, im.decode = _M(), _Voc(), True, torch.device("cpu"), 'beam1'
    im.predict_tokens({'encoder_input_tokens': np.zeros((2, 4, 3), np.float32)})
    assert 'logit_bias' not in seen[-1]
    im.logit_bias = np.zeros(8, np.float32)
    im.predict_tokens({'encoder_input_tokens': np.zeros((2, 4, 3), np.float32)})
    assert seen[-1]['logit_bias'] is im.logit_bias and seen[-1]['decode'] == 'beam1'
    with pytest.raises(ValueError):
        inference.InferenceModel('synthetic', 'mt3', programs=[300])


def test_abi_biased_entry_point():
    """mt3_generate_biased is exported and bound; a NULL handle is MT3_ERR_BAD_ARG without a device"""
    from mt3_b200 import _lib
    header = open(os.path.join(DK.ROOT, "include", "mt3_b200.h")).read()
    assert "int mt3_generate_biased(" in header and "mt3_generate_biased" in _lib.EXPORTS
    lib = _lib.load()
    assert lib.mt3_generate_biased(None, None, 1, 0, None, 0, None, None, None, None, None, 0, None, None, 0, None) == -1


# ------------------------------------------------------------------------------------------------
# GPU: the pickers alone (libmt3kernels.so)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(DK.TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, F = C.c_void_p, C.c_int, C.c_float
    greedy = [P, I, I, P, P, P, P, I, P, P, P, I, I, P, P, I, I, P, I]
    beam = [P, I, I, P, P, P, P, I, P, P, P, P, P, F, I, P, P, I, I, P]
    sample = [P, I, I, P, P, P, P, I, P, P, P, I, F, P, P, I, I, P]
    sig = {"kh_last_error": ([], C.c_char_p), "kh_argmax_step_forced": (greedy, I), "kh_argmax_step_biased": (greedy + [P], I),
           "kh_beam1_step_forced": (beam, I), "kh_beam1_step_biased": (beam + [P], I), "kh_sample_step": (sample, I),
           "kh_sample_step_biased": (sample + [P], I), "kh_beam1_finalize_scored": ([P, I, I, I, P, P, P, P, P], I)}
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    return lib


def _run(kh, kind, lg, bias, plen, prompt, scored, sp=None, D=32):
    """`kind` ('greedy' | 'beam1' | 'sample') over the logits stream lg [steps, B, V] from position 0, every buffer with a
    sentinel row or column past its end; bias [B, V] (the biased kernel) or None (the unbiased one).  prompt [B, steps]
    holds the forced tokens at positions < plen.  beam1 ends with the finalize.  Returns every buffer the kernels write."""
    import torch
    steps, B, V = lg.shape
    L = steps + 2
    rng = np.random.default_rng(V)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    d_emb, d_pe = _dev(emb), _dev(DK._pe_with_guard(rng, steps + 1, D))
    d_lg = torch.full(((B + 1) * V,), float("nan"), dtype=torch.float32, device=DEV)
    d_bias = None if bias is None else _dev(np.concatenate([bias.ravel(), np.full(V, np.nan, np.float32)]))
    tok = np.full((B + 1, L), DK.SENT, np.int32)
    tok[:B, :steps] = np.where(np.arange(steps)[None] < plen[:, None], prompt, DK.SENT)
    fin = np.full(B + 1, DK.SENT, np.int32); fin[:B] = 0
    bf = np.full(2 * B + 2, np.nan, np.float32); bf[0:2 * B:2], bf[1:2 * B:2] = 0.0, -1.0e7
    bi = np.full(B + 1, DK.SENT, np.int32); bi[:B] = 0
    d = dict(tok=_dev(tok), fin=_dev(fin), st=_dev(np.array([0, 0, 0, DK.SENT], np.int32)), cur=_dev(np.full(B + 1, DK.SENT, np.int32)),
             y=torch.full(((B + 1) * D,), DK.YSENT, dtype=torch.float32, device=DEV), bf=_dev(bf), bi=_dev(bi),
             ts=torch.full(((B + 1) * L,), -5.0, dtype=torch.float32, device=DEV),
             fe=torch.full((B + 1,), float("nan"), dtype=torch.float32, device=DEV),
             sc=torch.full((B + 1,), float("nan"), dtype=torch.float32, device=DEV))
    d_pl = _dev(np.append(plen, DK.SENT).astype(np.int32))
    ts = _p(d["ts"]) if scored else None
    extra = () if bias is None else (_p(d_bias),)
    suffix = "" if bias is None else "_biased"
    d_sp = TS._sp_dev(sp) if kind == "sample" else None
    for s in range(steps):
        d_lg[:B * V] = _dev(lg[s].ravel())
        head = (_p(d_lg), V, B, _p(d["cur"]), _p(d["fin"]), _p(d["tok"]), ts, L, _p(d_pl))
        tail = (_p(d_emb), _p(d_pe), steps + 1, D, _p(d["y"]))
        if kind == "greedy":
            _call(kh, "kh_argmax_step" + (suffix or "_forced"), *head, None, _p(d["st"]), 1, 0, *tail, B, *extra)
        elif kind == "beam1":
            _call(kh, "kh_beam1_step" + (suffix or "_forced"), *head, _p(d["st"]), _p(d["bf"]), _p(d["fe"]) if scored else None,
                  _p(d["bi"]), ALPHA, steps, *tail, *extra)
        else:
            _call(kh, "kh_sample_step" + suffix, *head, _p(d["st"]), _p(d_sp), sp["topk"], sp["topp"], *tail, *extra)
    if kind == "beam1":
        _call(kh, "kh_beam1_finalize_scored", _p(d["tok"]), B, L, steps, _p(d["bi"]), ts, _p(d["bf"]), _p(d["fe"]) if scored else None,
              _p(d["sc"]) if scored else None)
    out = {k: _np(v) for k, v in d.items()}
    out["tok"], out["ts"] = out["tok"].reshape(B + 1, L), out["ts"].reshape(B + 1, L)
    assert (out["tok"][B] == DK.SENT).all() and (out["ts"][B] == -5.0).all()
    if kind != "beam1":                                  # the finalize zeroes the columns past the steps
        assert (out["tok"][:, steps:] == DK.SENT).all() and (out["ts"][:, steps:] == -5.0).all()
    return out


def _bias_rows(rng, lg, V, nan_allowed=True):
    """[B, V] biases over the stream lg [steps, B, V]: random finite ones, a program-style mask, -inf on the row maximum of
    the first step, on EOS, on all but one id (EOS, 0 or another), only one non-EOS id left, plus zeros.  NaN logits at a
    suppressed id, and with nan_allowed at an allowed id from step 2 on (in lg, in place)"""
    B = lg.shape[1]
    bias = (rng.standard_normal((B, V)) * 2).astype(np.float32)
    for b in range(B):
        k = b % 9
        if k == 0:
            bias[b] = 0.0
        elif k == 1:
            bias[b, V // 3:V // 3 + 250] = -np.inf
        elif k == 2:
            bias[b, int(np.argmax(np.where(np.isnan(lg[0, b]), -np.inf, lg[0, b])))] = -np.inf
        elif k == 3:
            bias[b, EOS] = -np.inf
        elif k in (4, 5):
            keep = (EOS, 0, 7 + b)[b % 3]
            bias[b] = -np.inf
            bias[b, keep] = 0.5
        elif k == 6:
            bias[b] = -np.inf
            bias[b, [EOS, 11 + b]] = 0.0
        elif k == 7:
            bias[b, :V // 2] = -np.inf
            lg[:, b, 5] = np.nan                    # suppressed: never emitted
        elif k == 8 and nan_allowed:
            lg[2:, b, V - 3] = np.nan                # allowed: a NaN row from step 2 on
    return bias


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664])
@pytest.mark.parametrize("kind", ["greedy", "beam1", "sample"])
def test_zero_bias_is_bit_identical(kh, kind, V):
    """The biased picker with a zero bias equals the unbiased kernel bit for bit -- tokens, token scores, finished, state,
    tok_cur, y_next and beam1's state -- over 10 steps of the crafted streams (ties, NaN, -inf, signed zeros, EOS wins),
    B = 64, scored and unscored, with forced prompt positions"""
    B, steps = 64, 10
    lg = DS._stream(V, B, steps, seed=V + 3)
    rng = np.random.default_rng(5)
    plen = np.where(np.arange(B) % 5 == 0, 4, 0).astype(np.int32)
    prompt = rng.integers(2, V, (B, steps)).astype(np.int32)
    configs = [None] if kind != "sample" else [{"temperature": T, "topk": k, "topp": p, "key": (3, 4), "rescale": r}
                                               for T, k, p, r in ((1.0, 0, 0.0, True), (0.7, 40, 0.9, True), (1.3, 0, 0.8, False))]
    for sp in configs:
        for scored in (False, True):
            want = _run(kh, kind, lg, None, plen, prompt, scored, sp)
            got = _run(kh, kind, lg, np.zeros((B, V), np.float32), plen, prompt, scored, sp)
            for k in want:
                _same_bits(f"{kind} V={V} scored={scored} {sp}: {k}", got[k], want[k])


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664])
def test_greedy_biased_against_restatement(kh, V):
    """argmax_step_biased_kernel over 10 steps, B = 64: tokens equal greedy's restatement fed l', token scores
    log_softmax64(l')[next] within lp_bar (NaN for a NaN row), forced prompt tokens emitted even where suppressed, with score
    0; no suppressed id emitted outside the prompt"""
    B, steps = 64, 10
    rng = np.random.default_rng(V)
    lg = DS._stream(V, B, steps, seed=V)
    bias = _bias_rows(rng, lg, V)
    plen = np.where(np.arange(B) % 4 == 1, 3, 0).astype(np.int32)
    prompt = np.zeros((B, steps), np.int32)
    prompt[:, :3] = rng.integers(2, V, (B, 3))
    for b in range(B):
        sup = np.flatnonzero(np.isneginf(bias[b]) & (np.arange(V) >= 2))
        if sup.size:
            prompt[b, 1] = sup[b % sup.size]             # a suppressed id, forced
    out = _run(kh, "greedy", lg, bias, plen, prompt, True)
    tok, ts = out["tok"][:B], out["ts"][:B]
    fin = np.zeros(B, bool)
    for s in range(steps):
        lp = biased(lg[s], bias)
        for b in range(B):
            if s < plen[b]:
                assert tok[b, s] == prompt[b, s] and ts[b, s] == 0.0
                continue
            if fin[b]:
                assert tok[b, s] == PAD and ts[b, s] == 0.0
                continue
            t = int(DK.argmax_ref(lp[b][None])[0])
            assert tok[b, s] == t, (s, b, tok[b, s], t)
            want = DS.log_softmax64(lp[b])[t]
            if np.isnan(want):
                assert np.isnan(ts[b, s])
            else:
                assert not np.isneginf(bias[b, t]) or np.isneginf(lp[b]).all()
                assert abs(ts[b, s] - want) <= DS.lp_bar(lp[b], lp[b, t]), (s, b, ts[b, s], want)
            fin[b] |= t == EOS
    np.testing.assert_array_equal(out["fin"][:B].astype(bool), fin)
    assert not fin[np.isneginf(bias[:, EOS])].any()


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664])
def test_beam1_biased_against_restatement(kh, V):
    """beam1_step_biased_kernel + finalize, 8 steps, on test_decode_loop_kernels' beam scenarios and random rows under the
    biases of _bias_rows (NaN at suppressed ids only: partly-NaN rows carry no beam1 parity claim): tokens, token scores and
    the score equal beam1_scored_trace fed l', within its bars; a row with one non-EOS id left continues with it"""
    sc = DK.beam_scenarios(V)
    L = DK.BEAM_L
    rng = np.random.default_rng(V + 1)
    rows = [sc[n] for n in sc]
    B = 45
    lg = np.stack(rows + [(rng.standard_normal((L, V)) * 3).astype(np.float32) for _ in range(B - len(rows))])   # [B, L, V]
    lg_s = np.ascontiguousarray(lg.transpose(1, 0, 2))
    bias = _bias_rows(rng, lg_s, V, nan_allowed=False)
    out = _run(kh, "beam1", lg_s, bias, np.zeros(B, np.int32), np.zeros((B, L), np.int32), True)
    tok, ts, score = out["tok"][:B, :L], out["ts"][:B, :L], out["sc"][:B]
    for b in range(B):
        lp = biased(lg_s[:, b], bias[b])
        with np.errstate(invalid="ignore"):
            t = DS.beam1_scored_trace(lp, L)
        bars = DK.beam1_trace(_finite_floor(lp), L)["steps"]          # beam1_trace's bars are NaN at -inf entries
        np.testing.assert_array_equal(tok[b], t["tokens"], err_msg=f"row {b}")
        n = t["fin_len"]
        upto = n if n else L
        for i in range(upto):
            v = lp[i, EOS] if n and i == n - 1 else lp[i, t["tokens"][i]]
            if np.isfinite(t["token_scores"][i]):
                assert abs(ts[b, i] - t["token_scores"][i]) <= DS.lp_bar(lp[i], v), (b, i)
        bar = bars[-1][3] if n else bars[-1][1]
        if np.isfinite(t["score"]) and len(bars) == len(t["steps"]):
            assert abs(score[b] - t["score"]) <= bar, (b, score[b], t["score"])
        if b % 9 == 6:                                   # EOS and one other id allowed
            assert set(tok[b, :upto].tolist()) <= {EOS, 11 + b}, tok[b]


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664])
def test_sample_biased_against_restatement(kh, V):
    """sample_step_biased_kernel, one step per configuration, B = 64: tokens and scores equal test_sampling's restatement fed
    l' outside flagged picks, forced suppressed prompt tokens, top-k larger than the allowed count, top-p, both, rescaled
    and raw scores; no suppressed id is drawn"""
    B = 64
    rng = np.random.default_rng(V + 2)
    flagged = total = 0
    for ci, (T, k, p, rescale) in enumerate(TS.KERNEL_CONFIGS + [(1.0, 600, 0.0, True), (0.8, 900, 0.95, False)]):
        sp = {"temperature": T, "topk": k, "topp": p, "key": (0xB1A5 + ci, 9), "rescale": rescale}
        lg = (rng.standard_normal((1, B, V)) * 2).astype(np.float32)
        bias = _bias_rows(rng, lg, V)
        plen = np.where(np.arange(B) % 10 == 3, 1, 0).astype(np.int32)
        prompt = np.zeros((B, 1), np.int32)
        prompt[:, 0] = [np.flatnonzero(np.isneginf(bias[b]) & (np.arange(V) >= 2))[0] if np.isneginf(bias[b, 2:]).any() else 5
                        for b in range(B)]
        out = _run(kh, "sample", lg, bias, plen, prompt, True, sp)
        lp = biased(lg[0], bias)
        nxt, s, fin, flag = TS.sample_step_ref(_finite_floor(lp), np.zeros(B, bool), plen, prompt[:, 0], 0, sp)
        got, ts = out["tok"][:B, 0], out["ts"][:B, 0]
        ok = ~flag
        flagged += int(flag.sum())
        total += B
        np.testing.assert_array_equal(got[ok], nxt[ok], err_msg=f"config {ci}")
        for b in range(B):
            if plen[b]:
                assert got[b] == prompt[b, 0] and ts[b] == 0.0
            elif not np.isnan(lp[b]).any():
                assert not np.isneginf(bias[b, got[b]]), (ci, b, got[b])
                _, lo, hi = TS.keep_mask(_finite_floor(lp[b]) / np.float32(T), k, p)
                if ok[b] and (not rescale or (lo == hi).all()):       # a kept set within the top-p bar of its cut: no score claim
                    bar = TS.score_bar(_finite_floor(lp[b]), T, k, p, nxt[b], rescale)
                    assert abs(ts[b] - s[b]) <= bar, (ci, b, ts[b], s[b], bar)
            else:
                assert np.isnan(ts[b])
    print(f"V={V}: {flagged} of {total} picks flagged")
    assert flagged <= total // 20


# ------------------------------------------------------------------------------------------------
# GPU: the model against the float64 oracle
# ------------------------------------------------------------------------------------------------
def _program_bias(config, V, rng):
    """a program mask (programs 0 and 1, no drums) of the config's codec, plus a small random bias on the allowed ids"""
    from mt3_b200 import vocabularies as VOC
    codec = VOC.build_codec(VOC.VocabularyConfig(num_velocity_bins=1 if config == "mt3" else 127))
    mask = VOC.program_logit_bias(codec, V, [0, 1], drums=False)
    return np.where(np.isneginf(mask), mask, (rng.standard_normal(V) * 0.3).astype(np.float32)).astype(np.float32)


MODEL_MODES = ["mt3-simt-f32", "mt3-tf32x3-p24", "ismir2021-tf32x3-p24"]


@pytest.mark.gpu
@pytest.mark.parametrize("decode", ["greedy", "beam1", "sample"])
@pytest.mark.parametrize("mode", MODEL_MODES)
def test_biased_generate_against_float64(mode, decode):
    """Biased generate on the 2-layer models (EOS-boosted weights, B = 8, 40 steps) with a program mask, without and with a
    3-token prompt that forces a suppressed id: graphs on equal graphs off bit for bit; no suppressed id outside the prompt;
    the rows teacher-forced through the float64 oracle: each free position picks the restatement's token from l' of the
    oracle's logits unless the pick is ambiguous within the logits' bar (the sampling tests' rule), token scores within
    twice that bar"""
    import torch
    from mt3_b200 import _lib
    config, gm, kv = mode.split("-")
    gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3}[gm]
    kv = {"f32": _lib.KV_F32, "p24": _lib.KV_P24}[kv]
    T_in, V = TS._CFG[config]
    L, B = TS._L, TS._B
    rng = np.random.default_rng(21)
    bias = _program_bias(config, V, rng)
    sup = np.flatnonzero(np.isneginf(bias))
    m = TS._model(config, gm, kv)
    x = TS._inputs(config)
    xg = torch.from_numpy(x).to(DEV)
    sp = {"temperature": 0.9, "topk": 0, "topp": 0.95, "key": (0, 31), "rescale": True}
    kw = dict(num_steps=L, stop_at_eos=False, decode=decode, return_scores=True, logit_bias=bias)
    if decode == "sample":
        kw.update(temperature=0.9, topp=0.95, seed=31)
    prompt = np.zeros((B, 3), np.int32)
    prompt[:, 0], prompt[:, 1], prompt[:, 2] = 7, sup[0], 9
    checked = 0
    for pr in (None, prompt):
        plen = np.zeros(B, np.int64) if pr is None else np.full(B, 3)
        tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, prompt=pr, **kw))
        plain = [t.cpu().numpy() for t in m.generate(xg, prompt=pr, use_graph=False, **kw)]
        np.testing.assert_array_equal(plain[0], tok)
        _same_bits(f"{mode} {decode}: token scores, graph vs plain", plain[1], ts)
        _same_bits(f"{mode} {decode}: scores, graph vs plain", plain[2], sc)
        free = np.arange(L)[None] >= plen[:, None]
        assert not np.isin(tok[free], sup).any(), "a suppressed id was emitted"
        l64, l32 = TS._oracle_along(config, x, tok)
        scale = np.abs(l64).max()
        bar = max(4 * np.abs(l32 - l64).max() / scale, 2e-5) * scale
        n_fin = np.where((tok == EOS).any(1), np.argmax(tok == EOS, 1) + 1, L)
        for b in range(B):
            for i in range(L):
                if i < plen[b]:
                    assert tok[b, i] == pr[b, i] and ts[b, i] == 0.0
                    continue
                if i >= n_fin[b]:
                    assert tok[b, i] == PAD and ts[b, i] == 0.0
                    continue
                lp = np.where(np.isneginf(bias), -np.inf, l64[b, i] + bias.astype(np.float64))
                if decode == "sample":
                    t, want, amb = TS.sample_pick_ref(_finite_floor(lp.astype(np.float32)), sp["temperature"], sp["topk"], sp["topp"],
                                                      sp["key"], b, i, sp["rescale"], lbar=bar)
                    sbar = 2 * bar / sp["temperature"]
                else:
                    cand = lp.copy()
                    eos_here = decode == "beam1" and i == n_fin[b] - 1 and tok[b, i] == EOS
                    if decode == "beam1" and not eos_here:
                        cand[EOS] = -np.inf                  # the live prefix continues with the best non-EOS id
                    if eos_here:
                        t, amb = EOS, False
                    else:
                        srt = np.sort(cand)[::-1]
                        t, amb = int(np.argmax(cand)), srt[0] - srt[1] <= 2 * bar
                    want = DS.log_softmax64(lp)[tok[b, i]]
                    sbar = 2 * bar
                if amb:
                    continue
                checked += 1
                assert tok[b, i] == t, (mode, decode, b, i, tok[b, i], t)
                assert abs(ts[b, i] - want) <= sbar, (mode, decode, b, i, ts[b, i], want, sbar)
    print(f"{mode} {decode}: {checked} positions checked")
    assert checked >= B * 4


# ------------------------------------------------------------------------------------------------
# GPU: bench's configuration, errors, end to end
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_zero_bias_bit_identity_at_bench_configuration():
    """mt3, B = 64, 1024 steps, TF32X3, 24-bit rows, graphs: a zero bias gives the unbiased tokens and scores bit for bit
    in greedy, beam1 and sampled decoding; a [V] bias (bias_ld = 0) equals the same row repeated [B, V]"""
    import torch
    from mt3_b200 import _lib, inference
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=64, gemm_mode=_lib.GEMM_TF32X3, kv_format=_lib.KV_P24)
    m = im.model
    from mt3_b200 import spectrograms
    from oracle import mt3_oracle as O
    audio = np.stack([O.sine_mix(256 * 128, seed=4000 + i) for i in range(64)])
    x = spectrograms.compute_spectrogram(torch.from_numpy(audio).to(DEV), spectrograms.SpectrogramConfig())
    V = m.config.vocab_size
    row = _program_bias("mt3", V, np.random.default_rng(2))
    for decode, extra in (("greedy", {}), ("beam1", {}), ("sample", dict(temperature=1.0, topk=40, seed=5))):
        kw = dict(stop_at_eos=False, use_graph=True, decode=decode, return_scores=True, **extra)
        want = [t.cpu().numpy() for t in m.generate(x, **kw)]
        assert m.last_steps_run == 1024
        got = [t.cpu().numpy() for t in m.generate(x, logit_bias=np.zeros(V, np.float32), **kw)]
        for a, w, name in zip(got, want, ("tokens", "token scores", "scores")):
            _same_bits(f"{decode}: zero bias, {name}", a, w)
        one = [t.cpu().numpy() for t in m.generate(x, logit_bias=row, **kw)]
        rep = [t.cpu().numpy() for t in m.generate(x, logit_bias=np.tile(row, (64, 1)), **kw)]
        for a, w, name in zip(one, rep, ("tokens", "token scores", "scores")):
            _same_bits(f"{decode}: [V] vs [B, V], {name}", a, w)
        assert not np.isin(one[0], np.flatnonzero(np.isneginf(row))).any()
    del im, m
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_biased_generate_error_codes():
    """NaN, +inf, an all -inf row and a bad bias_ld are MT3_ERR_BAD_ARG before any decode; a following unbiased call equals
    a fresh model's, bit for bit"""
    import torch
    from mt3_b200 import _lib
    m = TS._model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    fresh = TS._model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    x = torch.from_numpy(TS._inputs("mt3")).to(DEV)
    B, L, V = TS._B, TS._L, TS._CFG["mt3"][1]
    want = [t.cpu().numpy() for t in fresh.generate(x, num_steps=L, stop_at_eos=False, return_scores=True)]
    m.generate(x, num_steps=L, stop_at_eos=False, logit_bias=np.zeros(V, np.float32))
    out = torch.empty((B, L), dtype=torch.int32, device=DEV)
    ran = C.c_int32(-1)

    def call(bias, ld):
        d = torch.from_numpy(np.ascontiguousarray(bias, np.float32)).to(DEV)
        r = m._lib.mt3_generate_biased(m._h, x.data_ptr(), L, 0, None, 0, out.data_ptr(), None, None, C.byref(ran), None, 0, None,
                                       d.data_ptr(), ld, m._stream())
        torch.cuda.synchronize()
        return r
    good = np.zeros((B, V), np.float32)
    assert call(good, V) == 0 and ran.value == L
    for bad_at, val in (((3, 17), np.nan), ((5, 2), np.inf), ((0, 0), np.nan)):
        b = good.copy()
        b[bad_at] = val
        ran.value = -1
        assert call(b, V) == -1 and ran.value == -1, (bad_at, val)
        assert "logit_bias row %d" % bad_at[0] in m._lib.mt3_last_error().decode()
    b = good.copy()
    b[6] = -np.inf
    assert call(b, V) == -1 and ran.value == -1
    for ld in (1, V - 1, -V):
        assert call(good, ld) == -1 and ran.value == -1, ld
    got = [t.cpu().numpy() for t in m.generate(x, num_steps=L, stop_at_eos=False, return_scores=True)]
    for a, w in zip(got, want):
        _same_bits("unbiased after refused biases vs a fresh model", a, w)
    with pytest.raises(ValueError):
        m.generate(x, logit_bias=np.full(V, np.nan, np.float32))


@pytest.mark.gpu
def test_transcribe_with_restricted_instruments(tmp_path, capsys):
    """InferenceModel(programs=[0], drums=False) on synthetic audio and weights: every note is program 0 and not a drum;
    no suppressed id in the raw tokens; the CLI with --programs 0 --no-drums writes the MIDI file the API calls build"""
    import test_transcribe_cli as TC
    from mt3_b200 import audio_io, inference, note_decoding, transcribe
    TC._wav(tmp_path / 'in.wav')
    audio = audio_io.load_audio(str(tmp_path / 'in.wav'), 16000)
    im = inference.InferenceModel('synthetic:3', 'mt3', device=DEV, batch_size=4, programs=[0], drums=False)
    sup = np.flatnonzero(np.isneginf(im.logit_bias))
    assert sup.size == 127 + 128
    ns = im(audio)
    print(f"{len(ns.notes)} notes")
    assert all(n.program == 0 and not n.is_drum for n in ns.notes)
    segs = np.stack([np.pad(a, (0, 256 * 128 - a.size)) for a in np.array_split(audio, 3)])
    raw = im.transcribe_segments(segs.astype(np.float32), decoded=False)
    assert not np.isin(raw, sup).any()
    for d in ("beam1", "sample"):
        im.decode = d
        assert not np.isin(im.transcribe_segments(segs.astype(np.float32), decoded=False), sup).any()
    rc = transcribe.main([str(tmp_path / 'in.wav'), str(tmp_path / 'out.mid'), '--checkpoint', 'synthetic:3', '--batch-size', '4',
                          '--programs', '0', '--no-drums'])
    assert rc == 0
    capsys.readouterr()
    assert (tmp_path / 'out.mid').read_bytes() == note_decoding.note_sequence_to_midi_bytes(ns)
