"""Prompted decoding (mt3_generate_prompted, Transformer.generate(prompt=...), predict_batch_with_aux(prompt_with_targets=True),
InferenceModel.transcribe_segments(prompts=...)): each row's non-zero prompt prefix is forced, the loop chooses from its end
on, and the prefix all rows share is prefilled into the K/V cache by one teacher-forced pass.

CPU: a numpy restatement of prompted greedy and prompted beam-size-1 (T5X's convention for forced prompts: forced tokens
score 0, make no finished hypothesis, and leave the live log-probability at 0), tied to oracle/beam_search.py on crafted
logits; the wrapper and the host-side prompt check.
GPU: the forced token pickers alone against the restatement; the model against float64 in SIMT and TF32X3 in every K/V
row format, ragged prompts, prefill below and above its threshold, against the step path, graph on and off; bench.py's
configuration (bit identity when unprompted, self-consistency with a greedy run); error codes; transcribe_segments.
"""
import ctypes as C

import numpy as np
import pytest

import test_decode_loop_kernels as DK
import test_decode_scores as DS
from oracle import beam_search as BS
from oracle import mt3_oracle as O

DEV = "cuda:0"
EOS, PAD = 1, 0
ALPHA = DK.ALPHA
_call, _p, _dev, _np, _same_bits = DK._call, DK._p, DK._dev, DK._np, DK._same_bits


# ------------------------------------------------------------------------------------------------
# numpy restatement
# ------------------------------------------------------------------------------------------------
def prompt_lengths(prompt):
    prompt = np.asarray(prompt)
    if prompt.shape[1] == 0:
        return np.zeros(prompt.shape[0], np.int64)
    z = prompt == 0
    return np.where(z.any(1), z.argmax(1), prompt.shape[1])


def prompted_decode(step_fn, B, L, prompt, beam1):
    """Prompted greedy (beam1=False) or T5X beam search at num_decodes = 1 (beam1=True), in float64, for B sequences that
    advance in lockstep.  step_fn(cur int [B], i) -> logits [B, V] of position i given the token fed there (BOS 0 at
    i = 0, then the previous emitted / live token); it is called for every i < L in order.  At i < p_b the prompt token
    is emitted with score 0; beam1 makes no finished hypothesis there and its live log-probability stays 0.  Returns
    tokens int32 [B, L], token scores [B, L] and sequence scores [B] as the library defines them."""
    prompt = np.zeros((B, 0), np.int64) if prompt is None else np.asarray(prompt)
    p = prompt_lengths(prompt)
    toks, ts = np.zeros((B, L), np.int32), np.zeros((B, L))
    cur = np.zeros(B, np.int64)
    done = np.zeros(B, bool)
    live, fin = np.zeros(B), np.full(B, BS.NEG_INF)
    fin_len, fin_lp_eos = np.zeros(B, np.int64), np.zeros(B)
    settled = np.zeros(B, bool)
    for i in range(L):
        lg = np.asarray(step_fn(cur.copy(), i))
        nxt = np.zeros(B, np.int64)
        for b in range(B):
            if i < p[b]:
                nxt[b] = toks[b, i] = prompt[b, i]
                continue
            lp = DS.log_softmax64(lg[b])
            if not beam1:
                t = PAD if done[b] else int(DK.argmax_ref(lg[b][None])[0])
                toks[b, i], nxt[b] = t, t
                ts[b, i] = 0.0 if done[b] else lp[t]
                done[b] |= t == EOS
                continue
            if i > 0 and fin_len[b] > 0 and not settled[b] and fin[b] > live[b] / BS.brevity_penalty(ALPHA, L):
                settled[b] = True
            order = sorted((k for k in range(lg.shape[1]) if k != EOS), key=lambda k: (-lg[b, k], k))
            t1, t2 = order[0], order[1]
            nxt[b] = t1
            if settled[b]:
                continue
            if lg[b, EOS] > lg[b, t2] or (lg[b, EOS] == lg[b, t2] and EOS < t2):
                cand = (live[b] + lp[EOS]) / BS.brevity_penalty(ALPHA, i + 1)
                if cand > fin[b]:
                    fin[b], fin_len[b], fin_lp_eos[b] = cand, i + 1, lp[EOS]
            live[b] += lp[t1]
            toks[b, i], ts[b, i] = t1, lp[t1]
        cur = nxt
    if not beam1:
        return toks, ts, ts.sum(1)
    for b in range(B):
        n = fin_len[b]
        if n:
            toks[b, n - 1], ts[b, n - 1] = EOS, fin_lp_eos[b]
            toks[b, n:], ts[b, n:] = 0, 0.0
    return toks, ts, np.where(fin_len > 0, fin, live)


def _table_fn(lg):
    """step_fn of prefix-independent tables lg [B, L, V]"""
    return lambda cur, i: lg[:, i]


def _crafted(V, B, L, seed):
    """[B, L, V] float32 logits: EOS on top at scattered positions, the rest Gaussian"""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((B, L, V)) * 3).astype(np.float32)
    for b in range(B):
        for i in range(L):
            if (b + 2 * i) % 5 == 0:
                x[b, i, EOS] = np.float32(20.0)
            elif (b + i) % 4 == 0:                         # EOS second: a beam1 finish without a greedy stop
                x[b, i, EOS] = x[b, i].max() - np.float32(0.05)
    return x


def test_empty_prompt_equals_greedy_and_beam_search():
    """An empty prompt (None, [B, 0], or all rows 0) reproduces BS.greedy and BS.beam_search exactly, on test_beam1's
    tables, the kernel tests' beam scenarios and crafted streams."""
    cases = {f"test_beam1/{k}": v[None] for k, v in DS._test_beam1_tables().items()}
    for V in (257, 33):
        cases.update({f"V={V}/{k}": v[None] for k, v in DK.beam_scenarios(V).items()})
    cases["crafted"] = _crafted(64, 6, 12, seed=1)
    for name, lg in cases.items():
        B, L, _ = lg.shape
        for prompt in (None, np.zeros((B, 0), np.int32), np.zeros((B, 3), np.int32)):
            tok, ts, sc = prompted_decode(_table_fn(lg), B, L, prompt, beam1=False)
            want = BS.greedy(lambda pre, s: lg[:, None, s], B, L)
            np.testing.assert_array_equal(tok, want, err_msg=name)
            tok, ts, sc = prompted_decode(_table_fn(lg), B, L, prompt, beam1=True)
            want, score = BS.beam_search(lambda pre, s: lg[:, None, s], B, L)
            np.testing.assert_array_equal(tok, want, err_msg=name)
            np.testing.assert_allclose(sc, score, rtol=1e-12, atol=0, err_msg=name)


def test_forced_prefix_scores_and_finishes():
    """Prompted restatement on crafted logits with EOS ranked first or second inside the prompts: the rows start with their
    prompts; forced positions score 0 and greedy's score is the sum over the free ones; no row finishes inside its prompt
    (beam1 makes no finished hypothesis there), and beam1's score at a finish is sum(free token scores) / bp(n), n the full
    length; the continuation after the prompt is the unprompted search started from the prompt's state."""
    V, B, L = 48, 6, 14
    lg = _crafted(V, B, L, seed=2)
    prompt = np.zeros((B, 9), np.int32)
    rng = np.random.default_rng(3)
    plen = [0, 1, 4, 9, 6, 9]
    for b, n in enumerate(plen):
        prompt[b, :n] = rng.integers(2, V, n)
        if n >= 2:
            lg[b, 1, EOS] = np.float32(20.0)            # EOS on top inside the prompt: ignored there
    for beam1 in (False, True):
        tok, ts, sc = prompted_decode(_table_fn(lg), B, L, prompt, beam1)
        for b, n in enumerate(plen):
            np.testing.assert_array_equal(tok[b, :n], prompt[b, :n])
            assert (ts[b, :n] == 0).all()
            assert not (tok[b, :n] == EOS).any()
            if n >= 2:
                assert lg[b, 1].argmax() == EOS
            if not beam1:
                assert sc[b] == ts[b].sum()
            elif (tok[b] == EOS).any():
                e = int(np.argmax(tok[b] == EOS)) + 1
                assert e > n
                assert abs(sc[b] - ts[b, :e].sum() / BS.brevity_penalty(ALPHA, e)) <= 1e-12 * abs(sc[b])
            else:
                assert abs(sc[b] - ts[b].sum()) <= 1e-12 * max(1.0, abs(sc[b]))
        # the continuation of a fully forced row is the unprompted search on the remaining table, positions shifted
        b, n = 3, plen[3]
        sub = lg[b:b + 1, n:]
        if beam1:
            want, _ = BS.beam_search(lambda pre, s: sub[:, None, s], 1, L - n)
        else:
            want = BS.greedy(lambda pre, s: sub[:, None, s], 1, L - n)
        if not beam1:
            np.testing.assert_array_equal(tok[b, n:], want[0])


# ------------------------------------------------------------------------------------------------
# wrapper and host-side check (CPU)
# ------------------------------------------------------------------------------------------------
class _PromptModule:
    def __init__(self):
        self.prompts = []

    def generate(self, x, stop_at_eos=True, decode='greedy', return_scores=False, prompt=None):
        self.prompts.append(None if prompt is None else np.array(prompt))
        toks = np.zeros((x.shape[0], 8), np.int32)
        return (toks, np.zeros((x.shape[0], 8), np.float32), np.zeros(x.shape[0], np.float32)) if return_scores else toks


def test_predict_batch_with_aux_prompt_with_targets():
    """prompt_with_targets=True hands decoder_input_tokens[:, 1:] to the module as its prompt; False hands none; a non-zero
    column 0 is rejected; predict_batch is unchanged."""
    from mt3_b200 import models
    din = np.array([[0, 5, 6, 0], [0, 7, 0, 0]], np.int32)
    batch = {'encoder_input_tokens': np.zeros((2, 5, 4), np.float32), 'decoder_input_tokens': din}
    mod = _PromptModule()
    m = models.ContinuousInputsEncoderDecoderModel(mod, input_depth=4)
    m.predict_batch_with_aux(None, batch, prompt_with_targets=True)
    np.testing.assert_array_equal(mod.prompts[-1], din[:, 1:])
    m.predict_batch_with_aux(None, batch)
    assert mod.prompts[-1] is None
    m.predict_batch(None, batch)
    assert mod.prompts[-1] is None
    bad = dict(batch, decoder_input_tokens=din + np.array([[0], [3]], np.int32) * (np.arange(4) == 0))
    with pytest.raises(ValueError, match="BOS"):
        m.predict_batch_with_aux(None, bad, prompt_with_targets=True)


def test_host_prompt_check():
    """Transformer's host-side prompt check: EOS, ids >= vocab, negative ids, non-zero ids after a 0, a length above
    num_steps and a batch mismatch are rejected; valid ragged prompts (numpy or torch) pass as int32."""
    import torch
    from mt3_b200 import network
    t = object.__new__(network.Transformer)
    t.device = torch.device("cpu")
    t.config = network.T5Config(vocab_size=16)
    ok = np.array([[2, 15, 0], [0, 0, 0], [4, 5, 6]], np.int64)
    assert t._check_prompt(ok, 3, 3).dtype == torch.int32
    assert t._check_prompt(torch.from_numpy(ok), 3, 5).shape == (3, 3)
    bad = {"EOS": [[2, 1, 0]], "vocab": [[2, 16, 0]], "negative": [[2, -3, 0]], "after": [[2, 0, 5]]}
    for name, rows in bad.items():
        p = ok.copy()
        p[0] = rows[0]
        with pytest.raises(ValueError):
            t._check_prompt(p, 3, 3)
    with pytest.raises(ValueError, match="num_steps"):
        t._check_prompt(ok, 3, 2)
    with pytest.raises(ValueError, match="batch"):
        t._check_prompt(ok, 2, 3)


def test_transcribe_segments_sharded_rejects_prompts():
    from mt3_b200 import inference
    im = object.__new__(inference.InferenceModel)
    with pytest.raises(ValueError, match="prompts"):
        im.transcribe_segments_sharded(np.zeros((2, 8), np.float32), prompts=np.zeros((2, 3), np.int32))


# ------------------------------------------------------------------------------------------------
# the forced token pickers alone (libmt3kernels.so)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_tools", DK.os.path.join(DK.TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, F = C.c_void_p, C.c_int, C.c_float
    sig = {
        "kh_last_error": ([], C.c_char_p),
        "kh_argmax_step_forced": ([P, I, I, P, P, P, P, I, P, P, P, I, I, P, P, I, I, P, I], I),
        "kh_beam1_step_forced": ([P, I, I, P, P, P, P, I, P, P, P, P, P, F, I, P, P, I, I, P], I),
        "kh_beam1_finalize_scored": ([P, I, I, I, P, P, P, P, P], I),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    return lib


def _forced_case(V, B, L, seed):
    """crafted logits [B, L, V] and ragged prompts [B, L]: free rows, short and full-length prompts; forced positions
    hold NaN rows or EOS on top"""
    lg = _crafted(V, B, L, seed)
    rng = np.random.default_rng(seed + 1)
    plen = np.array([[0, 1, 3, L, L - 2, 5][b % 6] for b in range(B)])
    prompt = np.zeros((B, L), np.int32)
    for b in range(B):
        prompt[b, :plen[b]] = rng.integers(2, V, plen[b])
        for i in range(plen[b]):
            if (b + i) % 3 == 0:
                lg[b, i, (b * 7 + i) % V] = np.nan
            elif (b + i) % 3 == 1:
                lg[b, i, EOS] = np.float32(50.0)
    return lg, prompt, plen


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 257])
@pytest.mark.parametrize("scored", [False, True])
def test_forced_argmax_step_kernel(kh, V, scored):
    """argmax_step_kernel with plen: forced positions emit the prompt (NaN rows and EOS on top ignored), score 0, finish
    nothing and feed the prompt token to tok_cur / y_next; free positions match the restatement (tokens exactly, scores
    within lp_bar)."""
    import torch
    B, L, D = 24, 10, 64
    lg, prompt, plen = _forced_case(V, B, L, seed=V)
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = DK._pe_with_guard(rng, L + 1, D)
    d_emb, d_pe = _dev(emb), _dev(pe)
    d_tok = _dev(prompt.copy())
    d_pl = _dev(plen.astype(np.int32))
    d_st, d_cur, d_fin = _dev(np.array([0, 0, 0, 0], np.int32)), _dev(np.zeros(B, np.int32)), _dev(np.zeros(B, np.int32))
    d_ts = torch.full((B * L,), float("nan"), dtype=torch.float32, device=DEV)
    d_y = torch.zeros((B * D,), dtype=torch.float32, device=DEV)
    for i in range(L):
        _call(kh, "kh_argmax_step_forced", _p(_dev(lg[:, i].ravel())), V, B, _p(d_cur), _p(d_fin), _p(d_tok), _p(d_ts) if scored else None,
              L, _p(d_pl), None, _p(d_st), 1, 0, _p(d_emb), _p(d_pe), L + 1, D, _p(d_y), B)
        cur = _np(d_cur)
        np.testing.assert_array_equal(cur, np.where(i < plen, prompt[:, min(i, L - 1)], cur))
        _same_bits(f"step {i}: y_next", _np(d_y).reshape(B, D), emb[cur] + pe[i + 1])
    tok, ts = _np(d_tok).reshape(B, L), _np(d_ts).reshape(B, L)
    want, wts, _ = prompted_decode(_table_fn(lg), B, L, prompt, beam1=False)
    np.testing.assert_array_equal(tok, want)
    assert (_np(d_fin) == (want == EOS).any(1)).all()
    if scored:
        for b in range(B):
            for i in range(L):
                if i < plen[b] or (want[b, :i] == EOS).any():
                    assert ts[b, i] == 0.0, (b, i, ts[b, i])
                elif np.isnan(wts[b, i]):
                    assert np.isnan(ts[b, i])
                else:
                    assert abs(ts[b, i] - wts[b, i]) <= DS.lp_bar(lg[b, i], lg[b, i, want[b, i]]), (b, i)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 257])
def test_forced_beam1_step_kernel(kh, V):
    """beam1_step_kernel with plen and the scored finalize: tokens equal the prompted restatement, forced positions score
    0, no finish inside a prompt, live log-probability 0 where the prompt ends, scores within beam1_trace's bars."""
    import torch
    B, L, D = 24, 10, 32
    lg, prompt, plen = _forced_case(V, B, L, seed=V + 5)
    rng = np.random.default_rng(0)
    d_emb, d_pe = _dev(rng.standard_normal((V, D)).astype(np.float32)), _dev(DK._pe_with_guard(rng, L, D))
    d_tok, d_pl = _dev(prompt.copy()), _dev(plen.astype(np.int32))
    bf = np.zeros(2 * B, np.float32); bf[1::2] = -1.0e7
    d_bf, d_bi, d_fin = _dev(bf), _dev(np.zeros(B, np.int32)), _dev(np.zeros(B, np.int32))
    d_st, d_cur = _dev(np.array([0, 0, 0, 0], np.int32)), _dev(np.zeros(B, np.int32))
    d_ts = torch.full((B * L,), float("nan"), dtype=torch.float32, device=DEV)
    d_fe, d_sc = torch.zeros((B,), dtype=torch.float32, device=DEV), torch.zeros((B,), dtype=torch.float32, device=DEV)
    d_y = torch.zeros((B * D,), dtype=torch.float32, device=DEV)
    for i in range(L):
        _call(kh, "kh_beam1_step_forced", _p(_dev(lg[:, i].ravel())), V, B, _p(d_cur), _p(d_fin), _p(d_tok), _p(d_ts), L, _p(d_pl),
              _p(d_st), _p(d_bf), _p(d_fe), _p(d_bi), ALPHA, L, _p(d_emb), _p(d_pe), L, D, _p(d_y))
        live = _np(d_bf)[0::2]
        for b in range(B):
            if i < plen[b]:
                assert live[b] == 0.0 and _np(d_bi)[b] == 0, (b, i)
    _call(kh, "kh_beam1_finalize_scored", _p(d_tok), B, L, L, _p(d_bi), _p(d_ts), _p(d_bf), _p(d_fe), _p(d_sc))
    tok, ts, sc = _np(d_tok).reshape(B, L), _np(d_ts).reshape(B, L), _np(d_sc)
    want, wts, wsc = prompted_decode(_table_fn(lg), B, L, prompt, beam1=True)
    np.testing.assert_array_equal(tok, want)
    for b in range(B):
        assert (ts[b, :plen[b]] == 0).all()
        n = int(np.argmax(want[b] == EOS)) + 1 if (want[b] == EOS).any() else 0
        assert n == 0 or n > plen[b]
        bar = sum(DS.lp_bar(lg[b, i], lg[b, i, want[b, i]]) for i in range(L) if i >= plen[b])
        assert abs(sc[b] - wsc[b]) <= bar + 16 * DK.U * abs(wsc[b]), (b, sc[b], wsc[b])


# ------------------------------------------------------------------------------------------------
# the model against float64 (-m gpu)
# ------------------------------------------------------------------------------------------------
_CFG = {"mt3": (64, 1536), "ismir2021": (512, 1664)}
_L, _B = 40, 4


def _ocfg(config):
    return O.T5Config(vocab_size=_CFG[config][1], num_encoder_layers=2, num_decoder_layers=2)


def _params(config):
    import test_gpu_parity as GP
    return GP._eos_params(_ocfg(config), seed=9, boost=4.0)


def _model(config, gm, kv, params):
    import test_gpu_parity as GP
    from mt3_b200 import network
    T, V = _CFG[config]
    return network.Transformer(GP._mt3_cfg(vocab_size=V, num_encoder_layers=2, num_decoder_layers=2), params, device=DEV,
                               max_batch=_B, max_input_length=T, max_decode_length=_L, gemm_mode=gm, kv_format=kv)


def _prompts(V, lens, width, seed):
    rng = np.random.default_rng(seed)
    p = np.zeros((len(lens), width), np.int32)
    for b, n in enumerate(lens):
        p[b, :n] = rng.integers(2, V, n)
    return p


# ragged prompts: with an empty row (P = 0: every prompt forced in the loop), a short shared prefix and a long one
PROMPT_CASES = {"with_empty_row": (0, 1, 5, 12), "short_shared": (3, 4, 7, 12), "long_shared": (20, 24, 33, 36)}

_ORACLE = {}


def _oracle(config, case, beam1):
    key = (config, case, beam1)
    if key not in _ORACLE:
        import test_gpu_parity as GP
        T, V = _CFG[config]
        params = _params(config)
        ocfg = _ocfg(config)
        x = GP._inputs(_B, t=T, seed=50)
        enc64 = O.encode(params, ocfg, x, np.float64)
        p64 = O._cast(params, np.float64)
        lens = PROMPT_CASES[case]
        prompt = _prompts(V, lens, max(lens), seed=len(case))
        state = O.init_decode_state(ocfg, _B, _L, np.float64)
        logits = []

        def step(cur, i):
            logits.append(O.decode_step(p64, ocfg, enc64, cur, state))
            return logits[-1]
        tok, ts, sc = prompted_decode(step, _B, _L, prompt, beam1)
        l64 = np.stack(logits, 1)
        # the float32 oracle along the same fed tokens: its deviation sets the bar, as in test_decode_scores
        fed = np.concatenate([np.zeros((_B, 1), np.int64), tok[:, :-1]], 1)
        if beam1:
            fed = None
        if fed is not None:
            _, l32 = O.greedy_decode(params, ocfg, O.encode(params, ocfg, x, np.float32), _L, np.float32, stop_at_eos=False,
                                     return_logits=True, forced_tokens=fed)
            e_f32 = np.abs(l32 - l64).max() / np.abs(l64).max()
        else:
            e_f32 = _oracle(config, case, False)[5]
        _ORACLE[key] = (x, prompt, tok, ts, sc, e_f32, l64)
    return _ORACLE[key]


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(PROMPT_CASES))
@pytest.mark.parametrize("decode", ["greedy", "beam1"])
@pytest.mark.parametrize("mode", ["simt-f32", "tf32x3-f32", "tf32x3-f16", "tf32x3-p24"])
def test_prompted_generate_against_float64(mode, decode, case):
    """mt3_generate_prompted on a 2-layer mt3 model (EOS-boosted weights, T = 64, B = 4, 40 steps) against the prompted
    restatement on the float64 oracle: tokens equal over the prefix where the float64 top-2 margins exceed twice the
    logit bar (beam1 in SIMT: every token), token scores within max(4 e_f32, 2e-5) of max |logit| there with fp32 and
    24-bit rows (fp16 rows: reported), forced positions exactly 0; graph replay equals plain launches bit for bit.  The
    shared prefix is 0, 3 (stepped in the loop) and 20 (prefilled)."""
    import torch
    from mt3_b200 import _lib
    gm, kv = mode.split("-")
    gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3}[gm]
    kv = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[kv]
    beam1 = decode == "beam1"
    x, prompt, want, wts, wsc, e_f32, l64 = _oracle("mt3", case, beam1)
    m = _model("mt3", gm, kv, _params("mt3"))
    xg = torch.from_numpy(x).to(DEV)
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, num_steps=_L, stop_at_eos=False, decode=decode, return_scores=True,
                                                         prompt=prompt))
    assert m.last_steps_run == _L
    plain = [t.cpu().numpy() for t in m.generate(xg, num_steps=_L, stop_at_eos=False, decode=decode, return_scores=True,
                                                 prompt=prompt, use_graph=False)]
    np.testing.assert_array_equal(plain[0], tok)
    _same_bits(f"{mode} {decode} {case}: token scores, graph vs plain", plain[1], ts)
    _same_bits(f"{mode} {decode} {case}: scores, graph vs plain", plain[2], sc)
    plen = prompt_lengths(prompt)
    scale = np.abs(l64).max()
    bar = max(4 * e_f32, 2e-5) * scale
    for b in range(_B):
        np.testing.assert_array_equal(tok[b, :plen[b]], prompt[b, :plen[b]])
        assert (ts[b, :plen[b]] == 0).all()
    srt = np.sort(l64, -1)
    forced = np.arange(_L)[None] < plen[:, None]
    safe = np.cumprod(forced | (srt[..., -1] - srt[..., -2] > 2 * bar), 1).astype(bool)
    if beam1 and mode == "simt-f32":
        safe[:] = True
    np.testing.assert_array_equal(tok[safe], want[safe])
    same = safe & ~forced & (np.cumprod(tok == want, 1) > 0)
    d = np.abs(ts - wts)[same]
    print(f"{mode} {decode} {case}: {int(safe.sum())} of {safe.size} positions safe; worst |dscore| "
          f"{d.max() if d.size else 0:.2e}, bar {bar:.2e}")
    assert safe[:, :10].all() and same.sum() >= _B * 4
    if kv != _lib.KV_F16:                      # fp16 rows are outside the logit bar unprompted too (DESIGN.md section 4)
        assert (d <= bar).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["with_empty_row", "long_shared"])
def test_prompted_generate_ismir2021(case):
    """The same check on the ismir2021 shapes (T = 512, V = 1664), TF32X3 with 24-bit rows, greedy."""
    import torch
    from mt3_b200 import _lib
    x, prompt, want, wts, wsc, e_f32, l64 = _oracle("ismir2021", case, False)
    m = _model("ismir2021", _lib.GEMM_TF32X3, _lib.KV_P24, _params("ismir2021"))
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(torch.from_numpy(x).to(DEV), num_steps=_L, stop_at_eos=False,
                                                         return_scores=True, prompt=prompt))
    plen = prompt_lengths(prompt)
    bar = max(4 * e_f32, 2e-5) * np.abs(l64).max()
    srt = np.sort(l64, -1)
    forced = np.arange(_L)[None] < plen[:, None]
    safe = np.cumprod(forced | (srt[..., -1] - srt[..., -2] > 2 * bar), 1).astype(bool)
    np.testing.assert_array_equal(tok[safe], want[safe])
    same = safe & ~forced
    assert safe[:, :10].all() and (np.abs(ts - wts)[same] <= bar).all()
    assert (ts[forced] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["short_shared", "long_shared"])
def test_prompted_generate_against_step_path(case):
    """A host loop of init_cache + decode(decode=True) feeding BOS, then the prompted run's own tokens: its log-softmax at
    those tokens equals the prompted run's token scores at the free positions within the teacher-forced-vs-step bound
    2 max(4 e_f32, 2e-5) of max |logit| (TF32X3, fp32 rows, greedy)."""
    import torch
    from mt3_b200 import _lib
    x, prompt, _, _, _, e_f32, l64 = _oracle("mt3", case, False)
    m = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_F32, _params("mt3"))
    xg = torch.from_numpy(x).to(DEV)
    tok, ts, _ = (t.cpu().numpy() for t in m.generate(xg, num_steps=_L, stop_at_eos=False, return_scores=True, prompt=prompt))
    enc = m.encode(xg)
    m.init_cache(enc)
    fed = np.concatenate([np.zeros((_B, 1), np.int32), tok[:, :-1]], 1)
    steps = [m.decode(enc, None, torch.from_numpy(fed[:, i:i + 1]).to(DEV)).cpu().numpy()[:, 0] for i in range(_L)]
    ls = np.stack(steps, 1)
    lp = np.take_along_axis(DS.log_softmax64(ls), tok[..., None].astype(np.int64), -1)[..., 0]
    plen = prompt_lengths(prompt)
    free = np.arange(_L)[None] >= plen[:, None]
    alive = np.cumsum(tok == EOS, 1) - (tok == EOS) == 0
    keep = free & alive
    bar = 2 * max(4 * e_f32, 2e-5) * np.abs(ls).max()
    d = np.abs(ts - lp)[keep]
    print(f"{case}: prompted loop vs step path worst |dscore| {d.max():.2e}, bar {bar:.2e}, {int(keep.sum())} positions")
    assert keep.sum() > 0 and (d <= bar).all()


@pytest.mark.gpu
def test_error_codes_and_isolation():
    """mt3_generate_prompted: each bad prompt is MT3_ERR_BAD_ARG, a short or misaligned workspace and a NULL workspace with
    prompt_len >= 1 are MT3_ERR_WORKSPACE, prompt_len > num_steps is MT3_ERR_BAD_ARG; after them an unprompted generate
    is bit-identical to one on a fresh model."""
    import torch
    from mt3_b200 import _lib
    x, _, _, _, _, _, _ = _oracle("mt3", "short_shared", False)
    params = _params("mt3")
    m = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24, params)
    xg = torch.from_numpy(x).to(DEV)
    m.generate(xg, num_steps=1)
    lib, V = m._lib, 1536
    pl = 6
    nbytes = int(lib.mt3_teacher_forced_workspace_bytes(m._h, _B, 64, pl))
    ws = torch.empty(nbytes + 512, dtype=torch.uint8, device=DEV)
    out = torch.empty((_B, _L), dtype=torch.int32, device=DEV)
    ran = C.c_int32(0)

    def call(prompt, plen=pl, ws_ptr=ws.data_ptr(), ws_bytes=nbytes, steps=_L):
        d = torch.from_numpy(np.ascontiguousarray(prompt, np.int32)).to(DEV)
        r = lib.mt3_generate_prompted(m._h, xg.data_ptr(), steps, 0, d.data_ptr(), plen, out.data_ptr(), None, None, C.byref(ran),
                                      ws_ptr, ws_bytes, m._stream())
        torch.cuda.synchronize()
        return r
    good = _prompts(V, (2, 3, 6, 4), pl, seed=1)
    assert call(good) == 0
    for name, (b, j, v) in {"EOS": (1, 1, EOS), "vocab": (2, 0, V), "negative": (0, 1, -2), "after_pad": (0, 4, 9),
                            "unk_2_is_fine_but_1": (3, 0, 1)}.items():
        p = good.copy()
        p[b, j] = v
        assert call(p) == -1, name
    assert call(good, ws_bytes=nbytes - 256) == -4
    assert call(good, ws_ptr=ws.data_ptr() + 4) == -4
    assert call(good, ws_ptr=None, ws_bytes=0) == -4
    assert call(good, steps=pl - 1) == -1
    got = [t.cpu().numpy() for t in m.generate(xg, num_steps=_L, stop_at_eos=False, return_scores=True)]
    fresh = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24, params)
    want = [t.cpu().numpy() for t in fresh.generate(xg, num_steps=_L, stop_at_eos=False, return_scores=True)]
    np.testing.assert_array_equal(got[0], want[0])
    _same_bits("token scores after failed prompted calls", got[1], want[1])
    _same_bits("scores after failed prompted calls", got[2], want[2])


# ------------------------------------------------------------------------------------------------
# bench.py's configuration
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bench_configuration(bench_inputs_prompted):
    """mt3, B = 64, 1024 steps, TF32X3, 24-bit rows, graphs.  An empty prompt and prompt_len = 0 give tokens and scores
    bit-identical to generate, greedy and beam1.  A greedy run g prompted with g[:, :P], P in {1, 128, 512}, reproduces g's
    continuation; a row may differ only where the teacher-forced logits of g have a top-2 gap below 2e-4 of the row's
    max |logit| at the first differing position (the prefilled K/V come from the pass's GEMMs, not the step's)."""
    import torch
    from mt3_b200 import _lib, inference
    x = bench_inputs_prompted
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=64, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format=_lib.KV_P24)
    m = im.model
    for decode in ("greedy", "beam1"):
        want = [t.cpu().numpy() for t in m.generate(x, stop_at_eos=False, decode=decode, return_scores=True)]
        for prompt in (np.zeros((64, 0), np.int32), np.zeros((64, 5), np.int32)):
            got = [t.cpu().numpy() for t in m.generate(x, stop_at_eos=False, decode=decode, return_scores=True, prompt=prompt)]
            np.testing.assert_array_equal(got[0], want[0])
            _same_bits(f"{decode} empty prompt: token scores", got[1], want[1])
            _same_bits(f"{decode} empty prompt: scores", got[2], want[2])
    g = m.generate(x, stop_at_eos=False).cpu().numpy()
    din = np.concatenate([np.zeros((64, 1), np.int32), g[:, :-1]], 1)
    tgt = np.where(g == 0, 7, g)                  # every key visible, as the loop sees it
    lg = m.decode(m.encode(x), None, torch.from_numpy(din).to(DEV), torch.from_numpy(tgt).to(DEV), decode=False).cpu().numpy()
    srt = np.sort(lg, -1)
    gap = (srt[..., -1] - srt[..., -2]) / np.abs(lg).max(-1)
    for P in (1, 128, 512):
        prompt = g[:, :P].copy()
        cut = np.cumsum((prompt == EOS) | (prompt == PAD), 1) > 0   # a row that ended inside P is prompted up to its EOS
        prompt[cut] = 0
        got = m.generate(x, stop_at_eos=False, prompt=prompt).cpu().numpy()
        np.testing.assert_array_equal(got[:, :P][~cut], g[:, :P][~cut])
        diff = (got != g).any(1)
        for b in np.nonzero(diff)[0]:
            i = int(np.argmax(got[b] != g[b]))
            assert gap[b, i] < 2e-4, (P, b, i, gap[b, i])
        print(f"P = {P}: {int(diff.sum())} of 64 rows differ from the unprompted run's continuation")
    del im, m
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def bench_inputs_prompted():
    import torch
    from mt3_b200 import spectrograms
    audio = np.stack([O.sine_mix(256 * 128, seed=4000 + i) for i in range(64)])
    return spectrograms.compute_spectrogram(torch.from_numpy(audio).to(DEV), spectrograms.SpectrogramConfig())


# ------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------
def tie_sections(targets, tie_id):
    """The tie section of each segment's target row (through the tie token), as an int32 [S, P] prompt"""
    lens = [int(np.argmax(row == tie_id)) + 1 if (row == tie_id).any() else 0 for row in targets]
    out = np.zeros((len(targets), max(1, max(lens))), np.int32)
    for i, n in enumerate(lens):
        out[i, :n] = targets[i, :n]
    return out


@pytest.mark.gpu
def test_transcribe_segments_with_tie_prompts():
    """InferenceModel.transcribe_segments(prompts=...) with the tie sections of segment_score_targets: every output row
    starts with its prompt, the rest decodes, and the raw rows decode to a NoteSequence."""
    from mt3_b200 import event_codec, inference, note_decoding as nd
    import test_teacher_forced as TF
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=2)
    audio = O.sine_mix(5 * 16000, 77).astype(np.float32)
    frames, times = im._audio_to_frames(audio)
    ds = im.preprocess(im.audio_to_dataset(audio))
    ns = TF._dense_note_sequence()
    tg = inference.segment_score_targets(ns, im.codec, im.vocabulary, times, im.inputs_length, im.encoding_spec, 1024)
    tie_id = im.codec.encode_event(event_codec.Event('tie', 0)) + 3
    prompts = tie_sections(tg['decoder_target_tokens'], tie_id)
    assert (prompts[:, 0] != 0).sum() >= 2
    hop = im.spectrogram_config.hop_width
    segs = np.zeros((len(ds), im.inputs_length * hop), np.float32)
    for i, ex in enumerate(ds):
        flat = np.asarray(ex['inputs'], np.float32).reshape(-1)
        segs[i, :flat.size] = flat
    raw = im.transcribe_segments(segs, num_steps=96, decoded=False, prompts=prompts)
    for i, p in enumerate(prompts):
        n = int(prompt_lengths(p[None])[0])
        np.testing.assert_array_equal(raw[i, :n], p[:n])
    decoded = im.transcribe_segments(segs, num_steps=96, prompts=prompts)
    preds = [{'raw_inputs': [], 'start_time': float(times[0]) + i * 2.048, 'est_tokens': decoded[i]} for i in range(len(ds))]
    res = nd.event_predictions_to_ns(preds, codec=im.codec, encoding_spec=im.encoding_spec)
    assert 'est_ns' in res
