"""Decode scores (mt3_generate_scored, Transformer.generate(return_scores=True), predict_batch_with_aux's aux['scores'],
InferenceModel.transcribe_segments(return_scores=True)): the log-probability of every emitted token and T5X's sequence
score, from the greedy and the beam-size-1 loops.

CPU: numpy restatements of the scored greedy and beam1 traces, tied to oracle/beam_search.py on the crafted tables of
test_beam1.py and test_decode_loop_kernels.py; the wrapper's aux dict and return_all_decodes shapes with stand-in modules.
GPU: the scored token pickers alone against float64 and against token_score_kernel bit for bit, with the unscored launch's
tokens and state unchanged; the loop against the teacher-forced pass and against the float64 oracle; bit identity of
tokens and scores at bench.py's configuration across scoring, graphs and the early stop; the InferenceModel surface.
"""
import math

import numpy as np
import pytest

import test_beam1 as TB
import test_decode_loop_kernels as DK
from oracle import beam_search as BS
from oracle import mt3_oracle as O

DEV = "cuda:0"
U = DK.U
EOS, PAD = 1, 0
ALPHA = DK.ALPHA


# ------------------------------------------------------------------------------------------------
# numpy restatements
# ------------------------------------------------------------------------------------------------
def log_softmax64(x):
    """float64 log-softmax of float32 rows (NaN anywhere in a row: NaN for the whole row)"""
    with np.errstate(invalid="ignore", over="ignore"):
        return BS.log_softmax(np.asarray(x, np.float64))


def lp_bar(row, v):
    """fp32 error bar of one kernel log-probability v - lse (block_logsumexp / beam1_step_kernel), beam1_trace's bound"""
    l = np.asarray(row, np.float64)
    V = l.size
    gmx = l.max()
    x = l - gmx
    e = np.exp(x)
    tot = e.sum()
    lse = gmx + math.log(tot)
    pos = e > 0                      # -inf entries add nothing (and 0 * inf would be NaN)
    ep = float((e[pos] * np.abs(x[pos])).sum() / tot)
    return U * (4 + math.ceil(V / 256) + 13 + ep + 2 * abs(math.log(tot)) + abs(lse) + abs(float(v) - lse))


def greedy_scored_trace(lg, L):
    """The scored greedy loop for one element from fp32 logits lg [>= L, V]: tokens (PAD after the first EOS), token scores
    in float64 (0 after EOS) and their sum."""
    toks, ts = np.zeros(L, np.int32), np.zeros(L)
    done = False
    for i in range(L):
        if done:
            continue
        t = int(DK.argmax_ref(lg[i][None])[0])
        toks[i], ts[i] = t, log_softmax64(lg[i])[t]
        done = t == EOS
    return dict(tokens=toks, token_scores=ts, score=ts.sum())


def beam1_scored_trace(lg, L):
    """beam1_trace (tokens, finish length, score) with the winning hypothesis's token scores in float64: the live prefix's
    log-probabilities, the EOS log-probability at position n - 1 and 0 from n on; the live prefix's when nothing
    finished."""
    t = DK.beam1_trace(lg, L)
    n = t["fin_len"]
    ts = np.zeros(L)
    for i in range(n - 1 if n else t["calls"]):
        ts[i] = log_softmax64(lg[i])[t["tokens"][i]]
    if n:
        ts[n - 1] = log_softmax64(lg[n - 1])[EOS]
    return dict(t, token_scores=ts)


def _test_beam1_tables():
    """test_beam1.py's crafted step tables, [L, V] float64 log-probabilities"""
    p = TB._p
    tables = {
        "decisive": [p(a=0.97, eos=0.001), p(b=0.97, eos=0.001), p(eos=0.97, c=0.01), p(c=0.5, eos=0.3)],
        "runner_up_eos_wins": [p(a=0.9, eos=0.01), p(a=0.6, eos=0.35), p(b=0.5, eos=0.02), p(eos=0.9, c=0.05), p(eos=0.9, c=0.05)],
        "first_eos_loses": [p(a=0.9, eos=0.01), p(eos=0.5, a=0.45), p(b=0.99, eos=0.002), p(c=0.99, eos=0.002),
                            p(eos=0.99, c=0.002), p(eos=0.99, c=0.002)],
        "never": [p(a=0.7, eos=0.0001)] * 3,
    }
    return {k: np.log(np.stack([v[min(i, len(v) - 1)] for i in range(TB.L)])) for k, v in tables.items()}


def test_beam1_scored_trace_matches_beam_search():
    """On test_beam1.py's tables and on the kernel tests' crafted streams: the restated tokens and score are
    BS.beam_search's, and score == sum(token_scores[:n]) / bp(n) for a finished hypothesis, the plain sum otherwise."""
    cases = {f"test_beam1/{k}": (v, TB.L) for k, v in _test_beam1_tables().items()}
    for V in (1536, 257, 33):
        cases.update({f"V={V}/{k}": (v, DK.BEAM_L) for k, v in DK.beam_scenarios(V).items()})
    for name, (lg, L) in cases.items():
        t = beam1_scored_trace(lg, L)
        want, score = BS.beam_search(lambda p, s: lg[None, None, s], 1, L)
        np.testing.assert_array_equal(t["tokens"], want[0], err_msg=name)
        assert abs(t["score"] - score[0]) <= 1e-12 * max(1.0, abs(score[0])), name
        n = t["fin_len"]
        total = t["token_scores"][:n].sum() / BS.brevity_penalty(ALPHA, n) if n else t["token_scores"].sum()
        assert abs(total - score[0]) <= 1e-12 * max(1.0, abs(score[0])), (name, total, score[0])
        assert (t["token_scores"][max(n, t["calls"]):] == 0).all(), name


def test_greedy_scored_trace_matches_greedy():
    """The scored greedy restatement emits BS.greedy's tokens; its scores are log_softmax at them, 0 after EOS."""
    for V in (1536, 257):
        for name, lg in DK.beam_scenarios(V).items():
            t = greedy_scored_trace(lg, DK.BEAM_L)
            want = BS.greedy(lambda p, s: lg[None, None, s], 1, DK.BEAM_L)[0]
            np.testing.assert_array_equal(t["tokens"], want, err_msg=name)
            if (want == EOS).any():
                e = int(np.argmax(want == EOS))
                assert (t["token_scores"][e + 1:] == 0).all() and t["token_scores"][e] < 0, name


# ------------------------------------------------------------------------------------------------
# predict_batch_with_aux (CPU, stand-in modules)
# ------------------------------------------------------------------------------------------------
class _ScoringModule:
    """network.Transformer's generate contract with return_scores"""

    def __init__(self, L=8):
        self.calls, self.L = [], L

    def generate(self, x, stop_at_eos=True, decode='greedy', return_scores=False):
        self.calls.append((tuple(x.shape), stop_at_eos, decode, return_scores))
        b = x.shape[0]
        toks = np.arange(b * self.L, dtype=np.int32).reshape(b, self.L)
        if not return_scores:
            return toks
        return toks, -np.ones((b, self.L), np.float32), -np.arange(1, b + 1, dtype=np.float32)


class _PlainModule:
    def generate(self, x, stop_at_eos=True, decode='greedy'):
        return np.zeros((x.shape[0], 8), np.int32)


def test_predict_batch_with_aux_scores_and_all_decodes():
    """aux['scores'] float32 [B] from a module that can score, {} from one that cannot; return_all_decodes=True gives
    T5X's shapes (tokens [B, 1, L], scores [B, 1]); predict_batch asks for no scores."""
    from mt3_b200 import models
    batch = {'encoder_input_tokens': np.zeros((3, 5, 4), np.float32)}
    mod = _ScoringModule()
    m = models.ContinuousInputsEncoderDecoderModel(mod, input_depth=4)
    toks, aux = m.predict_batch_with_aux(None, batch)
    assert toks.shape == (3, 8) and set(aux) == {'scores'}
    assert aux['scores'].shape == (3,) and aux['scores'].dtype == np.float32
    np.testing.assert_array_equal(aux['scores'], [-1, -2, -3])
    assert mod.calls[-1] == ((3, 5, 4), True, 'beam1', True)
    toks_all, aux_all = m.predict_batch_with_aux(None, batch, return_all_decodes=True)
    assert toks_all.shape == (3, 1, 8) and aux_all['scores'].shape == (3, 1)
    np.testing.assert_array_equal(toks_all[:, 0], toks)
    np.testing.assert_array_equal(m.predict_batch(None, batch), toks)
    assert mod.calls[-1][3] is False
    plain = models.ContinuousInputsEncoderDecoderModel(_PlainModule(), input_depth=4, decode_fn='greedy')
    toks, aux = plain.predict_batch_with_aux(None, batch)
    assert aux == {} and toks.shape == (3, 8)
    toks, aux = plain.predict_batch_with_aux(None, batch, return_all_decodes=True)
    assert aux == {} and toks.shape == (3, 1, 8)
    with pytest.raises(ValueError):
        m.predict_batch_with_aux(None, batch, num_decodes=2)


@pytest.mark.parametrize("rank,shard", [(3, 0), (0, 2), (2, 1)])
def test_transcribe_segments_sharded_scores_gather(monkeypatch, rank, shard):
    """transcribe_segments_sharded(return_scores=True) on rank `rank` of 4 with S = 5 segments (shards of 2, 2, 1 and none):
    every rank, the one with an empty shard included, hands the all-gather tokens [n, 1024] int32, token scores
    [n, 1024] float32 and scores [n, 1] float32, and returns (tokens [S, 1024], token_scores [S, 1024], scores [S])."""
    import torch
    from mt3_b200 import distributed, inference
    S, L = 5, 1024
    im = object.__new__(inference.InferenceModel)
    im.outputs_length, im.device = L, torch.device("cpu")
    monkeypatch.setattr(distributed, "world", lambda: (rank, 4))
    handed = []

    def gather(local, num_segments):
        handed.append((tuple(local.shape), local.dtype))
        fill = torch.arange(num_segments * local.shape[1], dtype=torch.float64).reshape(num_segments, -1)
        return fill.to(local.dtype)

    def transcribe(a, n_valid_frames=None, **kw):
        assert kw["return_scores"] and a.shape[0] == shard and len(n_valid_frames) == shard
        return np.ones((shard, L), np.int32), -np.ones((shard, L), np.float32), -np.ones((shard,), np.float32)

    monkeypatch.setattr(distributed, "gather_tokens", gather)
    monkeypatch.setattr(im, "transcribe_segments", transcribe)
    toks, ts, sc = im.transcribe_segments_sharded(np.zeros((S, 8), np.float32), n_valid_frames=np.arange(S), return_scores=True)
    assert handed == [((shard, L), torch.int32), ((shard, L), torch.float32), ((shard, 1), torch.float32)]
    assert toks.shape == (S, L) and toks.dtype == np.int32
    assert ts.shape == (S, L) and ts.dtype == np.float32
    assert sc.shape == (S,) and sc.dtype == np.float32
    np.testing.assert_array_equal(sc, np.arange(S))


# ------------------------------------------------------------------------------------------------
# the kernels alone (libmt3kernels.so)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    import ctypes as C
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
        "kh_argmax_step": ([P, I, I, P, P, P, I, P, P, I, I, P, P, I, I, P, I], I),
        "kh_argmax_step_scored": ([P, I, I, P, P, P, P, I, P, P, I, I, P, P, I, I, P, I], I),
        "kh_beam1_step": ([P, I, I, P, P, P, I, P, P, P, F, I, P, P, I, I, P], I),
        "kh_beam1_step_scored": ([P, I, I, P, P, P, P, I, P, P, P, P, F, I, P, P, I, I, P], I),
        "kh_beam1_finalize": ([P, I, I, I, P], I),
        "kh_beam1_finalize_scored": ([P, I, I, I, P, P, P, P, P], I),
        "kh_seq_score": ([P, I, I, P], I),
        "kh_token_score": ([P, I, I, I, I, I, P, P, P, P], I),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    return lib


_call, _p, _dev, _np, _same_bits = DK._call, DK._p, DK._dev, DK._np, DK._same_bits


def _greedy_pair(kh, lg_steps, V, B, D=64, split=False):
    """Runs the same logits through the unscored and the scored argmax_step_kernel (fresh state each); returns per step
    the (tokens_out, finished, state, tok_cur, y_next) of both and the scored token_scores buffer [B + 1, out_ld]."""
    import torch
    steps = len(lg_steps)
    rng = np.random.default_rng(V + B)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = DK._pe_with_guard(rng, steps + 1, D)
    out_ld = steps + 3
    d_emb, d_pe = _dev(emb), _dev(pe)
    runs = []
    for scored in (False, True):
        d_lg = torch.full(((B + 1) * V,), float("nan"), dtype=torch.float32, device=DEV)
        d_st = _dev(np.array([0, 0, 0, DK.SENT], np.int32))
        d_cur = _dev(np.full(B + 1, DK.SENT, np.int32))
        fin = np.full(B + 1, DK.SENT, np.int32); fin[:B] = 0
        d_fin = _dev(fin)
        d_tok = _dev(np.full((B + 1, out_ld), DK.SENT, np.int32))
        d_ts = torch.full(((B + 1) * out_ld,), float("nan"), dtype=torch.float32, device=DEV)
        d_y = torch.full(((B + 1) * D,), DK.YSENT, dtype=torch.float32, device=DEV)
        trace = []
        for step in range(steps):
            d_lg[:B * V] = _dev(lg_steps[step].ravel())
            parts = [(0, B)] if not split else [(0, B // 3), (B // 3, B)]
            for a, b in parts:
                head = (_p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok))
                tail = (out_ld, None, _p(d_st), 1, a, _p(d_emb), _p(d_pe), steps + 1, D, _p(d_y), b - a)
                if scored:
                    _call(kh, "kh_argmax_step_scored", *head, _p(d_ts), *tail)
                else:
                    _call(kh, "kh_argmax_step", *head, *tail)
            trace.append(tuple(_np(t).copy() for t in (d_tok, d_fin, d_st, d_cur, d_y)))
        runs.append((trace, _np(d_ts).reshape(B + 1, out_ld)))
    return runs[0][0], runs[1][0], runs[1][1]


def _stream(V, B, steps, seed):
    """[steps, B, V] logits: normal rows, test_decode_loop_kernels' crafted rows (ties, NaN, -inf, signed zeros,
    denormals) and EOS wins that finish the rows between steps 3 and 9"""
    rng = np.random.default_rng(seed)
    crafted = DK._crafted_rows(V)
    x = (rng.standard_normal((steps, B, V)) * 4).astype(np.float32)
    for s in range(steps):
        for b in range(B):
            k = (b * 5 + s) % (len(crafted) + 4)
            if k < len(crafted):
                x[s, b] = crafted[k][0]
            if s >= 3 and (b + s) % 7 == 0:
                x[s, b, EOS] = np.float32(30.0)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664, 1517])
@pytest.mark.parametrize("split", [False, True])
def test_argmax_step_scored_kernel(kh, V, split):
    """Scored argmax_step_kernel: tokens, finished, state, tok_cur and y_next bit-equal the unscored launch at every
    step; token scores against float64 log_softmax at the emitted id within lp_bar, exactly 0 for a row that had
    finished, NaN for a row with a NaN; columns past the steps and the guard row untouched."""
    B, steps = 40, 12
    lg = _stream(V, B, steps, seed=V)
    plain, scored, ts = _greedy_pair(kh, lg, V, B, split=split)
    for step, (a, b) in enumerate(zip(plain, scored)):
        for name, x, y in zip(("tokens_out", "finished", "state", "tok_cur"), a[:4], b[:4]):
            np.testing.assert_array_equal(y, x, err_msg=f"V={V} step {step}: {name}")
        _same_bits(f"V={V} step {step}: y_next", b[4], a[4])
    tok = plain[-1][0]
    assert np.isnan(ts[B]).all() and np.isnan(ts[:B, steps:]).all()
    done = np.zeros(B, bool)
    worst = 0.0
    n_nan = n_fin = 0
    for s in range(steps):
        for b in range(B):
            got = ts[b, s]
            if done[b]:
                assert tok[b, s] == PAD and got == 0.0 and not np.signbit(got), (s, b, got)
                n_fin += 1
                continue
            t = tok[b, s]
            assert t == DK.argmax_ref(lg[s, b][None])[0]
            want = log_softmax64(lg[s, b])[t]
            if np.isnan(want):
                assert np.isnan(got), (s, b, got)
                n_nan += 1
            else:
                bar = lp_bar(lg[s, b], lg[s, b, t])
                assert abs(got - want) <= bar, (V, s, b, got, want, bar)
                worst = max(worst, abs(got - want) / bar)
            done[b] |= t == EOS
    assert n_nan > 0 and n_fin > 0
    print(f"scored argmax V={V}: worst err/bar {worst:.3f}, {n_nan} NaN rows, {n_fin} finished-row zeros")


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1664, 1517])
def test_argmax_scores_bit_equal_token_score_kernel(kh, V):
    """One logits row gives the same log-probability bits in the decode loop and in the teacher-forced pass:
    argmax_step_kernel's token score == token_score_kernel's at target = the argmax (weight 1), NaN rows included."""
    import torch
    B = 48
    lg = _stream(V, B, 1, seed=V + 1)
    _, scored, ts = _greedy_pair(kh, lg, V, B)
    tok = scored[0][0][:B, 0]
    d_x, d_t, d_w = _dev(lg[0]), _dev(tok.astype(np.int32)), _dev(np.ones(B, np.int32))
    d_s = torch.full((B,), float("nan"), dtype=torch.float32, device=DEV)
    _call(kh, "kh_token_score", _p(d_x), V, 0, B, 1, 1, _p(d_t), _p(d_w), _p(d_s), None)
    _same_bits(f"V={V}: argmax token scores vs token_score_kernel", ts[:B, 0], _np(d_s))


def _run_beam_scored(kh, lg, L, scored, D=32):
    """beam1_step_kernel for L steps and the finalize, unscored or scored; returns tokens, beam_f, beam_i, token scores,
    scores, fin_lp_eos (the last three None unscored)"""
    import torch
    B, _, V = lg.shape
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    d_emb, d_pe = _dev(emb), _dev(DK._pe_with_guard(rng, L, D))
    d_lg = torch.full(((B + 1) * V,), float("nan"), dtype=torch.float32, device=DEV)
    bf = np.full(2 * B + 2, np.nan, np.float32); bf[0:2 * B:2], bf[1:2 * B:2] = 0.0, -1.0e7
    bi = np.full(B + 1, DK.SENT, np.int32); bi[:B] = 0
    fin = np.full(B + 1, DK.SENT, np.int32); fin[:B] = 0
    d_st, d_bf, d_bi, d_fin = _dev(np.array([0, 0, 0, DK.SENT], np.int32)), _dev(bf), _dev(bi), _dev(fin)
    d_cur, d_tok = _dev(np.full(B + 1, DK.SENT, np.int32)), _dev(np.full((B + 1) * L, DK.SENT, np.int32))
    d_y = torch.full(((B + 1) * D,), DK.YSENT, dtype=torch.float32, device=DEV)
    d_ts = torch.full(((B + 1) * L,), float("nan"), dtype=torch.float32, device=DEV)
    d_fe = torch.full((B + 1,), float("nan"), dtype=torch.float32, device=DEV)
    d_sc = torch.full((B + 1,), float("nan"), dtype=torch.float32, device=DEV)
    for step in range(L):
        d_lg[:B * V] = _dev(lg[:, step].ravel())
        head = (_p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok))
        tail = (_p(d_emb), _p(d_pe), L, D, _p(d_y))
        if scored:
            _call(kh, "kh_beam1_step_scored", *head, _p(d_ts), L, _p(d_st), _p(d_bf), _p(d_fe), _p(d_bi), ALPHA, L, *tail)
        else:
            _call(kh, "kh_beam1_step", *head, L, _p(d_st), _p(d_bf), _p(d_bi), ALPHA, L, *tail)
    if scored:
        _call(kh, "kh_beam1_finalize_scored", _p(d_tok), B, L, L, _p(d_bi), _p(d_ts), _p(d_bf), _p(d_fe), _p(d_sc))
    else:
        _call(kh, "kh_beam1_finalize", _p(d_tok), B, L, L, _p(d_bi))
    tok = _np(d_tok).reshape(B + 1, L)
    ts, sc, fe = _np(d_ts).reshape(B + 1, L), _np(d_sc), _np(d_fe)
    assert (tok[B] == DK.SENT).all() and np.isnan(_np(d_bf)[2 * B:]).all()
    if scored:
        assert np.isnan(ts[B]).all() and np.isnan(sc[B]) and np.isnan(fe[B])
    return tok[:B], _np(d_bf)[:2 * B].reshape(B, 2), _np(d_bi)[:B], (ts[:B], sc[:B], fe[:B]) if scored else None


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1516, 257, 33])
def test_beam1_scored_kernels(kh, V):
    """Scored beam1_step_kernel + beam1_finalize_kernel on every crafted stream as one batch: tokens, beam_f and beam_i
    bit-equal the unscored launches; scores == beam_f's finished score (or its live log-probability when nothing
    finished) exactly; token scores against beam1_scored_trace within lp_bar per token (the steps the restatement runs;
    the kernel keeps extending the live prefix after the search settled, which the finalize cuts); the score against the
    restatement within beam1_trace's bar."""
    sc = DK.beam_scenarios(V)
    names = list(sc)
    lg = np.stack([sc[n] for n in names])
    L = DK.BEAM_L
    tok0, bf0, bi0, _ = _run_beam_scored(kh, lg, L, False)
    tok, bf, bi, (ts, score, _) = _run_beam_scored(kh, lg, L, True)
    np.testing.assert_array_equal(tok, tok0)
    _same_bits(f"V={V} beam_f", bf, bf0)
    np.testing.assert_array_equal(bi, bi0)
    _same_bits(f"V={V} scores", score, np.where(bi > 0, bf[:, 1], bf[:, 0]))
    for b, n in enumerate(names):
        t = beam1_scored_trace(sc[n], L)
        np.testing.assert_array_equal(tok[b], t["tokens"], err_msg=n)
        fin_len = t["fin_len"]
        upto = fin_len if fin_len else L
        for i in range(upto):
            row = sc[n][i]
            v = row[EOS] if fin_len and i == fin_len - 1 else row[t["tokens"][i]]
            assert abs(ts[b, i] - t["token_scores"][i]) <= lp_bar(row, v), (n, i, ts[b, i], t["token_scores"][i])
        assert (ts[b, upto:] == 0).all(), n
        bar = t["steps"][-1][3] if fin_len else t["steps"][-1][1]
        assert abs(score[b] - t["score"]) <= bar, (n, score[b], t["score"], bar)


@pytest.mark.gpu
def test_seq_score_kernel(kh):
    """seq_score_kernel: the row sum against float64 within (L/128 + 7) roundings of sum |x|, rows of zeros give +0,
    NaN carries, rows past B untouched."""
    import torch
    B, L = 9, 1024
    rng = np.random.default_rng(3)
    x = -np.abs(rng.standard_normal((B, L)) * 3).astype(np.float32)
    x[:, 700:] = 0.0
    x[4] = 0.0
    x[6, 17] = np.nan
    d_s = torch.full((B + 1,), float("nan"), dtype=torch.float32, device=DEV)
    _call(kh, "kh_seq_score", _p(_dev(x)), B, L, _p(d_s))
    got = _np(d_s)
    assert np.isnan(got[B]) and np.isnan(got[6]) and got[4] == 0.0 and not np.signbit(got[4])
    ok = [b for b in range(B) if b != 6]
    want = x[ok].astype(np.float64).sum(1)
    bar = (L / 128 + 7) * U * np.abs(x[ok]).astype(np.float64).sum(1)
    assert (np.abs(got[ok] - want) <= bar).all(), (got[ok], want)


# ------------------------------------------------------------------------------------------------
# the loop (-m gpu)
# ------------------------------------------------------------------------------------------------
def _small_model(params, L, Bn, gm, kv):
    import test_gpu_parity as GP
    from mt3_b200 import network
    return network.Transformer(GP._mt3_cfg(num_encoder_layers=2, num_decoder_layers=2), params, device=DEV, max_batch=Bn,
                               max_input_length=64, max_decode_length=L, gemm_mode=gm, kv_format=kv)


@pytest.mark.gpu
def test_generate_with_a_full_graph_cache():
    """The step-graph cache holds 12 graphs over all (workspace, batch, input length) bindings.  A generate of 17 steps
    takes the binding's 16-step graph from the cache and then captures its single-step graph; when that capture fills the
    cache, the graphs evicted are other bindings', never the 16-step graph the call is about to replay.  Scored tokens and
    scores equal plain launches', bit for bit, before and after the eviction."""
    import torch
    import test_gpu_parity as GP
    from mt3_b200 import _lib
    ocfg = O.T5Config(vocab_size=1536, num_encoder_layers=2, num_decoder_layers=2)
    m = _small_model(O.init_params(ocfg, seed=5), 48, 8, _lib.GEMM_TF32X3, _lib.KV_F32)
    x = torch.from_numpy(GP._inputs(8, t=64, seed=70)).to(DEV)
    m.generate(x, num_steps=0)                       # the largest workspace first: every binding below shares its address

    def run(b, steps, graph):
        return [t.cpu().numpy() for t in m.generate(x[:b], num_steps=steps, stop_at_eos=False, use_graph=graph, return_scores=True)]

    want = run(1, 17, False)
    first = run(1, 16, True)                         # cache: B = 1's 16-step graph
    for b in range(2, 7):
        run(b, 17, True)                             # + 2 graphs per batch size: 11
    run(7, 16, True)                                 # 12: the next capture evicts
    got = run(1, 17, True)                           # B = 1's 16-step graph from the cache, then a capture
    for a, w in zip(got, want):
        _same_bits("17 steps at a full graph cache vs plain launches", a, w)
    np.testing.assert_array_equal(first[0][:, :16], want[0][:, :16])
    _same_bits("16 steps vs plain launches", first[1][:, :16], want[1][:, :16])
    np.testing.assert_array_equal(run(3, 17, True)[0], run(3, 17, False)[0])


@pytest.mark.gpu
def test_greedy_scores_match_teacher_forced_pass():
    """Greedy generate with scores (MT3_KV_F32, TF32X3, B = 8, EOS-boosted weights so that sequences end at different
    steps) against Transformer.score on the generated tokens, weights 1 through EOS: per token within twice the logit bar
    of test_agrees_with_step_path times max |logit|, sequence scores within the sum of the per-token bars.  The
    teacher-forced pass masks keys whose target is 0, the loop does not, so positions from a PAD emitted before EOS on
    are left out."""
    import torch
    import test_gpu_parity as GP
    from mt3_b200 import _lib
    ocfg = O.T5Config(vocab_size=1536, num_encoder_layers=2, num_decoder_layers=2)
    params = GP._eos_params(ocfg, seed=9, boost=6.0)
    L, Bn = 48, 8
    m = _small_model(params, L, Bn, _lib.GEMM_TF32X3, _lib.KV_F32)
    x = GP._inputs(Bn, t=64, seed=50)
    xg = torch.from_numpy(x).to(DEV)
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, stop_at_eos=True, use_graph=True, return_scores=True))
    ran = m.last_steps_run
    has_eos = (tok == EOS).any(1)
    assert 0 < has_eos.sum(), "the boosted weights should end some sequences"
    end = np.where(has_eos, np.argmax(tok == EOS, 1) + 1, ran)
    w = (np.arange(L)[None] < end[:, None]).astype(np.int32)
    din = np.concatenate([np.zeros((Bn, 1), np.int32), tok[:, :-1]], axis=1)
    ref = m.score(m.encode(xg), torch.from_numpy(din).to(DEV), torch.from_numpy(tok).to(DEV),
                  torch.from_numpy(w).to(DEV)).cpu().numpy()
    # the logit bar of test_agrees_with_step_path, from the float32 oracle's deviation on these tokens
    enc64 = O.encode(params, ocfg, x, np.float64)
    _, l64 = O.greedy_decode(params, ocfg, enc64, L, np.float64, stop_at_eos=False, return_logits=True, forced_tokens=din)
    _, l32 = O.greedy_decode(params, ocfg, enc64.astype(np.float32), L, np.float32, stop_at_eos=False, return_logits=True,
                             forced_tokens=din)
    real = w > 0
    scale = np.abs(l64[real]).max()
    e_f32 = np.abs(l32[real] - l64[real]).max() / scale
    bar = 2 * (2 * max(4 * e_f32, 2e-5)) * scale
    assert (ts[~real] == 0).all()
    pad_in = np.where(((tok == PAD) & real).any(1), np.argmax((tok == PAD) & real, 1), L)
    keep = real & (np.arange(L)[None] < pad_in[:, None])
    d = np.abs(ts - ref)[keep]
    print(f"loop vs teacher-forced pass: worst per-token |d| {d.max():.2e}, bar {bar:.2e} (e_f32 {e_f32:.2e}); steps run {ran}, "
          f"lengths {end.tolist()}")
    assert (d <= bar).all()
    whole = pad_in >= end
    assert whole.sum() >= Bn // 2
    assert (np.abs(sc - ref.astype(np.float64).sum(1))[whole] <= (bar * end)[whole]).all()


@pytest.mark.gpu
def test_scores_against_float64():
    """On the 2-layer model of test_generate_beam1_matches_t5x_beam_search_restatement: greedy token scores equal the
    float64 oracle's log_softmax at its tokens within max(4 e_f32, 2e-5) of max |logit| per token, over the prefix where
    the tokens agree; beam1's tokens equal BS.beam_search's and its score is within the summed per-token bar."""
    import torch
    import test_gpu_parity as GP
    from mt3_b200 import _lib
    ocfg = O.T5Config(vocab_size=1536, num_encoder_layers=2, num_decoder_layers=2)
    params = GP._eos_params(ocfg, seed=9, boost=4.0)
    L, Bn = 48, 8
    m = _small_model(params, L, Bn, _lib.GEMM_FP32_SIMT, _lib.KV_F32)
    x = GP._inputs(Bn, t=64, seed=50)
    xg = torch.from_numpy(x).to(DEV)
    enc64 = O.encode(params, ocfg, x, np.float64)
    ref, l64 = O.greedy_decode(params, ocfg, enc64, L, np.float64, stop_at_eos=False, return_logits=True)
    din = np.concatenate([np.zeros((Bn, 1), np.int64), ref[:, :-1]], axis=1)
    _, l32 = O.greedy_decode(params, ocfg, O.encode(params, ocfg, x, np.float32), L, np.float32, stop_at_eos=False,
                             return_logits=True, forced_tokens=din)
    scale = np.abs(l64).max()
    e_f32 = np.abs(l32 - l64).max() / scale
    bar = max(4 * e_f32, 2e-5) * scale
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, stop_at_eos=False, use_graph=True, return_scores=True))
    alive = np.cumsum(ref == EOS, 1) - (ref == EOS) == 0
    same = np.cumprod(tok == ref, 1).astype(bool) & alive
    lp64 = np.take_along_axis(BS.log_softmax(l64), ref[..., None].astype(np.int64), -1)[..., 0]
    d = np.abs(ts - lp64)[same]
    print(f"greedy token scores vs fp64: worst {d.max():.2e}, bar {bar:.2e} (e_f32 {e_f32:.2e}); {int(same.sum())} tokens")
    assert same.sum() >= Bn * 4 and (d <= bar).all()
    # beam1
    p64 = O._cast(params, np.float64)
    state = O.init_decode_state(ocfg, Bn, L, np.float64)

    def logits_fn(prefixes, step):
        cur = prefixes[:, 0, step - 1] if step > 0 else np.zeros((Bn,), np.int64)
        return O.decode_step(p64, ocfg, enc64, cur, state)[:, None, :]

    want, score = BS.beam_search(logits_fn, Bn, L, eos_id=O.EOS_ID, num_decodes=1)
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, stop_at_eos=False, use_graph=True, decode='beam1', return_scores=True))
    np.testing.assert_array_equal(tok, want)
    n = np.where((tok == EOS).any(1), np.argmax(tok == EOS, 1) + 1, L)
    print(f"beam1 scores vs fp64: worst {np.abs(sc - score).max():.2e}, lengths {n.tolist()}")
    assert (np.abs(sc - score) <= bar * n).all(), (sc, score)


@pytest.fixture(scope="module")
def bench_inputs():
    import torch
    from mt3_b200 import spectrograms
    audio = np.stack([O.sine_mix(256 * 128, seed=4000 + i) for i in range(64)])
    return spectrograms.compute_spectrogram(torch.from_numpy(audio).to(DEV), spectrograms.SpectrogramConfig())


@pytest.mark.gpu
@pytest.mark.parametrize("decode", ["greedy", "beam1"])
@pytest.mark.parametrize("kv", ["p24", "f32"])
def test_bit_identity_at_bench_configuration(bench_inputs, kv, decode):
    """bench.py's configuration (mt3, B = 64, 1024 steps, TF32X3, graphs): tokens with return_scores=True equal those
    without; scores from graph replay equal scores from plain launches bit for bit; with stop_at_eos=True the token scores
    and scores equal the full run's (the steps after the stop score 0 in both)."""
    import torch
    from mt3_b200 import _lib, inference
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=64, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format={"p24": _lib.KV_P24, "f32": _lib.KV_F32}[kv])
    m = im.model
    plain_tok = m.generate(bench_inputs, stop_at_eos=False, use_graph=True, decode=decode).cpu().numpy()
    g = [t.cpu().numpy() for t in m.generate(bench_inputs, stop_at_eos=False, use_graph=True, decode=decode, return_scores=True)]
    assert m.last_steps_run == 1024
    p = [t.cpu().numpy() for t in m.generate(bench_inputs, stop_at_eos=False, use_graph=False, decode=decode, return_scores=True)]
    s = [t.cpu().numpy() for t in m.generate(bench_inputs, stop_at_eos=True, use_graph=True, decode=decode, return_scores=True)]
    ran = m.last_steps_run
    np.testing.assert_array_equal(g[0], plain_tok)
    np.testing.assert_array_equal(p[0], plain_tok)
    _same_bits(f"{kv} {decode}: token scores, graph vs plain", g[1], p[1])
    _same_bits(f"{kv} {decode}: scores, graph vs plain", g[2], p[2])
    np.testing.assert_array_equal(s[0], plain_tok)
    _same_bits(f"{kv} {decode}: token scores, early stop vs full run", s[1], g[1])
    _same_bits(f"{kv} {decode}: scores, early stop vs full run", s[2], g[2])
    assert np.isfinite(g[1]).all() and (g[1] <= 1e-6).all() and g[1].dtype == np.float32
    print(f"{kv} {decode}: early stop after {ran} steps; scores {np.round(g[2][:4], 3).tolist()}")
    del im, m
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("decode", ["greedy", "beam1"])
def test_transcribe_segments_return_scores(decode):
    """InferenceModel.transcribe_segments(return_scores=True): host int32 [S, 1024], float32 [S, 1024], float32 [S]; the
    decoded tokens equal the return_scores=False call's; token scores are 0 after EOS and beyond the steps; greedy scores
    are the token scores' sums.  S = 5 in batches of 2 (a short tail batch), EOS-boosted weights."""
    from mt3_b200 import inference, weights
    im = inference.InferenceModel('synthetic:0', 'mt3', device=DEV, batch_size=2, decode=decode)
    p = weights.synthetic_params(im.model.config, 0)
    p["decoder/logits_dense/kernel"] = p["decoder/logits_dense/kernel"].copy()
    p["decoder/logits_dense/kernel"][:, EOS] *= 6.0
    im.restore_from_checkpoint(p)
    audio = np.stack([O.sine_mix(32768, 600 + i) for i in range(5)])
    steps = 40
    want = im.transcribe_segments(audio, num_steps=steps)
    tok, ts, sc = im.transcribe_segments(audio, num_steps=steps, return_scores=True)
    assert tok.shape == (5, 1024) and tok.dtype == np.int32
    assert ts.shape == (5, 1024) and ts.dtype == np.float32 and sc.shape == (5,) and sc.dtype == np.float32
    np.testing.assert_array_equal(tok, want)
    raw, ts_raw, sc_raw = im.transcribe_segments(audio, num_steps=steps, return_scores=True, decoded=False)
    _same_bits("token scores, decoded vs raw", ts_raw, ts)
    assert (ts[:, steps:] == 0).all()
    n_eos = 0
    for b in range(5):
        if (raw[b] == EOS).any():
            e = int(np.argmax(raw[b] == EOS))
            assert (ts[b, e + 1:] == 0).all() and ts[b, e] <= 0
            n_eos += 1
    if decode == "greedy":
        np.testing.assert_allclose(sc, ts.astype(np.float64).sum(1), rtol=1e-5, atol=1e-5)
    sh = im.transcribe_segments_sharded(audio, num_steps=steps, return_scores=True)
    for a, b_ in zip(sh, (tok, ts, sc)):
        np.testing.assert_array_equal(a, b_)
    print(f"{decode}: {n_eos} of 5 segments emitted EOS within {steps} steps; scores {np.round(sc, 3).tolist()}")
