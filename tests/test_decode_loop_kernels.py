"""The decode loop's token-selection kernels launched alone (mt3_b200/csrc/tools/kernel_harness.cu -> libmt3kernels.so), against
numpy restatements kept in this file: argmax_step_kernel (greedy pick, EOS/PAD bookkeeping, the arrival counter, the fused
next-step embedding), beam1_step_kernel + beam1_finalize_kernel (T5X beam search at num_decodes = 1, judged against
oracle/beam_search.py), embed_kernel, and the encoder's row_rstd_kernel / rmsnorm_kernel.

Token ids and the bookkeeping are compared exactly, on crafted logit rows where pickers go wrong: exact ties held by one
thread (ids i and i + 256), by adjacent lanes and by different warps, the maximum at id 0 and at id V - 1, all-equal and
all--inf rows, -0.0 tied with +0.0, denormals, NaN, V < 256.  Float outputs that are plain adds (y_next, embed) are compared
bit for bit with the float32 numpy add.  Buffers are padded and start as a sentinel (NaN for floats unless NaN is what a
defect would write, -7 for ints); after every launch nothing outside the logical output may have changed.

GPU tests carry the gpu mark one by one: the self-checks of the restatements run on the CPU.
"""
import ctypes as C
import importlib.util
import math
import os

import numpy as np
import pytest

from oracle import beam_search as BS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "mt3_b200", "csrc", "tools")
DEV = "cuda:0"
U = 2.0 ** -24            # fp32 unit roundoff
EOS, PAD = 1, 0
ALPHA = 0.6
SENT = -7                 # int sentinel
YSENT = -777.0            # y_next sentinel: finite, so that a read of the NaN guard rows past the PE table shows


# ------------------------------------------------------------------------------------------------
# numpy restatements
# ------------------------------------------------------------------------------------------------
def argmax_ref(x):
    """np.argmax's order, stated without np.argmax: NaN above every number, the first NaN / the first maximum wins."""
    x = np.asarray(x, np.float32)
    nan = np.isnan(x)
    xm = np.where(nan, -np.inf, x)
    first_max = (xm == xm.max(-1, keepdims=True)).argmax(-1)
    return np.where(nan.any(-1), nan.argmax(-1), first_max)


def greedy_step_ref(logits, finished):
    """One step of the greedy loop (BS.greedy): next = argmax; finished rows emit PAD; EOS marks finished.
    finished None: the raw pick (mt3_decode_step)."""
    nxt = argmax_ref(logits)
    if finished is None:
        return nxt, None
    nxt = np.where(finished, PAD, nxt)
    return nxt, finished | (nxt == EOS)


def _bp(n):
    return BS.brevity_penalty(ALPHA, n)


def beam1_trace(lg, L):
    """T5X beam search at num_decodes = 1 for ONE element, restated step by step in float64 from fp32 logits lg [>= L, V],
    together with an error bar for each value beam1_step_kernel computes in fp32.  Cross-checked against
    BS.beam_search (tokens, score, number of logits_fn calls) by test_beam1_trace_matches_beam_search.

    Bars (u = 2^-24).  One step's log-probability v - lse, lse = gmx + logf(tot), tot = sum_k expf(l_k - gmx):
      the argument l_k - gmx is rounded (relative u |x_k| on its exp term: u E_p|x| on tot), expf is <= 2 ulp (4u),
      tot sums ceil(V/256) terms per thread, a 5-level warp tree and 8 warp sums (ceil(V/256) + 13 roundings), logf is
      <= 1 ulp (2u |log tot|), then the add of gmx (u |lse|) and the subtraction from v (u |v - lse|);
    live_lp accumulates those (plus u |live| per add); a finish candidate (live + lp_eos) / bp(n) adds one add, the
    division and powf (<= 4 ulp of bp, argument rounded: 10u |cand| in all)."""
    L = int(L)
    V = lg.shape[-1]
    bpL = _bp(L)
    live, bar_live, fin, bar_fin, fin_len = 0.0, 0.0, BS.NEG_INF, 0.0, 0
    toks, steps, margins = [], [], []
    for i in range(L):
        if i > 0 and fin_len > 0:
            r = live / bpL
            margins.append(("settle", i, abs(fin - r), bar_fin + bar_live / bpL + 10 * U * abs(r)))
            if fin > r:
                break
        l = lg[i].astype(np.float64)
        gmx = l.max()
        x = l - gmx
        e = np.exp(x)
        tot = e.sum()
        lse = gmx + math.log(tot)
        ep = float((e * np.abs(x)).sum() / tot)
        base = U * (4 + math.ceil(V / 256) + 13 + ep + 2 * abs(math.log(tot)) + abs(lse))

        def e_lp(v):
            return base + U * abs(v - lse)
        order = sorted((k for k in range(V) if k != EOS), key=lambda k: (-lg[i, k], k))   # stable: lower id first
        i1, i2 = order[0], order[1] if len(order) > 1 else None
        v2 = lg[i, i2] if i2 is not None else -np.inf
        eos_top2 = lg[i, EOS] > v2 or (lg[i, EOS] == v2 and (i2 is None or EOS < i2))
        if eos_top2:
            s = live + (l[EOS] - lse)
            cand = s / _bp(i + 1)
            bar_c = (bar_live + e_lp(l[EOS]) + U * abs(s)) / _bp(i + 1) + 10 * U * abs(cand)
            margins.append(("finish", i, abs(cand - fin), bar_c + bar_fin))
            if cand > fin:                       # an existing finished hypothesis beats an equal newcomer
                fin, bar_fin, fin_len = cand, bar_c, i + 1
        live += l[i1] - lse
        bar_live += e_lp(l[i1]) + U * abs(live)
        toks.append(i1)
        steps.append((live, bar_live, fin, bar_fin, fin_len))
    out = np.zeros(L, np.int32)
    if fin_len:
        out[:fin_len - 1] = toks[:fin_len - 1]
        out[fin_len - 1] = EOS
    else:
        out[:len(toks)] = toks
    return dict(tokens=out, fin_len=fin_len, calls=len(steps), steps=steps, margins=margins,
                score=fin if fin_len else live)


def _probs_row(V, named):
    """log of a distribution over V ids: named masses, the rest spread evenly, as float32 logits"""
    p = np.zeros(V)
    for k, v in named.items():
        p[k] = v
    rest = p == 0
    p[rest] = (1.0 - p.sum()) / rest.sum()
    return np.log(p).astype(np.float32)


def _table(V, L, rows):
    """[L, V] logits: the given rows, the last one repeated"""
    return np.stack([rows[min(i, len(rows) - 1)] for i in range(L)])


BEAM_L = 8


def beam_scenarios(V):
    """Crafted logit streams [BEAM_L, V] (ids: 0 PAD, 1 EOS), name -> stream."""
    rng = np.random.default_rng(V)
    P = lambda **kw: _probs_row(V, {int(k[1:]): v for k, v in kw.items()})     # P(i2=.9, i1=.01): id 2 .9, EOS .01
    hi = V - 1
    sc = {
        # EOS decisive at step 1; settles at once
        "eos_first_settles": [P(i2=.9, i1=.01), P(i1=.97, i4=.01), P(i4=.5, i1=.3)],
        # EOS ranks second at step 1 and wins on the normalised score over greedy's later finish
        "eos_second_wins": [P(i2=.9, i1=.01), P(i2=.6, i1=.35), P(i3=.5, i1=.02), P(i1=.9, i4=.05)],
        # EOS ranks first at step 1 but the runner-up's later finish scores better
        "eos_first_loses": [P(i2=.9, i1=.01), P(i1=.5, i2=.45), P(i3=.99, i1=.002), P(i4=.99, i1=.002), P(i1=.99, i4=.002)],
        "no_eos": [P(i2=.7, i1=.0001)],
    }
    # an exact tie between EOS and the runner-up: at id 0 the runner-up ranks first (no finish), at id 7 EOS does
    for r in (0, 7):
        row = rng.uniform(-3, -2, V).astype(np.float32)
        row[5], row[EOS], row[r] = 1.0, -0.5, -0.5
        sc[f"eos_ties_runner_up_id{r}"] = [row, P(i3=.9, i1=.00001)]
    # EOS tied with the best non-EOS (at id 0 and at id V - 1): both rank in the top 2
    for r in (0, hi):
        row = rng.uniform(-3, -2, V).astype(np.float32)
        row[EOS], row[r] = 0.5, 0.5
        sc[f"eos_ties_best_id{r}"] = [P(i2=.8, i1=.01), row, P(i4=.7, i1=.2), P(i1=.95, i4=.01)]
    # non-EOS ties (best and second best) held by one thread (i, i + 256), adjacent lanes, different warps
    adj = min(40, V - 3)
    pairs = [(3, 3 + 256) if V > 259 else (3, 4), (adj, adj + 1), (5, min(5 + 32 * 5, hi)), (0, hi)]
    rows = []
    for a, b in pairs:
        row = rng.uniform(-3, -2, V).astype(np.float32)
        row[a] = row[b] = 1.0
        row[2] = row[6] = 0.25                               # second-best tie
        row[EOS] = -1.0
        rows.append(row)
    sc["non_eos_ties"] = rows + [P(i1=.9, i4=.01)]
    # logits of magnitude ~1e3: the log-sum-exp's rounding is ~1e3 u per step
    big = []
    for i in range(4):
        row = (rng.uniform(-1, 0.4, V) * 1e3).astype(np.float32)
        row[2 + i] = 1000.0
        row[EOS] = 998.5 if i < 3 else 1003.0
        big.append(row)
    sc["magnitude_1e3"] = big
    return {k: _table(V, BEAM_L, v) for k, v in sc.items()}


# ------------------------------------------------------------------------------------------------
# CPU self-checks of the restatements
# ------------------------------------------------------------------------------------------------
def _crafted_rows(V):
    """Tie / NaN / signed-zero / denormal rows and the id np.argmax gives each."""
    rows = []

    def row(fill=-1.0):
        return np.full(V, fill, np.float32)
    r = row(); j = 3 if V > 259 else 40 % (V - 1); k = j + 256 if V > 259 else j + 1; r[j] = r[k] = 10; rows.append((r, j))
    r = row(); r[min(40, V - 2)] = r[min(40, V - 2) + 1] = 10; rows.append((r, min(40, V - 2)))
    r = row(); r[5] = r[min(V - 1, 5 + 32 * 5)] = 10; rows.append((r, 5))
    r = row(); r[0] = 10; rows.append((r, 0))
    r = row(); r[V - 1] = 10; rows.append((r, V - 1))
    rows.append((row(0.25), 0))
    rows.append((row(-np.inf), 0))
    r = row(); r[3] = -0.0; r[9] = 0.0; rows.append((r, 3))
    r = row(); r[3] = 0.0; r[9] = -0.0; rows.append((r, 3))
    r = row(0.0); r[7] = 1.4e-45; r[V - 2] = 2.8e-45; rows.append((r, V - 2))
    r = row(-1e-45); r[4] = r[V - 1] = 3e-45; rows.append((r, 4))
    rows.append((row(np.nan), 0))
    r = row(); j = min(17, V - 3); r[V - 1] = np.inf; r[j] = r[j + 2] = np.nan; rows.append((r, j))
    r = row(); r[0] = np.inf; r[V - 1] = np.nan; rows.append((r, V - 1))
    r = row(); r[EOS] = 10; rows.append((r, EOS))
    return rows


@pytest.mark.parametrize("V", [1536, 1516, 257, 33])
def test_argmax_restatement_matches_np_argmax_and_greedy(V):
    """argmax_ref == np.argmax on tie / NaN / signed-zero / denormal rows; iterating greedy_step_ref == BS.greedy."""
    rows = _crafted_rows(V)
    x = np.stack([r for r, _ in rows])
    with np.errstate(invalid="ignore"):
        np.testing.assert_array_equal(argmax_ref(x), np.argmax(x, -1))
    np.testing.assert_array_equal(argmax_ref(x), [w for _, w in rows])
    rng = np.random.default_rng(V)
    B, L = 5, len(rows) + 3
    stream = rng.standard_normal((L, B, V)).astype(np.float32)
    for i in range(L):
        for b in range(B):
            if (i + 3 * b) % 2 == 0:
                stream[i, b] = rows[(i + b) % len(rows)][0]
    stream[L - 1, :, EOS] = np.inf                            # every element ends
    fin = np.zeros(B, bool)
    mine = np.zeros((B, L), np.int32)
    for i in range(L):
        mine[:, i], fin = greedy_step_ref(stream[i], fin)
    with np.errstate(invalid="ignore"):
        want = BS.greedy(lambda prefixes, step: stream[step][:, None, :], B, L)
    np.testing.assert_array_equal(mine, want)


@pytest.mark.parametrize("V", [1536, 1516, 257, 33])
def test_beam1_trace_matches_beam_search(V):
    """beam1_trace (which the kernel test reads beam_f bars and settle steps from) == BS.beam_search on every crafted
    stream: tokens, score, and number of logits_fn calls; and every float64 finish / settle comparison of every stream
    has a margin larger than its fp32 bar, so no stream depends on a near-tie."""
    for name, lg in beam_scenarios(V).items():
        t = beam1_trace(lg, BEAM_L)
        calls = []
        want, score = BS.beam_search(lambda p, s: (calls.append(s), lg[None, None, s])[1], 1, BEAM_L)
        np.testing.assert_array_equal(t["tokens"], want[0], err_msg=name)
        assert abs(t["score"] - score[0]) <= 1e-12 * max(1.0, abs(score[0])), name
        assert t["calls"] == len(calls), name
        for kind, i, m, bar in t["margins"]:
            assert m > bar, f"{name}: {kind} comparison at step {i} has margin {m:.3e} <= bar {bar:.3e}"
    sc = beam_scenarios(V)
    lens = {k: beam1_trace(v, BEAM_L)["fin_len"] for k, v in sc.items()}
    assert lens["no_eos"] == 0 and lens["eos_first_settles"] == 2 and lens["eos_second_wins"] == 2
    assert lens["eos_first_loses"] > 2
    assert lens["eos_ties_runner_up_id0"] == 0 and lens["eos_ties_runner_up_id7"] == 1


def test_beam1_all_nan_row_restatement():
    """On an all-NaN row the restatement's stable top-2 is ids 0 and 1: id 0 is the best non-EOS extension, which
    beam1_step_kernel continues with, and the EOS candidate's score is NaN, so nothing finishes.  (Its live re-sort then
    ranks the NaN score of id 0 below the NEG_INF it gives the EOS extension; the kernel never continues with EOS.)"""
    lg = np.full((4, 9), np.nan, np.float32)
    with np.errstate(invalid="ignore"):
        top = np.argsort(-BS.log_softmax(lg[0].astype(np.float64)), kind="stable")[:2]
        out, score = BS.beam_search(lambda p, s: lg[None, None, s], 1, 4)
    np.testing.assert_array_equal(top, [0, 1])
    assert score[0] == BS.NEG_INF and (out[0] == EOS).all()           # nothing finished: it returns that live beam


# ------------------------------------------------------------------------------------------------
# the harness library
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def kh():
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(TOOLS, "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if bt.harness_stale():
        bt.main()
    lib = C.CDLL(bt.HARNESS)
    P, I, F = C.c_void_p, C.c_int, C.c_float
    sig = {
        "kh_last_error": ([], C.c_char_p),
        "kh_argmax_step": ([P, I, I, P, P, P, I, P, P, I, I, P, P, I, I, P, I], I),
        "kh_beam1_step": ([P, I, I, P, P, P, I, P, P, P, F, I, P, P, I, I, P], I),
        "kh_beam1_finalize": ([P, I, I, I, P], I),
        "kh_embed": ([P, P, I, I, P, P, P, I, I], I),
        "kh_row_rstd": ([P, P, I, I, I, F, P], I),
        "kh_rmsnorm": ([P, P, I, I, I, F, P, P, I], I),
    }
    for name, (args, res) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, res
    return lib


def _call(kh, fn, *args):
    import torch
    r = getattr(kh, fn)(*args)
    assert r == 0, f"{fn} -> {r}: {kh.kh_last_error().decode()}"
    torch.cuda.synchronize()


def _p(t):
    return None if t is None else t.data_ptr()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(t):
    return t.cpu().numpy()


def _same_bits(name, got, want):
    """float32 arrays equal bit for bit (NaN payloads aside: NaN where NaN is expected)"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    ok = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not ok.all():
        i = np.unravel_index(np.argmin(ok), ok.shape)
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.size} elements differ; at {i}: got {got[i]!r} want {want[i]!r}")


def _pe_with_guard(rng, rows, D):
    """[rows + 2, D] table whose last two rows are NaN: a read past row rows - 1 stays inside the allocation and shows"""
    pe = np.full((rows + 2, D), np.nan, np.float32)
    pe[:rows] = rng.standard_normal((rows, D)).astype(np.float32)
    return pe


# ------------------------------------------------------------------------------------------------
# argmax_step_kernel
# ------------------------------------------------------------------------------------------------
def _greedy_logits(rng, B, V, step, crafted):
    x = rng.standard_normal((B, V)).astype(np.float32)
    for b in range(B):
        k = (b * 7 + step) % (len(crafted) + 3)
        if k < len(crafted):
            x[b] = crafted[k][0]
        if step >= 10 and (b + step) % 17 == 0:               # EOS wins: every element ends between steps 10 and 26
            x[b, EOS] = np.float32(20.0)
    return x


GREEDY_SHAPES = {
    # name: (tok_cur, finished, tokens_out, tok_user, y_next, advance)
    "generate": (1, 1, 1, 0, 1, 1),
    "decode_step": (0, 0, 0, 1, 0, 1),
    "advance0": (1, 1, 1, 1, 1, 0),
}


def _run_greedy(kh, B, V, shape, split, steps=40, D=512, seed=0):
    import torch
    use_cur, use_fin, use_out, use_user, use_y, advance = GREEDY_SHAPES[shape]
    rng = np.random.default_rng(seed + B * 7 + V)
    crafted = _crafted_rows(V)
    p0 = 5 if not advance else 8
    pe_rows = p0 + steps                                     # the last step (pos = pe_rows - 1) has no PE row after it
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = _pe_with_guard(rng, pe_rows, D)
    out_ld = pe_rows + 3
    d_emb, d_pe = _dev(emb), _dev(pe)
    d_lg = torch.full(((B + 1) * V,), float("nan"), dtype=torch.float32, device=DEV)
    st = np.array([p0, 0, 0, SENT], np.int32)
    cur = np.full(B + 1, SENT, np.int32)
    fin = np.full(B + 1, SENT, np.int32); fin[:B] = 0
    tok = np.full((B + 1, out_ld), SENT, np.int32)
    usr = np.full(B + 1, SENT, np.int32)
    d_st, d_cur, d_fin, d_tok, d_usr = (_dev(a) for a in (st, cur, fin, tok, usr))
    d_y = torch.full(((B + 1) * D,), YSENT, dtype=torch.float32, device=DEV)
    fin_ref = np.zeros(B, bool) if use_fin else None
    pos = p0
    for step in range(steps):
        lg = _greedy_logits(rng, B, V, step, crafted)
        d_lg[:B * V] = _dev(lg.ravel())
        d_y.fill_(YSENT)
        ptrs = (_p(d_cur) if use_cur else None, _p(d_fin) if use_fin else None, _p(d_tok) if use_out else None, out_ld,
                _p(d_usr) if use_user else None, _p(d_st), advance)
        tail = (_p(d_emb), _p(d_pe), pe_rows, D, _p(d_y) if use_y else None)
        parts = [(0, B)] if not split else [(0, B // 3), (B // 3, B)]
        for j, (a, b) in enumerate(parts):
            _call(kh, "kh_argmax_step", _p(d_lg), V, B, *ptrs, a, *tail, b - a)
            if j + 1 < len(parts) and advance:               # the counter holds the arrivals; the position has not moved
                s = _np(d_st)
                assert s[0] == pos and s[1] == b, (step, s)
        nxt, fin_new = greedy_step_ref(lg, fin_ref)
        assert ((nxt >= 0) & (nxt < V)).all()
        if use_cur:
            cur[:B] = nxt
        if use_fin:
            fin[:B] = fin_new
            fin_ref = fin_new
        if use_out:
            tok[:B, pos] = nxt
        if use_user:
            usr[:B] = nxt
        if advance:
            st[:3] = [pos + 1, 0, int(fin_ref.all()) if use_fin else 0]
        for name, d, want in (("state", d_st, st), ("tok_cur", d_cur, cur), ("finished", d_fin, fin), ("tokens_out", d_tok, tok),
                              ("tok_user", d_usr, usr)):
            np.testing.assert_array_equal(_np(d), want, err_msg=f"{shape} B={B} V={V} step {step}: {name}")
        y = np.full((B + 1, D), YSENT, np.float32)
        if use_y and pos + 1 < pe_rows:
            y[:B] = emb[nxt] + pe[pos + 1]
        _same_bits(f"{shape} B={B} V={V} step {step}: y_next", _np(d_y).reshape(B + 1, D), y)
        if advance:
            pos += 1
    if use_fin:
        assert fin_ref.all() and st[2] == advance            # every element ended between steps 10 and 26


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1516, 257, 33])
@pytest.mark.parametrize("B", [1, 64, 96])
@pytest.mark.parametrize("shape", list(GREEDY_SHAPES))
def test_argmax_step_kernel(kh, shape, B, V):
    """40 steps of fresh logits with crafted rows; after every step tokens_out (column pos only), tok_cur, tok_user,
    finished, state (position advanced once, counter back to 0, all-finished only once every row has finished, 0
    without `finished`) and y_next = E[next] + PE[pos + 1] (bit for bit; untouched at the last step, where pos + 1 is
    past the PE table) match the restatement."""
    _run_greedy(kh, B, V, shape, split=False)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 33])
@pytest.mark.parametrize("B", [64, 96])
def test_argmax_step_kernel_two_launches(kh, B, V):
    """The batch as two launches (b0 = 0 and b0 > 0, uneven halves) with one arrival counter: the position advances
    once, after the second launch."""
    _run_greedy(kh, B, V, "generate", split=True)


@pytest.mark.gpu
def test_argmax_step_nan_rows(kh):
    """All-NaN and partly NaN rows pick the first NaN (np.argmax), never an id outside [0, V)."""
    V, B = 1536, 4
    rng = np.random.default_rng(1)
    lg = rng.standard_normal((B, V)).astype(np.float32)
    lg[0] = np.nan
    lg[1, 700] = lg[1, 900] = np.nan
    lg[2, 0] = np.inf; lg[2, 1535] = np.nan
    want = argmax_ref(lg)
    np.testing.assert_array_equal(want[:3], [0, 700, 1535])
    d_lg, d_st, d_usr = _dev(lg), _dev(np.array([0, 0, 0, SENT], np.int32)), _dev(np.full(B + 1, SENT, np.int32))
    _call(kh, "kh_argmax_step", _p(d_lg), V, B, None, None, None, 0, _p(d_usr), _p(d_st), 1, 0, None, None, 0, 0, None, B)
    np.testing.assert_array_equal(_np(d_usr), list(want) + [SENT])


@pytest.mark.gpu
def test_step_kernels_skip_y_next_past_pe_table(kh):
    """At pos = pe_rows - 1 neither step kernel writes y_next: PE has no row pos + 1 (the rows after the table are NaN
    guards inside the same allocation, so a read of them would show as NaN); at pos = pe_rows - 2 both write
    E[next] + PE[pos + 1]."""
    import torch
    V, B, D, rows = 1536, 3, 512, 6
    rng = np.random.default_rng(2)
    lg = rng.standard_normal((B, V)).astype(np.float32)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = _pe_with_guard(rng, rows, D)
    d_lg, d_emb, d_pe = _dev(lg), _dev(emb), _dev(pe)
    for kind in ("greedy", "beam1"):
        for pos in (rows - 2, rows - 1):
            d_st = _dev(np.array([pos, 0, 0, SENT], np.int32))
            d_cur, d_fin = _dev(np.full(B, SENT, np.int32)), _dev(np.zeros(B, np.int32))
            d_tok = _dev(np.full((B, rows), SENT, np.int32))
            d_bf, d_bi = _dev(np.tile(np.float32([0.0, -1.0e7]), B)), _dev(np.zeros(B, np.int32))
            d_y = torch.full((B * D,), YSENT, dtype=torch.float32, device=DEV)
            if kind == "greedy":
                _call(kh, "kh_argmax_step", _p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), rows, None, _p(d_st), 1, 0,
                      _p(d_emb), _p(d_pe), rows, D, _p(d_y), B)
            else:
                _call(kh, "kh_beam1_step", _p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), rows, _p(d_st), _p(d_bf), _p(d_bi),
                      ALPHA, rows, _p(d_emb), _p(d_pe), rows, D, _p(d_y))
            nxt = _np(d_cur)
            assert ((nxt >= 0) & (nxt < V)).all() and (_np(d_tok)[:, pos] == nxt).all()
            y = emb[nxt] + pe[pos + 1] if pos + 1 < rows else np.full((B, D), YSENT, np.float32)
            _same_bits(f"{kind} y_next at pos {pos} of {rows} PE rows", _np(d_y).reshape(B, D), y)


# ------------------------------------------------------------------------------------------------
# beam1_step_kernel + beam1_finalize_kernel
# ------------------------------------------------------------------------------------------------
def _run_beam(kh, lg, L, D=64, seed=0):
    """lg [B, L, V] fp32: L kernel steps (the whole loop, as with stop_at_eos off) and the finalize.  Returns the finalized
    tokens, beam_i, the first step count at which each finished[b] was 1 (L + 1: never), and beam_f after every step."""
    import torch
    B, _, V = lg.shape
    rng = np.random.default_rng(seed)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = _pe_with_guard(rng, L, D)
    d_emb, d_pe = _dev(emb), _dev(pe)
    d_lg = torch.full(((B + 1) * V,), float("nan"), dtype=torch.float32, device=DEV)
    bf = np.full(2 * B + 2, np.nan, np.float32); bf[0:2 * B:2], bf[1:2 * B:2] = 0.0, -1.0e7
    bi = np.full(B + 1, SENT, np.int32); bi[:B] = 0
    fin = np.full(B + 1, SENT, np.int32); fin[:B] = 0
    d_st, d_bf, d_bi, d_fin = _dev(np.array([0, 0, 0, SENT], np.int32)), _dev(bf), _dev(bi), _dev(fin)
    d_cur = _dev(np.full(B + 1, SENT, np.int32))
    d_tok = _dev(np.full((B + 1) * L, SENT, np.int32))
    d_y = torch.full(((B + 1) * D,), YSENT, dtype=torch.float32, device=DEV)
    first_fin = np.full(B, L + 1)
    bfs = []
    for step in range(L):
        d_lg[:B * V] = _dev(lg[:, step].ravel())
        d_y.fill_(YSENT)
        _call(kh, "kh_beam1_step", _p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), L, _p(d_st), _p(d_bf), _p(d_bi), ALPHA, L,
              _p(d_emb), _p(d_pe), L, D, _p(d_y))
        f, st, cur = _np(d_fin), _np(d_st), _np(d_cur)
        assert f[B] == SENT and cur[B] == SENT and ((cur[:B] >= 0) & (cur[:B] < V)).all(), step
        np.testing.assert_array_equal(st, [step + 1, 0, int((f[:B] == 1).all()), SENT])
        first_fin = np.where((f[:B] == 1) & (first_fin > L), step + 1, first_fin)
        b_f = _np(d_bf)
        assert np.isnan(b_f[2 * B:]).all()
        bfs.append(b_f[:2 * B].reshape(B, 2).astype(np.float64))
        y = np.full((B + 1, D), YSENT, np.float32)
        if step + 1 < L:
            y[:B] = emb[cur[:B]] + pe[step + 1]
        _same_bits(f"beam y_next step {step}", _np(d_y).reshape(B + 1, D), y)
    _call(kh, "kh_beam1_finalize", _p(d_tok), B, L, L, _p(d_bi))
    tok = _np(d_tok).reshape(B + 1, L)
    assert (tok[B] == SENT).all()
    b_i = _np(d_bi)
    assert b_i[B] == SENT
    return tok[:B], b_i[:B], first_fin, np.stack(bfs, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1536, 1516, 257, 33])
def test_beam1_step_kernel(kh, V):
    """Every crafted stream alone (B = 1) and all of them as one batch, against BS.beam_search (via beam1_trace, which
    test_beam1_trace_matches_beam_search ties to it): finalized tokens exact, beam_i = the finish length, the step at
    which finished[b] first becomes 1 = the number of logits_fn calls the restatement makes for that element alone, and
    beam_f = {live_lp, finished score} within the fp32 bar of beam1_trace after every step the restatement runs."""
    sc = beam_scenarios(V)
    names = list(sc)
    worst = 0.0
    for batch in [[n] for n in names] + [names]:
        lg = np.stack([sc[n] for n in batch])
        tok, b_i, first_fin, bfs = _run_beam(kh, lg, BEAM_L)
        for b, n in enumerate(batch):
            t = beam1_trace(sc[n], BEAM_L)
            want, _ = BS.beam_search(lambda p, s: sc[n][None, None, s], 1, BEAM_L)
            np.testing.assert_array_equal(tok[b], want[0], err_msg=n)
            assert b_i[b] == t["fin_len"], (n, b_i[b], t["fin_len"])
            assert min(first_fin[b], BEAM_L) == t["calls"], (n, first_fin[b], t["calls"])
            for i, (live, bar_live, fin, bar_fin, _) in enumerate(t["steps"]):
                got_live, got_fin = bfs[b, i]
                assert abs(got_live - live) <= bar_live, (n, i, got_live, live, bar_live)
                assert abs(got_fin - fin) <= bar_fin, (n, i, got_fin, fin, bar_fin)
                worst = max(worst, abs(got_live - live) / bar_live, abs(got_fin - fin) / bar_fin if bar_fin else 0.0)
    print(f"beam_f V={V}: worst err/bar {worst:.3f}")


@pytest.mark.gpu
def test_beam1_step_nan_rows(kh):
    """An all-NaN row continues with id 0 and finishes nothing (the restatement's stable sort); a partly NaN row
    carries no parity claim but every id it emits is in [0, V); a finite row beside them is unaffected."""
    V, L = 300, 5
    sc = beam_scenarios(V)
    lg = np.stack([np.full((L, V), np.nan, np.float32), sc["eos_second_wins"][:L].copy(), sc["eos_first_loses"][:L]])
    lg[1][:, [7, 290]] = np.nan
    tok, b_i, first_fin, _ = _run_beam(kh, lg, L)
    np.testing.assert_array_equal(tok[0], 0)
    assert b_i[0] == 0 and first_fin[0] > L
    assert ((tok[1] >= 0) & (tok[1] < V)).all()
    want, _ = BS.beam_search(lambda p, s: lg[2][None, None, s], 1, L)
    np.testing.assert_array_equal(tok[2], want[0])


# ------------------------------------------------------------------------------------------------
# embed_kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [512, 384, 4])
def test_embed_kernel(kh, D):
    """y[b] = E[clamp(tok[b], 0, V - 1)] + PE[pos] bit for bit, rows b0 .. b0 + n - 1 only."""
    import torch
    V, B, rows = 37, 11, 9
    rng = np.random.default_rng(D)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = _pe_with_guard(rng, rows, D)
    tok = np.array([0, -1, -2147483648, V - 1, V, 2147483647, 5, 1, 36, 17, -5], np.int32)
    d_tok, d_emb, d_pe = _dev(tok), _dev(emb), _dev(pe)
    for b0, n, pos in ((0, B, 0), (3, 6, rows - 1), (10, 1, 4)):
        d_y = torch.full(((B + 1) * D,), float("nan"), dtype=torch.float32, device=DEV)
        d_pos = _dev(np.array([pos], np.int32))
        _call(kh, "kh_embed", _p(d_tok), _p(d_emb), D, V, _p(d_pe), _p(d_pos), _p(d_y), b0, n)
        want = np.full((B + 1, D), np.nan, np.float32)
        want[b0:b0 + n] = emb[np.clip(tok[b0:b0 + n], 0, V - 1)] + pe[pos]
        _same_bits(f"embed b0={b0} n={n} pos={pos}", _np(d_y).reshape(B + 1, D), want)


# ------------------------------------------------------------------------------------------------
# row_rstd_kernel / rmsnorm_kernel
# ------------------------------------------------------------------------------------------------
# rstd = 1/sqrtf(s/D + eps), s = sum x^2 in fp32: each lane sums D/128 float4 groups of 4 squares, then a 5-level warp
# tree -- at most D/32 + 5 roundings of s (relative); x = hi + lo rounded once (2u on each square); the division by D, the
# add of eps, sqrtf and 1/ are correctly rounded (u each).  rstd moves by half the relative error of its argument:
# (D/32 + 5 + 2 + 2) u / 2 + 2u.  y = x * rstd * g adds two roundings.
def _tol_rstd(D):
    return ((D // 32 + 9) / 2 + 2) * U


@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 512])
@pytest.mark.parametrize("M", [1, 7, 9, 300])
@pytest.mark.parametrize("lo", [False, True])
def test_row_rstd_and_rmsnorm(kh, M, D, lo):
    """Against float64, per element |got - ref| <= tol * |ref| (rstd) and tol * |x rstd g| (y), at M not a multiple of
    the 8 rows per CTA, row pitch ld > D (the columns past D hold NaN and must not be read), hi/lo input, and zero rows
    (rstd = 1/sqrt(eps))."""
    import torch
    eps = np.float32(1e-6)
    ld, ldy = D + 20, D + 12
    rng = np.random.default_rng(M * D + lo)
    x = (rng.uniform(-0.5, 1.0, (M, D)) * rng.uniform(0.01, 30, (M, 1))).astype(np.float32)
    x[::5] = 0.0
    g = rng.uniform(0.5, 1.5, D).astype(np.float32)
    xp = np.full((M, ld), np.nan, np.float32)
    lop = np.full((M, ld), np.nan, np.float32)
    if lo:
        hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
        xp[:, :D], lop[:, :D] = hi, x - hi
        assert ((xp[:, :D] + lop[:, :D]) == x).all()
    else:
        xp[:, :D] = x
    d_x, d_lo, d_g = _dev(xp), (_dev(lop) if lo else None), _dev(g)
    d_r = torch.full((M + 3,), float("nan"), dtype=torch.float32, device=DEV)
    d_y = torch.full((M + 1, ldy), float("nan"), dtype=torch.float32, device=DEV)
    _call(kh, "kh_row_rstd", _p(d_x), _p(d_lo), ld, M, D, eps, _p(d_r))
    _call(kh, "kh_rmsnorm", _p(d_x), _p(d_lo), ld, M, D, eps, _p(d_g), _p(d_y), ldy)
    x64 = x.astype(np.float64)
    r64 = 1.0 / np.sqrt((x64 ** 2).mean(1) + float(eps))
    r, y = _np(d_r), _np(d_y)
    assert np.isnan(r[M:]).all() and np.isnan(y[M:]).all() and np.isnan(y[:, D:]).all()
    tol = _tol_rstd(D)
    err_r = np.abs(r[:M] - r64) / (tol * r64)
    yref = x64 * r64[:, None] * g
    err_y = np.abs(y[:M, :D] - yref) / ((tol + 2 * U) * np.abs(yref) + 1e-300)
    print(f"rstd M={M} D={D} lo={lo}: worst err/bar {err_r.max():.3f}; rmsnorm {err_y.max():.3f}")
    assert (err_r <= 1).all(), err_r.max()
    assert (err_y <= 1).all(), err_y.max()


# ------------------------------------------------------------------------------------------------
# the model at max_decode_length = 2048 (the PE table's length)
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("decode", ["greedy", "beam1"])
def test_generate_all_2048_steps(decode):
    """A 1-layer model at max_decode_length = 2048 generates all 2048 steps (its last step is at pos = 2047, the PE
    table's last row); graph replay and plain launches agree."""
    import torch
    from mt3_b200 import network
    from oracle import mt3_oracle as O
    ocfg = O.T5Config(vocab_size=1536, num_encoder_layers=1, num_decoder_layers=1)
    params = O.init_params(ocfg, seed=3)
    cfg = network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=1, num_decoder_layers=1, head_dim=64,
                           mlp_dim=1024, mlp_activations=('gelu', 'linear'))
    L = 2048
    m = network.Transformer(cfg, params, device=DEV, max_batch=2, max_input_length=64, max_decode_length=L)
    audio = np.stack([O.sine_mix(64 * 128, seed=77 + i) for i in range(2)])
    x = torch.from_numpy(O.compute_spectrogram(audio, np.float32)).to(DEV)
    plain = m.generate(x, stop_at_eos=False, use_graph=False, decode=decode).cpu().numpy()
    assert m.last_steps_run == L
    graph = m.generate(x, stop_at_eos=False, use_graph=True, decode=decode).cpu().numpy()
    assert m.last_steps_run == L
    torch.cuda.synchronize()
    np.testing.assert_array_equal(plain, graph)
    assert ((plain >= 0) & (plain < 1536)).all()
