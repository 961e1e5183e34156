"""Temperature sampling (mt3_generate_sampled, Transformer.generate(decode='sample'), predict_batch_with_aux with
decode_fn='temperature_sample' and num_decodes, InferenceModel(decode='sample')).

The library's sampling contract, restated here in numpy (sample_pick_ref) and checked against the kernels:
  * z = logits / temperature, an IEEE float32 division; temperature <= 1e-4 runs the greedy loop unchanged.
  * top-k (0 < topk < V): keep every id whose z is >= the k-th largest z, ties at the k-th value included.
  * top-p (0 < topp < 1), after top-k: keep id i iff the softmax mass of the kept ids with z_j > z_i is below topp -- the
    smallest most-likely set that reaches topp, ties at the boundary kept.
  * next = argmax_i (z_i + g_i) over the kept ids, g_i = -log(-log(u_i)), the first id winning a tie (Gumbel-max: the
    distribution of a categorical draw from the kept softmax).  u_i = (2 (w >> 9) + 1) 2^-24 from Philox4x32-10 with the
    64-bit key, counter (i // 4, pos, r, 0) and word i % 4; r = row0 + b is the row's stream.
  * scores: rescale_log_probs=True: z[next] - logsumexp(kept z); False: logits[next] - logsumexp(logits), greedy's.  The
    sequence score is their sum.
  * greedy's bookkeeping: finished rows emit PAD with score 0, EOS finishes, a NaN row emits its first NaN id and scores
    NaN, forced prompt positions emit the prompt with score 0 and cannot finish.
  * num_decodes = n: input i's samples are rows i n .. i n + n - 1, sorted by sequence score ascending (stable), best last.
Ambiguous picks -- the top two perturbed values within the float32 error of logf / expf, or a top-p cut within the
float32 summation bar of the mass -- are flagged by the restatement and counted, not compared.
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import test_decode_loop_kernels as DK
import test_decode_scores as DS

ROOT = DK.ROOT
DEV = "cuda:0"
U = DK.U
EOS, PAD = 1, 0
_call, _p, _dev, _np, _same_bits = DK._call, DK._p, DK._dev, DK._np, DK._same_bits
MIN_TEMPERATURE = 1e-4
PBAR = 1e-5                 # float32 summation bar of a top-p mass (sums of <= 16 + 8 + 8 positive terms, expf 2 ulp)


# ------------------------------------------------------------------------------------------------
# numpy restatement
# ------------------------------------------------------------------------------------------------
def philox_np(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (broadcast): the four output words"""
    M = np.uint64(0xFFFFFFFF)
    c = [np.asarray(x, np.uint64) & M for x in (c0, c1, c2, c3)]
    k = [np.asarray(k0, np.uint64) & M, np.asarray(k1, np.uint64) & M]
    for r in range(10):
        if r:
            k = [(k[0] + np.uint64(0x9E3779B9)) & M, (k[1] + np.uint64(0xBB67AE85)) & M]
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & M, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & M]
    return [x.astype(np.uint32) for x in c]


def uniforms(key, r, pos, V):
    """u [V] (float64, each exactly a float32) of stream r at position pos"""
    j = np.arange((V + 3) // 4)
    w = np.stack(philox_np(j, pos, r, 0, key[0], key[1]), 1).reshape(-1)[:V]
    return (2.0 * (w >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24


def keep_mask(z, topk, topp, zbar=0.0):
    """kept ids of a NaN-free float32 row z, and two bounds lo <= kept <= hi of the set the kernel can keep: z values off
    by up to zbar move the k-th value, and the float32 sums (PBAR) and those z errors move a top-p mass"""
    z = np.asarray(z, np.float32)
    z64 = z.astype(np.float64)
    V = z.size
    keep = np.ones(V, bool)
    lo, hi = keep.copy(), keep.copy()
    if 0 < topk < V:
        zk = float(np.sort(z)[::-1][topk - 1])
        keep = z >= np.float32(zk)
        lo, hi = keep & (z64 >= zk + 2 * zbar), z64 >= zk - 2 * zbar
    if 0 < topp < 1:
        srt = np.sort(z64[keep])[::-1]
        with np.errstate(invalid="ignore"):
            p = np.exp(srt - srt[0])
        cum = np.concatenate([[0.0], np.cumsum(p / p.sum())])
        mass = cum[np.searchsorted(-srt, -z64, "left")]                  # the kept mass of values above z_i
        bar = PBAR + 4 * zbar
        keep, lo, hi = keep & (mass < topp), lo & (mass < topp - bar), hi & (mass < topp + bar)
    return keep, lo, hi


def sample_pick_ref(l, temperature, topk, topp, key, r, pos, rescale=True, lbar=0.0):
    """One row's pick: (next, score float64, flagged).  lbar: an absolute error bar on the logits (model tests), widening
    the ambiguity of every cut and of the Gumbel comparison."""
    l = np.asarray(l, np.float32)
    V = l.size
    nan = np.isnan(l)
    if nan.any():
        return int(nan.argmax()), math.nan, False
    z = l / np.float32(temperature)
    zbar = lbar / temperature
    keep, lo, hi = keep_mask(z, topk, topp, zbar)
    g = -np.log(-np.log(uniforms(key, r, pos, V)))
    z64 = z.astype(np.float64)
    v = z64 + g
    nxt = int(np.argmax(np.where(keep, v, -np.inf)))
    # the pick is settled when the smallest and the largest set the kernel may keep give it (the kept set lies between
    # them), and no other id of the largest set comes within the float32 error of logf, expf and z
    amb = not lo.any() or int(np.argmax(np.where(lo, v, -np.inf))) != int(np.argmax(np.where(hi, v, -np.inf)))
    err = 8 * U * (1 + np.abs(g) + np.abs(z64)) + 2 * zbar
    others = hi & (np.arange(V) != nxt)
    if others.any():
        amb |= bool((v[nxt] - v[others] <= err[nxt] + err[others]).any())
    if rescale:
        zk = z64[keep]
        m = zk.max()
        score = z64[nxt] - (m + math.log(np.exp(zk - m).sum()))
    else:
        score = float(DS.log_softmax64(l)[nxt])
    return nxt, score, amb


def score_bar(l, temperature, topk, topp, nxt, rescale):
    """float32 error bar of the kernel's token score (block_logsumexp over the masked z row, or over the logits)"""
    l = np.asarray(l, np.float32)
    if not rescale:
        return DS.lp_bar(l, l[nxt])
    z = l / np.float32(temperature)
    keep = keep_mask(z, topk, topp)[0]
    zm = np.where(keep, z, np.float32(-np.inf)).astype(np.float32)
    return DS.lp_bar(zm, z[nxt])


def sample_step_ref(lg, finished, plen, prompt_tok, pos, sp, row0=0):
    """One step of the sampling loop for rows lg [B, V]: (next [B], scores [B], finished', flagged [B])"""
    B = lg.shape[0]
    nxt, sc, flag = np.zeros(B, np.int64), np.zeros(B), np.zeros(B, bool)
    fin = finished.copy()
    for b in range(B):
        t, s, a = sample_pick_ref(lg[b], sp["temperature"], sp["topk"], sp["topp"], sp["key"], row0 + b, pos, sp["rescale"])
        if pos < plen[b]:
            t, s, a = prompt_tok[b], 0.0, False
        elif fin[b]:
            t, s, a = PAD, 0.0, False
        if pos >= plen[b] and t == EOS:
            fin[b] = True
        nxt[b], sc[b], flag[b] = t, s, a
    return nxt, sc, fin, flag


# ------------------------------------------------------------------------------------------------
# CPU: Philox, the restatement, its distribution
# ------------------------------------------------------------------------------------------------
KAT = [  # Random123's published Philox4x32-10 known answers: (counter, key) -> output
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


def test_philox_known_answers():
    for ctr, key, want in KAT:
        got = [int(w) for w in philox_np(*ctr, *key)]
        assert got == list(want), (ctr, key, [hex(x) for x in got])


def test_philox_header_matches_restatement(tmp_path):
    """philox.cuh compiled host-only with g++ gives the restatement's words and uniforms over a sweep of counters and keys"""
    src = tmp_path / "philox_host.cpp"
    src.write_text('#include "philox.cuh"\n'
                   'extern "C" void run(const unsigned* in, int n, unsigned* out, float* u) {\n'
                   '  for (int i = 0; i < n; ++i) {\n'
                   '    const unsigned* a = in + 6 * i;\n'
                   '    mt3::philox4x32_10(a[0], a[1], a[2], a[3], a[4], a[5], out + 4 * i);\n'
                   '    for (int q = 0; q < 4; ++q) u[4 * i + q] = mt3::philox_uniform(out[4 * i + q]);\n'
                   '  }\n'
                   '}\n')
    so = tmp_path / "philox_host.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-I", os.path.join(ROOT, "mt3_b200", "csrc"), "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    lib = C.CDLL(str(so))
    rng = np.random.default_rng(0)
    n = 4096
    inp = rng.integers(0, 2 ** 32, (n, 6), dtype=np.uint64).astype(np.uint32)
    inp[:64, :4] = np.arange(64 * 4, dtype=np.uint32).reshape(64, 4) % 7      # small counters, as the picker uses them
    inp[64:128] = 0xffffffff
    for (ctr, key, _), row in zip(KAT, (0, 64, 200)):
        inp[row] = np.array([*ctr, *key], np.uint32)
    out = np.zeros((n, 4), np.uint32)
    u = np.zeros((n, 4), np.float32)
    lib.run(inp.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p), u.ctypes.data_as(C.c_void_p))
    want = np.stack(philox_np(*inp.T), 1)
    np.testing.assert_array_equal(out, want)
    np.testing.assert_array_equal(out[[0, 64, 200]], np.array([k[2] for k in KAT], np.uint32))
    wu = (2.0 * (want >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24
    np.testing.assert_array_equal(u.astype(np.float64), wu)
    assert (u > 0).all() and (u < 1).all()


def test_keep_mask_crafted_rows():
    """top-k ties at the k-th value, topk = 1, topk >= V, topp 0 and 1, a tie at the top-p boundary"""
    z = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 0.5, 2.0], np.float32)
    np.testing.assert_array_equal(keep_mask(z, 3, 0)[0], z >= 2.0)          # the k-th value 2.0 is tied three ways
    np.testing.assert_array_equal(keep_mask(z, 2, 0)[0], z >= 3.0)
    np.testing.assert_array_equal(keep_mask(z, 1, 0)[0], z >= 3.0)          # topk = 1 keeps both maxima
    for k in (0, 7, 100):
        assert keep_mask(z, k, 0)[0].all()
    for p in (0.0, 1.0):
        assert keep_mask(z, 0, p)[0].all()
    # id 0 alone has mass e / (e + 2) = 0.576; the tie group {1, 2} after it
    z = np.array([1.0, 0.0, 0.0] + [-40.0] * 5, np.float32)
    np.testing.assert_array_equal(keep_mask(z, 0, 0.5)[0], np.arange(8) == 0)
    np.testing.assert_array_equal(keep_mask(z, 0, 0.6)[0], np.arange(8) < 3)   # both tied ids kept, none of the tail
    _, lo, hi = keep_mask(z, 0, math.e / (math.e + 2))                       # a cut exactly at the boundary: both sides
    assert not lo[1:3].any() and hi[1:3].all()
    # top-k before top-p: the kept set's own softmax
    z = np.array([2.0, 1.0, 1.0, 0.0, -1.0], np.float32)
    keep = keep_mask(z, 3, 0.7)[0]
    p = np.exp([2.0, 1.0, 1.0]) / np.exp([2.0, 1.0, 1.0]).sum()
    assert p[0] < 0.7 and keep[:3].all() and not keep[3:].any()


def test_sample_pick_ref_bookkeeping():
    """NaN rows, finished rows, forced positions, EOS finishing, and rescale on / off scores"""
    V = 40
    rng = np.random.default_rng(1)
    lg = rng.standard_normal((5, V)).astype(np.float32)
    lg[1, [7, 30]] = np.nan
    lg[3, EOS] = 60.0
    sp = {"temperature": 1.0, "topk": 0, "topp": 0.0, "key": (3, 4), "rescale": True}
    nxt, sc, fin, _ = sample_step_ref(lg, np.array([False, False, True, False, False]), np.array([0, 0, 0, 0, 9]),
                                      np.array([0, 0, 0, 0, 17]), 2, sp)
    assert nxt[1] == 7 and np.isnan(sc[1])
    assert nxt[2] == PAD and sc[2] == 0 and fin[2]
    assert nxt[3] == EOS and fin[3] and abs(sc[3]) < 1e-12
    assert nxt[4] == 17 and sc[4] == 0 and not fin[4]
    t, s1, _ = sample_pick_ref(lg[0], 2.0, 5, 0.0, (1, 2), 0, 0, rescale=True)
    _, s0, _ = sample_pick_ref(lg[0], 2.0, 5, 0.0, (1, 2), 0, 0, rescale=False)
    assert s0 == pytest.approx(DS.log_softmax64(lg[0])[t], abs=1e-12)
    z = (lg[0] / np.float32(2.0)).astype(np.float64)
    zk = np.sort(z)[::-1][:5]
    assert s1 == pytest.approx(z[t] - (zk.max() + np.log(np.exp(zk - zk.max()).sum())), abs=1e-12)


def _chi2_p(counts, probs):
    from scipy import stats
    exp = probs * counts.sum()
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    e = np.append(exp[big], exp[~big].sum())
    if e[-1] == 0:
        assert obs[-1] == 0
        obs, e = obs[:-1], e[:-1]
    return stats.chisquare(obs, e).pvalue


def kept_softmax(l, temperature, topk, topp):
    z = np.asarray(l, np.float32) / np.float32(temperature)
    keep = keep_mask(z, topk, topp)[0]
    p = np.where(keep, np.exp(z.astype(np.float64) - z[keep].max()), 0.0)
    return p / p.sum()


def test_restatement_distribution():
    """With a fixed key, over 2e5 (stream, position) counters, the restatement's draws from one row follow the kept-set
    softmax (chi-square); dropped ids are never drawn."""
    V, n = 48, 200_000
    rng = np.random.default_rng(5)
    l = (rng.standard_normal(V) * 1.5).astype(np.float32)
    key = (0x12345678, 0x9abcdef0)
    rs, ps = np.divmod(np.arange(n), 1000)
    j = np.arange(V // 4)
    w = np.stack(philox_np(j[None, :], ps[:, None], rs[:, None], 0, *key), 2).reshape(n, V)
    g = -np.log(-np.log((2.0 * (w >> np.uint32(9)).astype(np.float64) + 1.0) * 2.0 ** -24))
    for T, k, p in ((1.0, 0, 0.0), (0.7, 10, 0.0), (1.3, 0, 0.9), (1.0, 20, 0.8)):
        z = (l / np.float32(T)).astype(np.float64)
        keep = keep_mask(l / np.float32(T), k, p)[0]
        draws = np.argmax(np.where(keep, z + g, -np.inf), 1)
        for q in range(5):                               # the vectorised draw is sample_pick_ref's
            assert draws[q] == sample_pick_ref(l, T, k, p, key, rs[q], ps[q])[0]
        counts = np.bincount(draws, minlength=V)
        probs = kept_softmax(l, T, k, p)
        assert (counts[probs == 0] == 0).all()
        assert _chi2_p(counts, probs) > 1e-4, (T, k, p)


# ------------------------------------------------------------------------------------------------
# CPU: the wrappers and the ABI
# ------------------------------------------------------------------------------------------------
class _SampleModule:
    """generate stand-in: scores from a table keyed by (row_offset + row), tokens [row id, stream]"""
    def __init__(self, scores):
        self.scores, self.calls = scores, []

    def generate(self, x, stop_at_eos=True, decode='greedy', return_scores=False, prompt=None, seed=0, row_offset=0,
                 temperature=1.0, topk=0, topp=0.0):
        import torch
        self.calls.append(dict(shape=tuple(x.shape), decode=decode, seed=seed, row_offset=row_offset, temperature=temperature,
                               topk=topk, topp=topp, prompt=None if prompt is None else np.array(prompt), x=np.asarray(x) if isinstance(x, np.ndarray) else x.numpy()))
        B = x.shape[0]
        toks = torch.zeros((B, 4), dtype=torch.int32)
        toks[:, 0] = torch.as_tensor(np.asarray(x)[:, 0, 0]).to(torch.int32)     # which input the row holds
        toks[:, 1] = torch.arange(B, dtype=torch.int32) + row_offset            # which stream
        sc = torch.as_tensor(self.scores[row_offset:row_offset + B], dtype=torch.float32)
        return (toks, torch.zeros((B, 4)), sc) if return_scores else toks


def test_temperature_sample_wrapper():
    """decode_fn='temperature_sample': the arguments reach generate, inputs are expanded with repeat_interleave (input i's
    samples are rows i n .. i n + n - 1, streams i n + k), the decodes come back sorted ascending (stable) with the best
    last, shapes with and without return_all_decodes; rng forms; the existing decode_fns keep their contracts."""
    import torch
    from mt3_b200 import models
    B, n = 3, 4
    x = np.zeros((B, 5, 4), np.float32)
    x[:, 0, 0] = [10, 11, 12]
    scores = np.array([0.5, -1.0, 0.5, -3.0, 2.0, 2.0, 1.0, -2.0, 0.0, 0.0, 0.0, 0.0], np.float32)
    mod = _SampleModule(scores)
    m = models.ContinuousInputsEncoderDecoderModel(mod, input_depth=4, decode_fn='temperature_sample')
    toks, aux = m.predict_batch_with_aux(None, {'encoder_input_tokens': x}, rng=np.array([0, 7], np.uint32),
                                         decoder_params={'temperature': 0.8, 'topk': 40}, num_decodes=n, return_all_decodes=True)
    c = mod.calls[-1]
    assert c['shape'] == (B * n, 5, 4) and c['decode'] == 'sample' and c['row_offset'] == 0
    assert c['temperature'] == 0.8 and c['topk'] == 40 and c['topp'] == 0.0
    np.testing.assert_array_equal(np.asarray(c['seed']), [0, 7])
    np.testing.assert_array_equal(c['x'][:, 0, 0], np.repeat([10, 11, 12], n))
    assert toks.shape == (B, n, 4) and aux['scores'].shape == (B, n)
    for i in range(B):
        sc = scores[i * n:(i + 1) * n]
        order = np.argsort(sc, kind="stable")
        np.testing.assert_array_equal(aux['scores'][i].numpy(), sc[order])
        np.testing.assert_array_equal(toks[i, :, 1].numpy(), i * n + order)          # the streams, ties in decode order
        assert (toks[i, :, 0].numpy() == 10 + i).all()
    best, aux1 = m.predict_batch_with_aux(None, {'encoder_input_tokens': torch.from_numpy(x)}, rng=5, num_decodes=n)
    assert best.shape == (B, 4) and aux1['scores'].shape == (B,)
    np.testing.assert_array_equal(best.numpy(), toks[:, -1].numpy())
    assert mod.calls[-1]['seed'] == 5
    # num_decodes = 1: no expansion; the key from decoder_params; no key at all is key 0
    _, aux = m.predict_batch_with_aux(None, {'encoder_input_tokens': x}, decoder_params={'decode_rng': 9, 'topp': 0.9})
    assert mod.calls[-1]['seed'] == 9 and mod.calls[-1]['topp'] == 0.9 and mod.calls[-1]['shape'] == (B, 5, 4)
    m.predict_batch(None, {'encoder_input_tokens': x})
    assert mod.calls[-1]['seed'] == 0 and mod.calls[-1]['decode'] == 'sample'
    with pytest.raises(ValueError, match="not both"):
        m.predict_batch_with_aux(None, {'encoder_input_tokens': x}, rng=1, decoder_params={'decode_rng': 2})
    with pytest.raises(ValueError):
        m.predict_batch_with_aux(None, {'encoder_input_tokens': x}, decoder_params={'temprature': 1.0})
    with pytest.raises(ValueError):
        m.predict_batch_with_aux(None, {'encoder_input_tokens': x}, num_decodes=0)
    # prompts are expanded with their inputs
    din = np.array([[0, 5, 0], [0, 6, 7], [0, 0, 0]], np.int32)
    m.predict_batch_with_aux(None, {'encoder_input_tokens': x, 'decoder_input_tokens': din}, num_decodes=2, prompt_with_targets=True)
    np.testing.assert_array_equal(mod.calls[-1]['prompt'], np.repeat(din[:, 1:], 2, axis=0))
    for fn in ('beam_search', 'greedy'):
        d = models.ContinuousInputsEncoderDecoderModel(mod, input_depth=4, decode_fn=fn)
        with pytest.raises(ValueError):
            d.predict_batch_with_aux(None, {'encoder_input_tokens': x}, num_decodes=2)
        with pytest.raises(ValueError):
            d.predict_batch_with_aux(None, {'encoder_input_tokens': x}, decoder_params={'decode_rng': 1})
    with pytest.raises(ValueError):
        models.ContinuousInputsEncoderDecoderModel(mod, decode_fn='sample')


def test_sample_key_and_host_checks():
    """seed forms (int -> jax.random.PRNGKey's words, two uint32 words as they are) and the host-side argument checks"""
    import torch
    from mt3_b200 import network
    assert network.sample_key(0) == (0, 0)
    assert network.sample_key(7) == (0, 7)
    assert network.sample_key((5 << 32) | 9) == (5, 9)
    assert network.sample_key(np.array([3, 4], np.uint32)) == (3, 4)
    assert network.sample_key(torch.tensor([1, 2], dtype=torch.int64)) == (1, 2)
    for bad in (-1, 2 ** 64, [1, 2, 3], np.array([1.0, 2.0]), [2 ** 32, 0]):
        with pytest.raises(ValueError):
            network.sample_key(bad)
    t = object.__new__(network.Transformer)
    t.config = network.T5Config(vocab_size=1536)
    sp = t._sample_params(0.5, 40, 0.9, 11, 3, False, 8)
    assert (sp.temperature, sp.topk, sp.topp, list(sp.key), sp.row0, sp.rescale_log_probs) == (0.5, 40, pytest.approx(0.9), [0, 11], 3, 0)
    for kw in ({'temperature': -1.0}, {'temperature': float('inf')}, {'temperature': float('nan')}, {'topk': -1}, {'topk': 1.5},
               {'topp': 1.5}, {'topp': float('nan')}, {'row_offset': -1}):
        args = dict(temperature=1.0, topk=0, topp=0.0, seed=0, row_offset=0, rescale_log_probs=True, batch=4)
        args.update(kw)
        with pytest.raises(ValueError):
            t._sample_params(**args)
    t.config = network.T5Config(vocab_size=5000)
    t._sample_params(1.0, 0, 0.0, 0, 0, True, 4)                      # no filter: any vocabulary
    with pytest.raises(ValueError, match="vocab"):
        t._sample_params(1.0, 10, 0.0, 0, 0, True, 4)


def test_inference_model_seed_and_streams(monkeypatch):
    """InferenceModel(decode='sample'): predict_tokens passes its seed; transcribe_segments_sharded gives each shard its
    first global segment index as the stream offset"""
    import torch
    from mt3_b200 import distributed, inference
    im = object.__new__(inference.InferenceModel)
    im.decode, im.sample_params = 'sample', {'temperature': 0.9, 'topk': 5}
    assert im._sample_kw(4, 16) == {'temperature': 0.9, 'topk': 5, 'seed': 4, 'row_offset': 16}
    im.decode = 'greedy'
    assert im._sample_kw(4, 16) == {}
    im.decode = 'sample'
    seen = []

    class _M:
        def generate(self, x, **kw):
            seen.append(kw)
            return torch.full((x.shape[0], 3), 5, dtype=torch.int32)

    class _Voc:
        def decode_tf(self, t):
            return t
    im.model, im.vocabulary, im.use_graph, im.device = _M(), _Voc(), True, torch.device("cpu")
    im.predict_tokens({'encoder_input_tokens': np.zeros((2, 4, 3), np.float32)}, seed=77)
    assert seen[-1]['seed'] == 77 and seen[-1]['row_offset'] == 0 and seen[-1]['decode'] == 'sample'
    calls = []
    im.outputs_length = 3
    monkeypatch.setattr(im, 'transcribe_segments', lambda a, **kw: calls.append(kw) or np.zeros((a.shape[0], 3), np.int32),
                        raising=False)
    monkeypatch.setattr(distributed, 'world', lambda: (1, 2))
    monkeypatch.setattr(distributed, 'gather_tokens', lambda t, S: torch.zeros((S, t.shape[1]), dtype=t.dtype))
    im.transcribe_segments_sharded(np.zeros((7, 8), np.float32), seed=3)
    lo, _ = distributed.shard_range(7, 1, 2)
    assert calls[-1]['segment_offset'] == lo and calls[-1]['seed'] == 3
    with pytest.raises(ValueError):
        inference.InferenceModel.__init__(object.__new__(inference.InferenceModel), 'synthetic', sample_params={'tempreature': 1})


def test_abi_sampled_entry_point():
    """mt3_generate_sampled is exported, MT3_GEN_SAMPLE and mt3_sample_params match the header, and a NULL handle is
    MT3_ERR_BAD_ARG without a device"""
    import re
    from mt3_b200 import _lib
    header = open(os.path.join(ROOT, "include", "mt3_b200.h")).read()
    assert int(re.search(r"MT3_GEN_SAMPLE\s*=\s*(\d+)", header).group(1)) == _lib.GEN_SAMPLE
    body = re.search(r"typedef struct mt3_sample_params \{(.*?)\}", header, re.S).group(1)
    fields = re.findall(r"\b(float|int32_t|uint32_t)\s+(\w+)(\[2\])?;", body)
    assert [f[1] for f in fields] == [f[0] for f in _lib.SampleParams._fields_]
    assert C.sizeof(_lib.SampleParams) == 28
    lib = _lib.load()
    assert "mt3_generate_sampled" in _lib.EXPORTS and hasattr(lib, "mt3_generate_sampled")
    sp = _lib.SampleParams()
    sp.temperature = 1.0
    assert lib.mt3_generate_sampled(None, None, 1, _lib.GEN_SAMPLE, None, 0, None, None, None, None, None, 0, C.byref(sp), None) == -1


# ------------------------------------------------------------------------------------------------
# GPU: sample_step_kernel alone (libmt3kernels.so)
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
    lib.kh_last_error.argtypes, lib.kh_last_error.restype = [], C.c_char_p
    lib.kh_sample_step.argtypes = [P, I, I, P, P, P, P, I, P, P, P, I, F, P, P, I, I, P]
    lib.kh_sample_step.restype = I
    return lib


def _sp_dev(sp, row0=0):
    """mt3_sample_params on the device"""
    w = np.zeros(7, np.uint32)
    w[0] = np.float32(sp["temperature"]).view(np.uint32)
    w[1] = np.uint32(sp["topk"])
    w[2] = np.float32(sp["topp"]).view(np.uint32)
    w[3], w[4] = sp["key"]
    w[5], w[6] = row0, int(sp["rescale"])
    return _dev(w)


def _crafted_sample_rows(V, rng):
    """rows where a sampler goes wrong: ties across threads and warps and at the k-th value, a tie at the top-p boundary,
    NaN rows, denormals and signed zeros, EOS on top"""
    rows = []
    x = (rng.standard_normal(V) * 0.1 - 5).astype(np.float32)
    for i in (3, min(259, V - 2), V // 2, V - 1):
        x[i] = 4.0                                          # a four-way tie on top, over lanes / warps
    x[V // 3] = 3.0
    rows.append(x)
    x = np.full(V, -30.0, np.float32)
    x[10], x[V // 2], x[V // 2 + 1] = 1.0, 0.0, 0.0        # top-p boundary tie: mass(id 10) = e / (e + 2)
    rows.append(x)
    rows.append(np.zeros(V, np.float32))                    # all equal: the Gumbel numbers alone decide
    x = rng.standard_normal(V).astype(np.float32)
    x[[V // 5, V - 3]] = np.nan
    rows.append(x)
    rows.append(np.full(V, np.nan, np.float32))
    x = (rng.standard_normal(V) * 1e-39).astype(np.float32)     # denormals and signed zeros
    x[::7] = -0.0
    x[1::7] = 0.0
    rows.append(x)
    x = rng.standard_normal(V).astype(np.float32)
    x[EOS] = 30.0
    rows.append(x)
    x = (rng.standard_normal(V) * 3).astype(np.float32)
    x[0] = x.max() + 1                                      # the maximum at id 0 and at id V - 1
    rows.append(x)
    x = (rng.standard_normal(V) * 3).astype(np.float32)
    x[V - 1] = x.max() + 1
    rows.append(x)
    return rows


KERNEL_CONFIGS = [
    # temperature, topk, topp, rescale
    (1.0, 0, 0.0, True), (1.0, 0, 0.0, False), (0.7, 40, 0.0, True), (1.3, 0, 0.9, True), (1.0, 20, 0.8, True),
    (1.0, 2, 0.0, True), (1.0, 1, 0.0, True), (1.0, 5000, 0.0, True), (1.0, 0, 0.6, True), (1e-3, 0, 0.0, True),
    (10.0, 0, 0.5, True), (10.0, 3, 0.0, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("V", [200, 1536, 1664])
def test_sample_step_kernel(kh, V):
    """One sample_step_kernel launch per configuration on crafted and random rows, B = 40, with finished rows and forced
    prompt positions: tokens, finished, state, tok_cur and y_next (bit for bit) equal the restatement outside flagged picks,
    padding rows stay sentinels, scores lie within their bar."""
    import torch
    rng = np.random.default_rng(V)
    B, D, L = 40, 64, 12
    pos = 6
    crafted = _crafted_sample_rows(V, rng)
    emb = rng.standard_normal((V, D)).astype(np.float32)
    pe = DK._pe_with_guard(rng, L, D)
    d_emb, d_pe = _dev(emb), _dev(pe)
    flagged = total = 0
    for ci, (T, k, p, rescale) in enumerate(KERNEL_CONFIGS):
        sp = {"temperature": T, "topk": k, "topp": p, "key": (0xC0FFEE + ci, 77), "rescale": rescale}
        lg = (rng.standard_normal((B, V)) * 2).astype(np.float32)
        for i, row in enumerate(crafted):
            lg[i] = row
        fin0 = np.zeros(B, bool)
        fin0[[20, 33]] = True
        plen = np.zeros(B, np.int32)
        plen[[21, 34]] = pos + 1
        tok = np.full((B + 1, L), DK.SENT, np.int32)
        tok[21, pos], tok[34, pos] = 5, V - 1
        row0 = 1000 * ci
        d_lg = _dev(np.concatenate([lg.ravel(), np.full(V, np.nan, np.float32)]))
        d_cur = _dev(np.full(B + 1, DK.SENT, np.int32))
        d_fin = _dev(np.append(fin0.astype(np.int32), DK.SENT).astype(np.int32))
        d_tok = _dev(tok.copy())
        d_ts = torch.full(((B + 1) * L,), -5.0, dtype=torch.float32, device=DEV)
        d_pl = _dev(plen)
        d_st = _dev(np.array([pos, 0, 0, DK.SENT], np.int32))
        d_y = torch.full(((B + 1) * D,), DK.YSENT, dtype=torch.float32, device=DEV)
        _call(kh, "kh_sample_step", _p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), _p(d_ts), L, _p(d_pl), _p(d_st), _p(_sp_dev(sp, row0)),
              k, p, _p(d_emb), _p(d_pe), L, D, _p(d_y))
        nxt, sc, fin, flag = sample_step_ref(lg, fin0, plen, tok[:B, pos], pos, sp, row0)
        got = _np(d_tok).reshape(B + 1, L)
        ok = ~flag
        flagged += int(flag.sum())
        total += B
        np.testing.assert_array_equal(got[:B, pos][ok], nxt[ok], err_msg=f"V={V} config {ci}")
        want_tok = tok.copy()
        want_tok[:B, pos] = got[:B, pos]
        np.testing.assert_array_equal(got, want_tok, err_msg=f"V={V} config {ci}: outside column {pos}")
        t = got[:B, pos]
        assert ((t >= 0) & (t < V)).all()
        np.testing.assert_array_equal(_np(d_cur), np.append(t, DK.SENT))
        fin_got = _np(d_fin)
        assert fin_got[B] == DK.SENT
        np.testing.assert_array_equal(fin_got[:B][ok].astype(bool), fin[ok])
        np.testing.assert_array_equal(_np(d_st), [pos + 1, 0, int(fin_got[:B].all()), DK.SENT])
        y = np.full((B + 1, D), DK.YSENT, np.float32)
        y[:B] = emb[t] + pe[pos + 1]
        _same_bits(f"V={V} config {ci}: y_next", _np(d_y).reshape(B + 1, D), y)
        ts = _np(d_ts).reshape(B + 1, L)
        assert (ts[B] == -5.0).all() and (np.delete(ts[:B], pos, 1) == -5.0).all()
        for b in range(B):
            if not ok[b]:
                continue
            if fin0[b] or pos < plen[b]:
                assert ts[b, pos] == 0.0, (ci, b)
            elif np.isnan(sc[b]):
                assert np.isnan(ts[b, pos]), (ci, b)
            else:
                bar = score_bar(lg[b], T, k, p, nxt[b], rescale)
                assert abs(ts[b, pos] - sc[b]) <= bar, (ci, b, ts[b, pos], sc[b], bar)
    print(f"V={V}: {flagged} of {total} picks flagged")
    assert flagged <= total // 20


@pytest.mark.gpu
def test_sample_step_kernel_refuses_filters_past_sort_limit(kh):
    """top-k / top-p at V > 4096 are MT3_ERR_UNSUPPORTED; unfiltered sampling runs there"""
    import torch
    V, B = 5000, 2
    d_lg = _dev(np.zeros(B * V, np.float32))
    d_cur, d_fin, d_tok = _dev(np.zeros(B, np.int32)), _dev(np.zeros(B, np.int32)), _dev(np.zeros(B * 4, np.int32))
    d_st = _dev(np.zeros(4, np.int32))
    for k, p, want in ((10, 0.0, -3), (0, 0.5, -3), (0, 0.0, 0), (V, 1.0, 0)):
        sp = _sp_dev({"temperature": 1.0, "topk": k, "topp": p, "key": (1, 2), "rescale": True})
        r = kh.kh_sample_step(_p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), None, 4, None, _p(d_st), _p(sp), k, p, None, None, 0, 0, None)
        torch.cuda.synchronize()
        assert r == want, (k, p, r)


DIST_CONFIGS = [(1.0, 0, 0.0), (0.7, 40, 0.0), (1.3, 0, 0.9), (1.0, 20, 0.8)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", DIST_CONFIGS, ids=[f"T{t}-k{k}-p{p}" for t, k, p in DIST_CONFIGS])
def test_sample_step_kernel_distribution(kh, cfg):
    """One row replicated over B = 64 rows and 1600 positions (102400 draws, fixed key): the kernel's draws follow the
    kept-set softmax (chi-square), never a dropped id, and equal the restatement at a sample of (row, position) pairs."""
    import torch
    T, k, p = cfg
    V, B, P = 1536, 64, 1600
    rng = np.random.default_rng(11)
    l = (rng.standard_normal(V) * 1.5).astype(np.float32)
    l[EOS] = -np.inf                                        # no row finishes
    sp = {"temperature": T, "topk": k, "topp": p, "key": (0xDEADBEEF, 0x5EED), "rescale": True}
    d_lg = _dev(np.tile(l, B))
    d_cur, d_fin = _dev(np.zeros(B, np.int32)), _dev(np.zeros(B, np.int32))
    d_tok = torch.zeros((B * P,), dtype=torch.int32, device=DEV)
    d_st = _dev(np.zeros(4, np.int32))
    d_sp = _sp_dev(sp)
    for _ in range(P):
        r = kh.kh_sample_step(_p(d_lg), V, B, _p(d_cur), _p(d_fin), _p(d_tok), None, P, None, _p(d_st), _p(d_sp), k, p, None, None, 0, 0,
                              None)
        assert r == 0, kh.kh_last_error().decode()
    torch.cuda.synchronize()
    draws = _np(d_tok).reshape(B, P)
    assert _np(d_st)[0] == P
    probs = kept_softmax(l, T, k, p)
    counts = np.bincount(draws.ravel(), minlength=V)
    assert (counts[probs == 0] == 0).all()
    pv = _chi2_p(counts, probs)
    print(f"T={T} k={k} p={p}: chi-square p = {pv:.3g}, {int((probs > 0).sum())} kept ids")
    assert pv > 1e-4
    for b, q in zip(rng.integers(0, B, 40), rng.integers(0, P, 40)):
        t, _, amb = sample_pick_ref(l, T, k, p, sp["key"], b, q)
        assert amb or draws[b, q] == t, (b, q)


# ------------------------------------------------------------------------------------------------
# GPU: the model
# ------------------------------------------------------------------------------------------------
_CFG = {"mt3": (64, 1536), "ismir2021": (512, 1664)}
_L, _B = 40, 8
_ORACLE = {}


def _params(config):
    import test_gpu_parity as GP
    from oracle import mt3_oracle as O
    return GP._eos_params(O.T5Config(vocab_size=_CFG[config][1], num_encoder_layers=2, num_decoder_layers=2), seed=9, boost=4.0)


def _model(config, gm, kv):
    import test_gpu_parity as GP
    from mt3_b200 import network
    T, V = _CFG[config]
    return network.Transformer(GP._mt3_cfg(vocab_size=V, num_encoder_layers=2, num_decoder_layers=2), _params(config), device=DEV,
                               max_batch=_B, max_input_length=T, max_decode_length=_L, gemm_mode=gm, kv_format=kv)


def _inputs(config):
    import test_gpu_parity as GP
    return GP._inputs(_B, t=_CFG[config][0], seed=50)


def _oracle_along(config, x, tok):
    """float64 and float32 oracle logits [B, L, V] with the sampled rows teacher-forced as decoder inputs"""
    from oracle import mt3_oracle as O
    ocfg = O.T5Config(vocab_size=_CFG[config][1], num_encoder_layers=2, num_decoder_layers=2)
    params = _params(config)
    fed = np.concatenate([np.zeros((x.shape[0], 1), np.int64), tok[:, :-1]], 1)
    out = []
    for dt in (np.float64, np.float32):
        _, lg = O.greedy_decode(params, ocfg, O.encode(params, ocfg, x, dt), _L, dt, stop_at_eos=False, return_logits=True,
                                forced_tokens=fed)
        out.append(np.asarray(lg, np.float64))
    return out


def _check_against_oracle(config, x, tok, ts, sp, plen=None, prompt=None, tag=""):
    """Every free position up to a row's first EOS: the restatement fed the float64 logits picks the sampled token unless
    it flags the position; token scores within twice max(4 e_f32, 2e-5) of max |logit| (scaled by 1 / T with rescale).
    Returns the flags [B, L]."""
    l64, l32 = _oracle_along(config, x, tok)
    scale = np.abs(l64).max()
    e_f32 = np.abs(l32 - l64).max() / scale
    bar = max(4 * e_f32, 2e-5) * scale
    B = tok.shape[0]
    plen = np.zeros(B, np.int64) if plen is None else plen
    flags = np.zeros(tok.shape, bool)
    checked = 0
    for b in range(B):
        for i in range(_L):
            if i < plen[b]:
                assert tok[b, i] == prompt[b, i] and ts[b, i] == 0.0
                continue
            if i > 0 and (tok[b, :i] == EOS).any():
                assert tok[b, i] == PAD and ts[b, i] == 0.0
                continue
            t, s, amb = sample_pick_ref(l64[b, i].astype(np.float32), sp["temperature"], sp["topk"], sp["topp"], sp["key"],
                                        b, i, sp["rescale"], lbar=bar)
            flags[b, i] = amb
            if amb:
                continue
            checked += 1
            assert tok[b, i] == t, (tag, b, i, tok[b, i], t)
            want = sample_pick_ref(l64[b, i], sp["temperature"], sp["topk"], sp["topp"], sp["key"], b, i, sp["rescale"])[1]
            # the sampled token is rarely the row's maximum, so its logit's error and the log-sum-exp's do not cancel
            sbar = 2 * bar / (sp["temperature"] if sp["rescale"] else 1.0)
            assert abs(ts[b, i] - want) <= sbar, (tag, b, i, ts[b, i], want, sbar)
    print(f"{tag}: {checked} positions checked, {int(flags.sum())} flagged, logit bar {bar:.2e}")
    assert checked >= B * 4
    return flags


SAMPLE_CASES = {"T1": (1.0, 0, 0.0, True), "T0.7-k40": (0.7, 40, 0.0, True), "T1.3-p0.9": (1.3, 0, 0.9, True),
                "T1-k20-p0.8-raw": (1.0, 20, 0.8, False)}
MODEL_CASES = ([("mt3-simt-f32", c) for c in SAMPLE_CASES] + [("mt3-tf32x3-p24", c) for c in SAMPLE_CASES]
               + [("ismir2021-tf32x3-f32", "T1"), ("ismir2021-tf32x3-f32", "T1-k20-p0.8-raw"), ("ismir2021-tf32x3-p24", "T0.7-k40"),
                  ("ismir2021-tf32x3-p24", "T1.3-p0.9")])


@pytest.mark.gpu
@pytest.mark.parametrize("mode,case", MODEL_CASES)
def test_sampled_generate_against_float64(mode, case):
    """mt3_generate_sampled on the 2-layer models (EOS-boosted weights, B = 8, 40 steps), its rows teacher-forced through the
    float64 oracle: each unflagged position picks the restatement's token from the oracle's logits and the same Philox
    words, its score within 2 max(4 e_f32, 2e-5) max |logit| / T; graph replay equals plain launches bit for bit."""
    import torch
    from mt3_b200 import _lib
    config, gm, kv = mode.split("-")
    gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3}[gm]
    kv = {"f32": _lib.KV_F32, "p24": _lib.KV_P24}[kv]
    T, k, p, rescale = SAMPLE_CASES[case]
    sp = {"temperature": T, "topk": k, "topp": p, "key": (0, 1234), "rescale": rescale}
    m = _model(config, gm, kv)
    x = _inputs(config)
    xg = torch.from_numpy(x).to(DEV)
    kw = dict(num_steps=_L, stop_at_eos=False, decode='sample', return_scores=True, temperature=T, topk=k, topp=p, seed=1234,
              rescale_log_probs=rescale)
    tok, ts, sc = (t.cpu().numpy() for t in m.generate(xg, **kw))
    plain = [t.cpu().numpy() for t in m.generate(xg, use_graph=False, **kw)]
    np.testing.assert_array_equal(plain[0], tok)
    _same_bits(f"{mode} {case}: token scores, graph vs plain", plain[1], ts)
    _same_bits(f"{mode} {case}: scores, graph vs plain", plain[2], sc)
    np.testing.assert_allclose(sc, ts.astype(np.float64).sum(1), rtol=1e-5, atol=1e-4)
    _check_against_oracle(config, x, tok, ts, sp, tag=f"{mode} {case}")


@pytest.mark.gpu
def test_sampled_generate_determinism_and_isolation():
    """Same key: bit-identical tokens and scores with graphs on and off, with num_steps = 37 (not a multiple of 16), on
    repeated calls and under stop_at_eos; another key changes the tokens.  temperature <= 1e-4 equals greedy bit for bit.
    Greedy and beam1 after sampled calls equal a fresh model's bit for bit."""
    import torch
    from mt3_b200 import _lib
    x = torch.from_numpy(_inputs("mt3")).to(DEV)
    m = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    fresh = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    ref = {d: [t.cpu().numpy() for t in fresh.generate(x, num_steps=_L, stop_at_eos=False, decode=d, return_scores=True)]
           for d in ("greedy", "beam1")}
    kw = dict(decode='sample', return_scores=True, temperature=1.0, topk=40, seed=77)
    for steps in (_L, 37):
        runs = [[t.cpu().numpy() for t in m.generate(x, num_steps=steps, stop_at_eos=False, use_graph=g, **kw)]
                for g in (True, False, True)]
        for r in runs[1:]:
            np.testing.assert_array_equal(r[0], runs[0][0])
            _same_bits(f"steps {steps}: token scores", r[1], runs[0][1])
            _same_bits(f"steps {steps}: scores", r[2], runs[0][2])
        if steps == _L:
            full = runs[0]
    stopped = [t.cpu().numpy() for t in m.generate(x, num_steps=_L, stop_at_eos=True, **kw)]
    ran = m.last_steps_run
    np.testing.assert_array_equal(stopped[0][:, :ran], full[0][:, :ran])
    _same_bits("stop_at_eos: token scores", stopped[1][:, :ran], full[1][:, :ran])
    if ran < _L:
        assert ((full[0][:, :ran] == EOS).any(1)).all()
    other = m.generate(x, num_steps=_L, stop_at_eos=False, **dict(kw, seed=78))[0].cpu().numpy()
    assert (other != full[0]).any()
    # a different row_offset is a different stream for every row
    shifted = m.generate(x, num_steps=_L, stop_at_eos=False, row_offset=1, **kw)[0].cpu().numpy()
    assert (shifted != full[0]).any()
    for T in (1e-4, 0.0):
        cold = [t.cpu().numpy() for t in m.generate(x, num_steps=_L, stop_at_eos=False, **dict(kw, temperature=T))]
        np.testing.assert_array_equal(cold[0], ref["greedy"][0])
        _same_bits(f"T={T}: token scores vs greedy", cold[1], ref["greedy"][1])
        _same_bits(f"T={T}: scores vs greedy", cold[2], ref["greedy"][2])
    for d in ("greedy", "beam1"):
        got = [t.cpu().numpy() for t in m.generate(x, num_steps=_L, stop_at_eos=False, decode=d, return_scores=True)]
        np.testing.assert_array_equal(got[0], ref[d][0])
        _same_bits(f"{d} after sampling: token scores", got[1], ref[d][1])
        _same_bits(f"{d} after sampling: scores", got[2], ref[d][2])


@pytest.mark.gpu
def test_sampled_generate_error_codes():
    """NULL params with MT3_GEN_SAMPLE, MT3_GEN_SAMPLE | MT3_GEN_BEAM1, bad temperature / topk / topp: MT3_ERR_BAD_ARG;
    the host raises ValueError first"""
    import torch
    from mt3_b200 import _lib
    m = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    x = torch.from_numpy(_inputs("mt3")).to(DEV)
    m.generate(x, num_steps=1)
    out = torch.empty((_B, _L), dtype=torch.int32, device=DEV)
    ran = C.c_int32(0)

    def call(flags, sp):
        return m._lib.mt3_generate_sampled(m._h, x.data_ptr(), _L, flags, None, 0, out.data_ptr(), None, None, C.byref(ran), None, 0,
                                           None if sp is None else C.byref(sp), m._stream())
    good = _lib.SampleParams()
    good.temperature = 1.0
    assert call(_lib.GEN_SAMPLE, None) == -1
    assert call(_lib.GEN_SAMPLE | _lib.GEN_BEAM1, good) == -1
    for field, val in (("temperature", float("nan")), ("temperature", -0.5), ("temperature", float("inf")), ("topk", -2),
                       ("topp", 1.5), ("topp", float("nan")), ("topp", -0.1)):
        bad = _lib.SampleParams()
        bad.temperature = 1.0
        setattr(bad, field, val)
        assert call(_lib.GEN_SAMPLE, bad) == -1, (field, val)
    assert call(_lib.GEN_SAMPLE, good) == 0 and ran.value == _L
    with pytest.raises(ValueError):
        m.generate(x, decode='sample', temperature=-1.0)


@pytest.mark.gpu
def test_sampled_generate_with_prompts():
    """Prompts with sampling: rows start with their prompts, forced positions score 0; with a shared prefix of 20 (prefilled
    by the teacher-forced pass) and with the same prompts forced in the loop (one more, empty row makes the shared prefix
    0) the streams agree up to each row's first flagged position, both checked against the float64 oracle."""
    import torch
    from mt3_b200 import _lib
    config = "mt3"
    V = _CFG[config][1]
    x = _inputs(config)
    rng = np.random.default_rng(4)
    lens = np.array([20, 22, 25, 20, 30, 21, 24])
    prompt = np.zeros((_B, 30), np.int32)
    for b, n in enumerate(lens):
        prompt[b, :n] = rng.integers(2, V, n)
    m = _model(config, _lib.GEMM_TF32X3, _lib.KV_F32)
    sp = {"temperature": 1.0, "topk": 0, "topp": 0.9, "key": (0, 99), "rescale": True}
    kw = dict(num_steps=_L, stop_at_eos=False, decode='sample', return_scores=True, topp=0.9, seed=99)
    B1 = _B - 1
    xp = torch.from_numpy(x[:B1]).to(DEV)
    tok_a, ts_a, _ = (t.cpu().numpy() for t in m.generate(xp, prompt=prompt[:B1], **kw))          # P = 20: prefilled
    tok_b, ts_b, _ = (t.cpu().numpy() for t in m.generate(torch.from_numpy(x).to(DEV), prompt=prompt, **kw))   # P = 0: loop
    tok_b, ts_b = tok_b[:B1], ts_b[:B1]
    fa = _check_against_oracle(config, x[:B1], tok_a, ts_a, sp, lens, prompt[:B1], tag="prefill")
    fb = _check_against_oracle(config, x[:B1], tok_b, ts_b, sp, lens, prompt[:B1], tag="loop")
    agree = 0
    for b in range(B1):
        stop = np.flatnonzero(fa[b] | fb[b])
        end = stop[0] if stop.size else _L
        np.testing.assert_array_equal(tok_a[b, :end], tok_b[b, :end], err_msg=f"row {b}")
        agree += end - lens[b]
    print(f"prefill vs loop: {agree} free positions agree before the first flag")
    assert agree >= B1 * 4


@pytest.mark.gpu
def test_num_decodes_through_the_wrapper():
    """predict_batch_with_aux(decode_fn='temperature_sample', num_decodes=4) on the model: the decodes of input i are the
    rows i n .. i n + n - 1 of one sampled generate of the expanded batch (streams i n + k), sorted by score ascending"""
    import torch
    from mt3_b200 import _lib, models
    m = _model("mt3", _lib.GEMM_TF32X3, _lib.KV_P24)
    x = torch.from_numpy(_inputs("mt3")[:2]).to(DEV)
    n = 4
    w = models.ContinuousInputsEncoderDecoderModel(m, input_depth=x.shape[-1], decode_fn='temperature_sample')
    toks, aux = w.predict_batch_with_aux(None, {'encoder_input_tokens': x}, rng=np.array([0, 5], np.uint32),
                                         decoder_params={'topk': 40}, num_decodes=n, return_all_decodes=True)
    assert toks.shape == (2, n, _L) and aux['scores'].shape == (2, n)
    tok, _, sc = (t.cpu().numpy() for t in m.generate(x.repeat_interleave(n, 0), stop_at_eos=True, decode='sample', return_scores=True,
                                                      topk=40, seed=5))
    for i in range(2):
        order = np.argsort(sc[i * n:(i + 1) * n], kind="stable")
        np.testing.assert_array_equal(toks[i].cpu().numpy(), tok[i * n + order])
        _same_bits(f"input {i}: scores", aux['scores'][i].cpu().numpy(), sc[i * n + order])
    assert (np.diff(aux['scores'].cpu().numpy(), axis=1) >= 0).all()
    best, aux1 = w.predict_batch_with_aux(None, {'encoder_input_tokens': x}, rng=np.array([0, 5], np.uint32),
                                          decoder_params={'topk': 40}, num_decodes=n)
    np.testing.assert_array_equal(best.cpu().numpy(), toks[:, -1].cpu().numpy())
