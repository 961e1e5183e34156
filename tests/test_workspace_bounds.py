"""The model stays inside the workspaces it asks for.

Each workspace -- the model workspace (mt3_workspace_bytes) and the teacher-forced one (mt3_teacher_forced_workspace_bytes)
-- is bound at exactly the reported size, NaN-filled, with NaN guard bytes after it.  Every path that writes workspace
runs: encode + init_cache + decode steps, greedy and beam-size-1 generate with graphs and scores, a prompted generate whose
shared prefix takes the prefill pass, decode(decode=False) and score.  The guards must be untouched and every output must
equal, bit for bit, a run in ample workspaces.  The cases cover each GEMM mode, two K/V row formats, input lengths whose
encoder attention runs on the wgmma kernel (256; 512, key-split) or on the exact-fp32 kernel (100), and
MT3_TC_ATTENTION=0: where the encoder's attention runs on the fp32 kernel its workspace holds no V^T or qkv lo plane.
"""
import numpy as np
import pytest
import torch

DEV = "cuda:0"
_B, _L, _P = 3, 48, 24      # P >= 20 shared prompt tokens: the prefill pass runs; L = 3 blocks of 16 graph steps
_GUARD = 64 * 1024          # bytes of NaN after each workspace
_NAN_BITS = 0x7FC00000

CASES = [  # gemm mode, K/V row format, input length, MT3_TC_ATTENTION
    ("simt", "f32", 256, None),
    ("simt", "p24", 100, None),
    ("tf32", "f16", 100, None),
    ("tf32", "p24", 512, None),
    ("tf32x3", "p24", 256, None),
    ("tf32x3", "f32", 100, None),
    ("tf32x3", "f16", 512, None),
    ("tf32x3", "p24", 256, "0"),
    ("tf32", "f32", 256, "0"),
]


def _cfg():
    from mt3_b200 import network
    return network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=2, num_decoder_layers=2, head_dim=64,
                            mlp_dim=1024, mlp_activations=('gelu', 'linear'))


@pytest.fixture(scope="module")
def params():
    from mt3_b200 import weights
    return weights.synthetic_params(_cfg(), 3)


class _Region:
    """A NaN-filled workspace of `nbytes` (exact) or `nbytes + slack` bytes, followed by _GUARD NaN bytes."""

    def __init__(self, nbytes, slack=0):
        assert nbytes > 0 and nbytes % 256 == 0
        self.nbytes = nbytes + slack
        self.raw = torch.full(((self.nbytes + _GUARD) // 4,), float("nan"), dtype=torch.float32, device=DEV).view(torch.uint8)
        self.ws = self.raw[:self.nbytes]

    def guard_intact(self):
        return bool((self.raw[self.nbytes:].view(torch.int32) == _NAN_BITS).all())


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


def _run(m, x, prompt, tok_in, tgt, slack):
    """Every workspace user once, each workspace bound at its reported size (+ slack); the outputs and the regions."""
    b, t, _ = x.shape
    regions = []

    def bind_model_ws():
        r = _Region(int(m._lib.mt3_workspace_bytes(m._h, b, t)), slack)
        m._ws, m._ws_key = r.ws, None
        regions.append(r)

    def bind_tf_ws(length):
        r = _Region(int(m._lib.mt3_teacher_forced_workspace_bytes(m._h, b, t, length)), slack)
        m._tf_ws = r.ws
        regions.append(r)

    out = {}
    bind_model_ws()
    enc = m.encode(x)
    out["encoded"] = enc.clone()
    m.init_cache(enc)
    for i in range(3):
        out[f"step{i}"] = m.decode(enc, None, tok_in[:, i:i + 1])
    for mode in ("greedy", "beam1"):
        tok, ts, sc = m.generate(x, num_steps=_L, stop_at_eos=False, use_graph=True, decode=mode, return_scores=True)
        out[mode] = (tok.clone(), ts, sc)
    bind_tf_ws(prompt.shape[1])
    tok, ts, sc = m.generate(x, num_steps=_L, stop_at_eos=False, use_graph=True, return_scores=True, prompt=prompt)
    out["prompted"] = (tok.clone(), ts, sc)
    bind_tf_ws(tgt.shape[1])
    out["logits"] = m.decode(enc, None, tok_in, tgt, decode=False)
    out["score"] = m.score(enc, tok_in, tgt)
    torch.cuda.synchronize()
    assert m.last_steps_run == _L
    return out, regions


def _flat(out):
    for k, v in out.items():
        for i, a in enumerate(v if isinstance(v, tuple) else (v,)):
            yield f"{k}[{i}]", _bits(a)


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,kv,T,tc_attn", CASES, ids=lambda v: str(v))
def test_workspaces_hold_what_the_model_writes(params, monkeypatch, gemm, kv, T, tc_attn):
    from mt3_b200 import _lib, network
    if tc_attn is None:
        monkeypatch.delenv("MT3_TC_ATTENTION", raising=False)
    else:
        monkeypatch.setenv("MT3_TC_ATTENTION", tc_attn)       # read when the model is created
    gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32": _lib.GEMM_TF32, "tf32x3": _lib.GEMM_TF32X3}[gemm]
    kf = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[kv]
    m = network.Transformer(_cfg(), params, device=DEV, max_batch=_B, max_input_length=T, max_decode_length=_L, gemm_mode=gm,
                            kv_format=kf)
    rng = np.random.default_rng(T + 7 * gm + kf)
    x = torch.from_numpy(rng.standard_normal((_B, T, 512)).astype(np.float32)).to(DEV)
    prompt = np.zeros((_B, _P + 4), np.int32)
    prompt[:, :_P] = rng.integers(2, 1536, _P)                  # every row shares the first _P tokens
    prompt[0, _P:_P + 3] = rng.integers(2, 1536, 3)             # and row 0 goes on, forced inside the loop
    tgt = rng.integers(2, 1536, (_B, _L)).astype(np.int32)
    tgt[1, 30:] = 0                                             # a padded row
    tok_in = np.concatenate([np.zeros((_B, 1), np.int32), tgt[:, :-1]], 1)
    prompt, tok_in, tgt = (torch.from_numpy(a).to(DEV) for a in (prompt, tok_in, tgt))

    exact, regions = _run(m, x, prompt, tok_in, tgt, slack=0)
    assert all(r.guard_intact() for r in regions), [r.nbytes for r in regions if not r.guard_intact()]
    ample, _ = _run(m, x, prompt, tok_in, tgt, slack=1 << 20)
    for (name, a), (_, b) in zip(_flat(exact), _flat(ample)):
        np.testing.assert_array_equal(a, b, err_msg=name)
    assert np.isfinite(exact["logits"].cpu().numpy()).all()
