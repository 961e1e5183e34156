"""The early L2 prefetch of each layer's self-attention K/V (MT3_PF_KV) changes cache state only: the arithmetic, its
order and the data layout are untouched, so token streams and logits must be bit-identical to the run with it off, in
every K/V row format, at the full batch of 64 and at a ragged batch, over cache positions that run past the attention
kernel's shared-memory ring (192 / 384 / 256 keys for fp32 / fp16 / p24 rows) and past the prefetched rows."""
import numpy as np
import pytest
import torch

from oracle import mt3_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
L = 400                     # cache capacity: not a multiple of any tile, past every ring
BASE = {"MT3_PF_KV": "0"}
SETTINGS = [
    {"MT3_PF_KV": "1"},
    {"MT3_PF_KV": "2"},
    {},                                         # the library defaults
]
KNOBS = ("MT3_PF_KV", "MT3_PDL")


def _run(cfg, params, x, forced, gmode, kvf):
    from mt3_b200 import network
    b = x.shape[0]
    m = network.Transformer(cfg, params, device=DEV, max_batch=b, max_input_length=256, max_decode_length=L, gemm_mode=gmode,
                            kv_format=kvf)
    toks = m.generate(x, stop_at_eos=False, use_graph=True).clone()
    lg = m.teacher_forced_logits(m.encode(x), forced).clone()
    torch.cuda.synchronize()
    del m
    return toks, lg


@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("kv", ["p24", "f16", "f32"])
def test_early_kv_prefetch_is_value_neutral(kv, B, monkeypatch):
    from mt3_b200 import _lib, network
    ocfg = O.T5Config(vocab_size=1536, num_encoder_layers=1, num_decoder_layers=8)
    params = O.init_params(ocfg, seed=41)
    cfg = network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=1, num_decoder_layers=8, head_dim=64,
                           mlp_dim=1024, mlp_activations=('gelu', 'linear'))
    audio = np.stack([O.sine_mix(256 * 128, seed=900 + i) for i in range(B)])
    x = torch.from_numpy(O.compute_spectrogram(audio, np.float32)).to(DEV)
    forced = torch.from_numpy(np.random.default_rng(B).integers(3, 1500, size=(B, L)).astype(np.int32)).to(DEV)
    gmode = _lib.GEMM_TF32X3
    kvf = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[kv]

    def setenv(env):
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)

    setenv(BASE)
    base_t, base_l = _run(cfg, params, x, forced, gmode, kvf)
    assert base_t.shape == (B, L) and base_l.shape == (B, L, 1536)
    for env in SETTINGS:
        setenv(env)
        t, lg = _run(cfg, params, x, forced, gmode, kvf)
        assert torch.equal(t, base_t), f"token streams differ under {env}"
        assert torch.equal(lg, base_l), f"logits differ under {env}"
