"""Programmatic edges between the decode GEMM nodes (MT3_PDL_GEMM) change only when each GEMM's CTAs start and where they
load and split their weight tiles: the instruction stream of the multiply, the reduction order and the data are the same,
so token streams and logits must be bit-identical to the run without the edges.

Bench's configuration (the mt3 model, weights `synthetic:0`, audio synth_audio(B, 1234), GPU spectrogram, 1024 greedy steps
through the 16-step graphs) at B = 64 and at a ragged B = 37, in gemm modes SIMT (exact fp32 multiply) and TF32X3 (3xTF32
wgmma multiply, hi / lo split of the weight tile before the wait), in every K/V row format.  The step path
(mt3_decode_step, plain launches) is compared at positions on both sides of the 256-key tile boundaries and at the last
cache row."""
import numpy as np
import pytest
import torch

import bench

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
T, L = 256, 1024
POS = [0, 1, 255, 256, 1023]       # decode positions whose step-path logits are compared
KNOBS = ("MT3_PDL_GEMM", "MT3_PDL", "MT3_PF_ATTN", "MT3_PF_KV")


def _cfg():
    from mt3_b200 import network
    return network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=8, num_decoder_layers=8, head_dim=64,
                            mlp_dim=1024, mlp_activations=('gelu', 'linear'))


@pytest.fixture(scope="module")
def params():
    from mt3_b200 import weights
    return weights.synthetic_params(_cfg(), 0)


def _run(params, spec, gm, kv, forced):
    """generate's 1024 tokens [B, L] and the step path's logits at POS [B, len(POS), V], the step path fed `forced` (or, when
    None, this run's own tokens: BOS then tokens[:, :-1])."""
    from mt3_b200 import network
    b = spec.shape[0]
    m = network.Transformer(_cfg(), params, device=DEV, max_batch=b, max_input_length=T, max_decode_length=L, gemm_mode=gm,
                            kv_format=kv)
    toks = m.generate(spec, num_steps=L, stop_at_eos=False, use_graph=True).clone()
    assert m.last_steps_run == L
    if forced is None:
        forced = torch.cat([torch.zeros((b, 1), dtype=torch.int32, device=DEV), toks[:, :-1]], dim=1)
    enc = m.encode(spec)
    m.init_cache(enc)
    kept = []
    for i in range(L):
        lg = m.decode(enc, None, forced[:, i:i + 1])
        if i in POS:
            kept.append(lg[:, 0].clone())
    torch.cuda.synchronize()
    del m
    torch.cuda.empty_cache()
    return toks, torch.stack(kept, dim=1), forced


@pytest.mark.parametrize("B", [64, 37])
@pytest.mark.parametrize("kv", ["p24", "f16", "f32"])
@pytest.mark.parametrize("mode", ["tf32x3", "simt"])
def test_gemm_edges_are_value_neutral(params, mode, kv, B, monkeypatch):
    from mt3_b200 import _lib, spectrograms
    gm = {"simt": _lib.GEMM_FP32_SIMT, "tf32x3": _lib.GEMM_TF32X3}[mode]
    kvf = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[kv]
    audio = torch.from_numpy(bench.synth_audio(B, 1234)).to(DEV)
    spec = spectrograms.compute_spectrogram(audio, spectrograms.SpectrogramConfig())
    assert tuple(spec.shape) == (B, T, 512)
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)

    monkeypatch.setenv("MT3_PDL_GEMM", "0")
    off_t, off_l, forced = _run(params, spec, gm, kvf, None)
    monkeypatch.delenv("MT3_PDL_GEMM")          # the library default: GEMM edges on
    on_t, on_l, _ = _run(params, spec, gm, kvf, forced)

    assert off_t.shape == (B, L) and off_l.shape == (B, len(POS), 1536)
    assert torch.isfinite(off_l).all()
    diff = (on_t != off_t).cpu().numpy()
    if diff.any():
        s = int(np.nonzero(diff.any(0))[0][0])
        raise AssertionError(f"token streams differ with the GEMM edges on, first at step {s} in {int(diff[:, s].sum())} of {B} "
                             f"sequences")
    for j, p in enumerate(POS):
        assert torch.equal(on_l[:, j], off_l[:, j]), f"step-path logits differ at position {p}"
