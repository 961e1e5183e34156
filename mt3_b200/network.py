"""T5-style encoder/decoder of MT3 on sm_90a: the reference's network.py surface.

`T5Config` mirrors network.py:25-41; `Transformer` exposes encode, decode -- one step (decode=True) or the
teacher-forced pass over a whole target sequence (decode=False) -- and __call__ like the Flax module (network.py:265-409),
plus `score` (the token scores of T5X's score_batch) and `generate`, which stands in for t5x's predict_batch_with_aux at
num_decodes=1 (models.py:121-138).  All compute runs in
libmt3b200.so; tensors are only the memory container.  Drop-in boundary B3 (SURVEY.md 8b).
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import _lib, weights as W

SAMPLE_MAX_FILTER_VOCAB = 4096      # top-k / top-p sort the logits row in one CTA's shared memory (layers.cuh)


def sample_key(seed):
    """The 64-bit Philox key (k0, k1) of a sampling seed: an int s in [0, 2**64) gives (s >> 32, s & 0xffffffff), the two
    words of jax.random.PRNGKey(s); two uint32 words (a PRNGKey, numpy or torch) are taken as they are."""
    if isinstance(seed, (int, np.integer)) and not isinstance(seed, bool):
        s = int(seed)
        if not 0 <= s < 2 ** 64:
            raise ValueError(f'seed must lie in [0, 2**64); got {s}')
        return s >> 32, s & 0xffffffff
    if isinstance(seed, torch.Tensor):
        seed = seed.detach().cpu().numpy()
    k = np.asarray(seed)
    if k.shape != (2,) or k.dtype.kind not in 'iu' or (k < 0).any() or (k >= 2 ** 32).any():
        raise ValueError(f'seed must be an int or two uint32 words; got {seed!r}')
    return int(k[0]), int(k[1])


@dataclasses.dataclass
class T5Config:
    """Global hyperparameters (network.py:25-41).  Defaults are the reference's class
    defaults; gin/model.gin:47-59 binds the MT3 values."""
    vocab_size: int
    dtype: str = 'float32'
    emb_dim: int = 512
    num_heads: int = 8
    num_encoder_layers: int = 6
    num_decoder_layers: int = 6
    head_dim: int = 64
    mlp_dim: int = 2048
    mlp_activations: Sequence[str] = ('relu',)
    dropout_rate: float = 0.1
    logits_via_embedding: bool = False
    input_depth: int = 512   # spectrograms.input_depth (models.py:135; gin/model.gin:43)


class Transformer:
    """An encoder-decoder Transformer model (network.py:265-409), inference only."""

    def __init__(self, config: T5Config, params: Dict[str, np.ndarray], *, device="cuda:0", max_batch: int = 8,
                 max_input_length: int = 256, max_decode_length: int = 1024, gemm_mode: int = _lib.GEMM_FP32_SIMT,
                 kv_format: int = _lib.KV_F32):
        if tuple(config.mlp_activations) != ('gelu', 'linear'):
            raise ValueError("only the gated-GELU MLP ('gelu','linear') of gin/model.gin:57 is built; got %r"
                             % (tuple(config.mlp_activations),))
        if config.logits_via_embedding:
            raise ValueError("logits_via_embedding=True is not on the MT3 path (gin/model.gin:59)")
        if config.dtype != 'float32':
            raise ValueError("the reference computes in float32 (gin/model.gin:50); got dtype=%r" % (config.dtype,))
        if not torch.cuda.is_available():
            raise RuntimeError("mt3_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.config = config
        self.device = torch.device(device)
        self.max_decode_length = int(max_decode_length)
        self._lib = _lib.load()
        self._cfg = _lib.ModelConfig(config.vocab_size, config.emb_dim, config.num_heads, config.head_dim,
                                     config.num_encoder_layers, config.num_decoder_layers, config.mlp_dim,
                                     config.input_depth, int(max_batch), int(max_input_length),
                                     int(max_decode_length), int(gemm_mode), int(kv_format))
        n = int(self._lib.mt3_model_num_params(C.byref(self._cfg)))
        if n != W.num_params(config):
            raise RuntimeError(f"parameter count mismatch: library {n}, host {W.num_params(config)}")
        blob = torch.from_numpy(W.flatten(params, config)).to(self.device)
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_model_create(C.byref(self._cfg), blob.data_ptr(), C.byref(h), self._stream()))
            torch.cuda.synchronize(self.device)
        del blob
        self._h = h
        self._ws = None
        self._ws_key = None
        self._tf_ws = None              # workspace of the teacher-forced pass (its own: the decode state stays untouched)

    # -- plumbing ---------------------------------------------------------------------
    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._lib.mt3_model_destroy(self._h)
        except Exception:
            pass

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def _bind(self, batch: int, length: int):
        key = (batch, length)
        if self._ws_key == key:
            return
        nbytes = int(self._lib.mt3_workspace_bytes(self._h, batch, length))
        if nbytes <= 0:
            raise _lib.Mt3Error(-2, f"no workspace layout for batch={batch}, input_length={length}")
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        _lib.check(self._lib.mt3_model_set_workspace(self._h, self._ws.data_ptr(), self._ws.numel(), batch, length))
        self._ws_key = key

    def _tf_workspace(self, batch: int, input_length: int, length: int) -> torch.Tensor:
        """The teacher-forced pass's workspace for `length` targets, grown when it is too small."""
        nbytes = int(self._lib.mt3_teacher_forced_workspace_bytes(self._h, batch, input_length, length))
        if nbytes <= 0:
            raise _lib.Mt3Error(-2, f"no teacher-forced workspace layout for batch={batch}, input_length={input_length}, length={length}")
        if self._tf_ws is None or self._tf_ws.numel() < nbytes:
            self._tf_ws = None
            self._tf_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._tf_ws

    def _check_inputs(self, x: torch.Tensor):
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32):
            raise TypeError("encoder_input_tokens must be a CUDA float32 tensor")
        assert x.dim() == 3, "encoder_input_tokens.ndim == 3  # (batch, length, depth) -- network.py:281"
        if x.shape[-1] != self.config.input_depth:
            raise ValueError(f"input depth {x.shape[-1]} != {self.config.input_depth}")
        return x.contiguous()

    # -- reference surface ------------------------------------------------------------
    def encode(self, encoder_input_tokens: torch.Tensor, encoder_segment_ids=None, enable_dropout: bool = False):
        """Transformer.encode (network.py:275-301): [B,T,depth] -> [B,T,emb]."""
        if enable_dropout:
            raise ValueError("inference only: enable_dropout must be False")
        if encoder_segment_ids is not None:
            raise ValueError("packing (encoder_segment_ids) is a training feature; not on this path")
        x = self._check_inputs(encoder_input_tokens)
        b, t, _ = x.shape
        self._bind(b, t)
        out = torch.empty((b, t, self.config.emb_dim), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_encode(self._h, x.data_ptr(), out.data_ptr(), self._stream()))
        return out

    def init_cache(self, encoded: torch.Tensor):
        """The cache-initialisation pass of t5x's predict_batch_with_aux: projects `encoded` to
        every decoder layer's cross K/V once, zeroes cache_index / position_embedder_index."""
        assert encoded.is_cuda and encoded.dtype == torch.float32 and encoded.dim() == 3
        b, t, _ = encoded.shape
        self._bind(b, t)
        enc = encoded.contiguous()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_cross_kv(self._h, enc.data_ptr(), self._stream()))

    def decode(self, encoded, encoder_input_tokens, decoder_input_tokens, decoder_target_tokens=None,
               encoder_segment_ids=None, decoder_segment_ids=None, decoder_positions=None, enable_dropout=False,
               decode=True, max_decode_length=None):
        """Transformer.decode (network.py:303-361).
        decode=True: one step, decoder_input_tokens int32 [B,1] -> logits float32 [B,1,V]; the KV cache lives in the model
        handle (call init_cache(encoded) first).
        decode=False: the teacher-forced pass over all L positions, decoder_input_tokens / decoder_target_tokens [B,L] ->
        logits float32 [B,L,V], with the self-attention mask make_decoder_mask(decoder_target_tokens).  Positions with
        target 0 (padding) get finite values that differ from the reference's (DESIGN.md section 1).  Touches no decode
        state."""
        if not decode:
            if enable_dropout:
                raise ValueError("inference only: enable_dropout must be False")
            if encoder_segment_ids is not None or decoder_segment_ids is not None:
                raise ValueError("packing (segment ids) is a training feature; not on this path")
            if decoder_target_tokens is None:
                raise ValueError("decode=False needs decoder_target_tokens (they make the self-attention mask)")
            del decoder_positions       # the reference ignores them too: positions are arange(L) (network.py:211-217)
            return self._teacher_forced(encoded, decoder_input_tokens, decoder_target_tokens, None, True, False)[0]
        if encoder_segment_ids is not None:
            raise ValueError('During decoding, packing should not be used but `encoder_segment_ids` was passed '
                             'to `Transformer.decode`.')
        tok = decoder_input_tokens
        if not isinstance(tok, torch.Tensor) or tok.dtype not in (torch.int32, torch.int64):
            raise ValueError('Input type must be an integer or unsigned integer.')   # layers.py:528-529
        assert tok.dim() == 2  # [batch, len] -- network.py:211
        b = tok.shape[0]
        if tok.shape[1] != 1:
            raise ValueError('Autoregressive cache shape error, expected query shape %s instead got %s.'
                             % ((b, 1), tuple(tok.shape)))                           # layers.py:266-270
        tok = tok.to(torch.int32).contiguous()
        logits = torch.empty((b, 1, self.config.vocab_size), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_decode_step(self._h, tok.data_ptr(), logits.data_ptr(), None, self._stream()))
        return logits

    def __call__(self, encoder_input_tokens, decoder_input_tokens, decoder_target_tokens, encoder_segment_ids=None,
                 decoder_segment_ids=None, encoder_positions=None, decoder_positions=None, *, enable_dropout: bool = False,
                 decode: bool = False):
        """Transformer.__call__ (network.py:363-409): encode, then decode(decode=False) -> logits float32 [B,L,V]."""
        del encoder_positions
        encoded = self.encode(encoder_input_tokens, encoder_segment_ids=encoder_segment_ids, enable_dropout=enable_dropout)
        return self.decode(encoded, encoder_input_tokens, decoder_input_tokens, decoder_target_tokens,
                           encoder_segment_ids=encoder_segment_ids, decoder_segment_ids=decoder_segment_ids,
                           decoder_positions=decoder_positions, enable_dropout=enable_dropout, decode=decode)

    def score(self, encoded: torch.Tensor, decoder_input_tokens, decoder_target_tokens, decoder_loss_weights=None) -> torch.Tensor:
        """Token scores float32 [B,L] of T5X's score_batch (z_loss 0): (logits[target] - logsumexp(logits)) * weight, weight
        = decoder_loss_weights or target > 0.  The logits are not materialised: they go through the library's workspace in
        chunks of rows."""
        return self._teacher_forced(encoded, decoder_input_tokens, decoder_target_tokens, decoder_loss_weights, False, True)[1]

    def _tokens(self, t, name: str, shape=None) -> torch.Tensor:
        if isinstance(t, np.ndarray):
            t = torch.from_numpy(t)
        if not isinstance(t, torch.Tensor) or t.dtype not in (torch.int32, torch.int64, torch.int16, torch.uint8):
            raise ValueError(f'{name}: input type must be an integer or unsigned integer.')   # layers.py:528-529
        if t.dim() != 2:
            raise ValueError(f'{name} must be [batch, length]; got shape {tuple(t.shape)}')
        if shape is not None and tuple(t.shape) != shape:
            raise ValueError(f'{name} has shape {tuple(t.shape)}, expected {shape}')
        return t.to(device=self.device, dtype=torch.int32).contiguous()

    def _teacher_forced(self, encoded, decoder_input_tokens, decoder_target_tokens, decoder_loss_weights, want_logits: bool,
                        want_scores: bool):
        """mt3_decode_teacher_forced: (logits [B,L,V] or None, token scores [B,L] or None)."""
        if not (isinstance(encoded, torch.Tensor) and encoded.is_cuda and encoded.dtype == torch.float32 and encoded.dim() == 3):
            raise TypeError("encoded must be a CUDA float32 tensor [batch, input_length, emb_dim]")
        if encoded.shape[-1] != self.config.emb_dim:
            raise ValueError(f"encoded width {encoded.shape[-1]} != emb_dim {self.config.emb_dim}")
        b, t, _ = encoded.shape
        tok_in = self._tokens(decoder_input_tokens, 'decoder_input_tokens')
        length = tok_in.shape[1]
        tgt = self._tokens(decoder_target_tokens, 'decoder_target_tokens', (b, length))
        wts = None if decoder_loss_weights is None else self._tokens(decoder_loss_weights, 'decoder_loss_weights', (b, length))
        if tok_in.shape[0] != b:
            raise ValueError(f'decoder tokens have batch {tok_in.shape[0]}, encoded has {b}')
        if not 0 < length <= self.max_decode_length:
            raise ValueError(f'decoder length {length} outside (0, max_decode_length={self.max_decode_length}]')
        if not 0 < b <= self._cfg.max_batch:
            raise ValueError(f'batch {b} outside (0, max_batch={self._cfg.max_batch}]')
        if not 0 < t <= self._cfg.max_input_length:
            raise ValueError(f'input length {t} outside (0, max_input_length={self._cfg.max_input_length}]')
        v = self.config.vocab_size
        for name, x in (('decoder_input_tokens', tok_in), ('decoder_target_tokens', tgt)):
            lo, hi = int(x.min()), int(x.max())
            if lo < 0 or hi >= v:
                raise ValueError(f'{name}: ids must lie in [0, vocab_size={v}); got [{lo}, {hi}]')
        ws = self._tf_workspace(b, t, length)
        logits = torch.empty((b, length, v), dtype=torch.float32, device=self.device) if want_logits else None
        scores = torch.empty((b, length), dtype=torch.float32, device=self.device) if want_scores else None
        enc = encoded.contiguous()
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_decode_teacher_forced(
                self._h, enc.data_ptr(), b, t, tok_in.data_ptr(), tgt.data_ptr(), None if wts is None else wts.data_ptr(), length,
                None if logits is None else logits.data_ptr(), None if scores is None else scores.data_ptr(),
                ws.data_ptr(), ws.numel(), self._stream()))
        return logits, scores

    # -- helpers built on the step ----------------------------------------------------
    def teacher_forced_logits(self, encoded: torch.Tensor, decoder_input_tokens: torch.Tensor) -> torch.Tensor:
        """Feeds decoder_input_tokens [B,L] one position at a time -> logits [B,L,V]."""
        self.init_cache(encoded)
        outs = [self.decode(encoded, None, decoder_input_tokens[:, i:i + 1]) for i in range(decoder_input_tokens.shape[1])]
        return torch.cat(outs, dim=1)

    def generate(self, encoder_input_tokens: torch.Tensor, num_steps: Optional[int] = None, stop_at_eos: bool = True,
                 use_graph: bool = True, out: Optional[torch.Tensor] = None, decode: str = 'greedy', return_scores: bool = False,
                 prompt=None, temperature: float = 1.0, topk: int = 0, topp: float = 0.0, seed=0, row_offset: int = 0,
                 rescale_log_probs: bool = True, logit_bias=None):
        """encode + decode from BOS=0 (models.py:121-138).  decode='greedy': argmax until EOS; decode='beam1': T5X's
        decoding.beam_search at num_decodes=1, the reference's decode_fn (models.py:127) -- they differ when EOS is one of the
        two best tokens without being decisive (tests/test_beam1.py).  Returns raw model ids int32 [B, max_decode_length],
        0 after EOS.
        return_scores=True returns (tokens, token_scores float32 [B, max_decode_length], scores float32 [B]) with the same
        tokens: each emitted token's log-probability (0 after EOS and beyond the steps run) and the sequence score -- greedy,
        the sum of the token scores; beam1, T5X beam_search's length-normalised score (mt3_generate_scored).
        prompt: int [B, P] (torch or numpy), T5X's prompt_with_targets: row b's non-zero prefix is forced -- the output row
        starts with it, its positions score 0, and the loop chooses from its end on.  Ids in [2, vocab_size), 0 after the
        prefix, no EOS, P <= num_steps (mt3_generate_prompted).  The prefix every row shares is prefilled by one
        teacher-forced pass.
        decode='sample': T5X's decoding.temperature_sample (mt3_generate_sampled).  Each free position draws its token from
        softmax(logits / temperature), cut to the top `topk` ids (0: off; ties at the k-th value kept) and then to the
        smallest most-likely set whose probability reaches `topp` (0 or 1: off).  temperature <= 1e-4 is greedy, bit for bit.
        `seed` is an int (the key of jax.random.PRNGKey(seed)) or a key's two uint32 words; row b draws from stream
        row_offset + b, so a row's tokens depend on (seed, row_offset + b) and its input only.  With return_scores, token
        scores are log-probabilities under the distribution sampled from (rescale_log_probs=True, T5X's default) or under
        the model's own softmax (False, greedy's), and the sequence score is their sum.
        logit_bias: float32 [V] (one row for every sequence) or [B, V] (numpy or torch), added to the logits of every free
        position before the token is picked, in every decode mode (mt3_generate_biased): -inf suppresses an id, whatever the
        model's logit.  Entries must be finite or -inf, with at least one finite entry per row.  Token and sequence scores
        are then log-probabilities under the biased logits; prompt tokens are forced even where suppressed, and a row whose
        EOS is -inf runs to num_steps.  score() and decode() stay unbiased."""
        if decode not in ('greedy', 'beam1', 'sample'):
            raise ValueError("decode must be 'greedy', 'beam1' or 'sample'")
        x = self._check_inputs(encoder_input_tokens)
        b, t, _ = x.shape
        sp = self._sample_params(temperature, topk, topp, seed, row_offset, rescale_log_probs, b) if decode == 'sample' else None
        steps = self.max_decode_length if num_steps is None else int(num_steps)
        if prompt is not None:
            prompt = self._check_prompt(prompt, b, steps)
        bias = None if logit_bias is None else self._check_logit_bias(logit_bias, b)
        self._bind(b, t)
        if out is None:
            out = torch.empty((b, self.max_decode_length), dtype=torch.int32, device=self.device)
        flags = (_lib.GEN_STOP_AT_EOS if stop_at_eos else 0) | (_lib.GEN_USE_GRAPH if use_graph else 0) | \
                (_lib.GEN_BEAM1 if decode == 'beam1' else 0) | (_lib.GEN_SAMPLE if sp is not None else 0)
        ran = C.c_int32(0)
        if sp is not None or bias is not None or (prompt is not None and prompt.shape[1] > 0):
            return self._generate_prompted(x, steps, flags, prompt, out, return_scores, sp, bias)
        if not return_scores:
            with torch.cuda.device(self.device):
                _lib.check(self._lib.mt3_generate(self._h, x.data_ptr(), steps, flags, out.data_ptr(), C.byref(ran), self._stream()))
            self.last_steps_run = int(ran.value)
            return out
        token_scores = torch.empty((b, self.max_decode_length), dtype=torch.float32, device=self.device)
        scores = torch.empty((b,), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.mt3_generate_scored(self._h, x.data_ptr(), steps, flags, out.data_ptr(), token_scores.data_ptr(),
                                                     scores.data_ptr(), C.byref(ran), self._stream()))
        self.last_steps_run = int(ran.value)
        return out, token_scores, scores

    def _check_prompt(self, prompt, batch: int, num_steps: int) -> torch.Tensor:
        """The host-side check of a generate prompt (the library checks it again on the device): int32 [B, P] on the device."""
        p = self._tokens(prompt, 'prompt')
        if p.shape[0] != batch:
            raise ValueError(f'prompt has batch {p.shape[0]}, the inputs have {batch}')
        if p.shape[1] > num_steps:
            raise ValueError(f'prompt length {p.shape[1]} exceeds num_steps={num_steps} (the steps include the prompt)')
        if p.numel():
            v = self.config.vocab_size
            lo, hi = int(p.min()), int(p.max())
            if lo < 0 or hi >= v:
                raise ValueError(f'prompt: ids must lie in [0, vocab_size={v}); got [{lo}, {hi}]')
            if bool((p == 1).any()):
                raise ValueError('prompt: EOS (1) is not allowed inside a prompt')
            ended = torch.cumsum((p == 0).to(torch.int32), dim=1) > 0
            if bool((ended & (p != 0)).any()):
                raise ValueError('prompt: a row has non-zero ids after its first 0 (PAD ends the prompt)')
        return p

    def _check_logit_bias(self, logit_bias, batch: int) -> torch.Tensor:
        """The host-side check of a generate logit bias (the library checks it again on the device): float32 [V] or [B, V] on
        the device, contiguous (its row stride is then 0 or V)."""
        t = torch.from_numpy(logit_bias) if isinstance(logit_bias, np.ndarray) else logit_bias
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
            raise ValueError('logit_bias must be a float32 numpy array or torch tensor')
        v = self.config.vocab_size
        if tuple(t.shape) not in ((v,), (batch, v)):
            raise ValueError(f'logit_bias must have shape ({v},) or ({batch}, {v}); got {tuple(t.shape)}')
        rows = t.detach().reshape(-1, v).cpu()
        if bool(torch.isnan(rows).any()) or bool((rows == math.inf).any()):
            raise ValueError('logit_bias: entries must be finite or -inf (no NaN, no +inf)')
        if not bool(torch.isfinite(rows).any(1).all()):
            raise ValueError('logit_bias: every row must keep at least one finite entry')
        return t.to(device=self.device).contiguous()

    def _sample_params(self, temperature, topk, topp, seed, row_offset, rescale_log_probs, batch: int) -> _lib.SampleParams:
        """The host-side check of generate's sampling arguments (the library checks them again)."""
        temperature, topp = float(temperature), float(topp)
        if not (math.isfinite(temperature) and temperature >= 0):
            raise ValueError(f'temperature must be finite and >= 0; got {temperature}')
        if int(topk) != topk or not 0 <= topk < 2 ** 31:
            raise ValueError(f'topk must be an int >= 0; got {topk!r}')
        if not 0.0 <= topp <= 1.0:
            raise ValueError(f'topp must lie in [0, 1]; got {topp}')
        v = self.config.vocab_size
        if v > SAMPLE_MAX_FILTER_VOCAB and (0 < topk < v or 0 < topp < 1):
            raise ValueError(f'top-k / top-p need vocab_size <= {SAMPLE_MAX_FILTER_VOCAB}; this model has {v}')
        if int(row_offset) != row_offset or not 0 <= row_offset <= 2 ** 32 - batch:
            raise ValueError(f'row_offset must be an int in [0, 2**32 - batch]; got {row_offset!r}')
        sp = _lib.SampleParams()
        sp.temperature, sp.topk, sp.topp = temperature, int(topk), topp
        sp.key[0], sp.key[1] = sample_key(seed)
        sp.row0, sp.rescale_log_probs = int(row_offset), int(bool(rescale_log_probs))
        return sp

    def _generate_prompted(self, x, steps: int, flags: int, prompt: Optional[torch.Tensor], out: torch.Tensor, return_scores: bool,
                           sp: Optional[_lib.SampleParams] = None, bias: Optional[torch.Tensor] = None):
        b, t, _ = x.shape
        plen = 0 if prompt is None else prompt.shape[1]
        ws = self._tf_workspace(b, t, plen) if plen else None
        token_scores = torch.empty((b, self.max_decode_length), dtype=torch.float32, device=self.device) if return_scores else None
        scores = torch.empty((b,), dtype=torch.float32, device=self.device) if return_scores else None
        ran = C.c_int32(0)
        args = (self._h, x.data_ptr(), steps, flags, prompt.data_ptr() if plen else None, plen, out.data_ptr(),
                None if token_scores is None else token_scores.data_ptr(), None if scores is None else scores.data_ptr(), C.byref(ran),
                ws.data_ptr() if plen else None, ws.numel() if plen else 0)
        with torch.cuda.device(self.device):
            if bias is not None:
                _lib.check(self._lib.mt3_generate_biased(*args, None if sp is None else C.byref(sp), bias.data_ptr(),
                                                         0 if bias.dim() == 1 else bias.shape[1], self._stream()))
            elif sp is None:
                _lib.check(self._lib.mt3_generate_prompted(*args, self._stream()))
            else:
                _lib.check(self._lib.mt3_generate_sampled(*args, C.byref(sp), self._stream()))
        self.last_steps_run = int(ran.value)
        return (out, token_scores, scores) if return_scores else out
