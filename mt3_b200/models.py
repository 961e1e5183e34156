"""Feature converter and model wrapper for an encoder-decoder with continuous inputs (the reference's models.py).

`ContinuousInputsEncDecFeatureConverter` (models.py:24-118) is the step between a task example and the network:
`inputs` float32 [frames, depth] is trimmed / zero-padded to the task's input length (0.0 rows -- a value in log-mel space,
not log(eps); SURVEY 8a row a8), `targets` int32 to the target length, the decoder input is the target shifted right
behind a 0 and the loss weights mark the non-padding targets.  seqio's packing is a training feature and is refused.

`ContinuousInputsEncoderDecoderModel` (models.py:121-152) pairs a `network.Transformer` with the converter and a decode
function: `predict_batch` is T5X's predict_batch_with_aux at num_decodes = 1 (BOS 0, EOS 1, at most max_decode_length
steps) -- `decode_fn='beam_search'` is the reference's default (models.py:127) and runs the library's beam-size-1
bookkeeping, `decode_fn='greedy'` the plain argmax loop, `decode_fn='temperature_sample'` T5X's decoding.temperature_sample with
num_decodes samples per input.  `score_batch` is T5X's EncoderDecoderModel.score_batch (which
the reference's model inherits): the log-likelihood of given targets, from the teacher-forced decoder pass.  Training
(loss, optimizer, label smoothing) is out of scope.
"""
from __future__ import annotations

import inspect
from typing import Any, Dict, List, Mapping, Sequence

import numpy as np


class ContinuousInputsEncDecFeatureConverter:
    """Feature converter for an encoder-decoder with continuous inputs."""

    TASK_FEATURES = {'inputs': {'dtype': np.float32, 'rank': 2}, 'targets': {'dtype': np.int32, 'rank': 1}}
    MODEL_FEATURES = {'encoder_input_tokens': {'dtype': np.float32, 'rank': 2}, 'decoder_target_tokens': {'dtype': np.int32, 'rank': 1},
                      'decoder_input_tokens': {'dtype': np.int32, 'rank': 1}, 'decoder_loss_weights': {'dtype': np.int32, 'rank': 1}}

    def __init__(self, pack: bool = False):
        if pack:
            raise ValueError('packing is a training feature; the inference path converts one example per row')
        self.pack = False

    @staticmethod
    def _trim_or_pad(x: np.ndarray, length: int) -> np.ndarray:
        x = x[:length]
        if x.shape[0] == length:
            return x
        return np.concatenate([x, np.zeros((length - x.shape[0],) + x.shape[1:], x.dtype)], axis=0)

    def convert_example(self, features: Mapping[str, Any], task_feature_lengths: Mapping[str, int]) -> Dict[str, np.ndarray]:
        """One task example -> the model features of fixed length (models.py:77-98 after seqio's trim / pad)."""
        missing = [k for k in task_feature_lengths if k not in features]
        if missing:
            raise ValueError('task_feature_lengths names features the example does not have: %s' % missing)
        inputs = np.asarray(features['inputs'], np.float32)
        if inputs.ndim != 2:
            raise ValueError('inputs must have rank 2 (frames, depth); got shape %s' % (inputs.shape,))
        targets = np.asarray(features.get('targets', np.zeros((0,), np.int32)), np.int32)
        if targets.ndim != 1:
            raise ValueError('targets must have rank 1; got shape %s' % (targets.shape,))
        inputs = self._trim_or_pad(inputs, int(task_feature_lengths['inputs']))
        targets = self._trim_or_pad(targets, int(task_feature_lengths['targets']))
        shifted = np.concatenate([np.zeros((1,), np.int32), targets[:-1]]) if targets.size else targets
        return {'encoder_input_tokens': inputs, 'decoder_target_tokens': targets, 'decoder_input_tokens': shifted,
                'decoder_loss_weights': (targets != 0).astype(np.int32)}

    def __call__(self, ds: Sequence[Mapping[str, Any]], task_feature_lengths: Mapping[str, int]) -> List[Dict[str, np.ndarray]]:
        return [self.convert_example(ex, task_feature_lengths) for ex in ds]

    def get_model_feature_lengths(self, task_feature_lengths: Mapping[str, int]) -> Dict[str, int]:
        """Length relationship between task and model features (models.py:100-118)."""
        enc, dec = task_feature_lengths['inputs'], task_feature_lengths['targets']
        return {'encoder_input_tokens': enc, 'decoder_target_tokens': dec, 'decoder_input_tokens': dec, 'decoder_loss_weights': dec}


class ContinuousInputsEncoderDecoderModel:
    """Encoder-decoder model with continuous inputs: a `network.Transformer` (or anything with its `generate`) behind
    T5X's predict_batch surface."""

    FEATURE_CONVERTER_CLS = ContinuousInputsEncDecFeatureConverter
    DECODE_FNS = {'beam_search': 'beam1', 'greedy': 'greedy', 'temperature_sample': 'sample'}
    SAMPLE_PARAMS = ('temperature', 'topk', 'topp')

    def __init__(self, module, input_vocabulary=None, output_vocabulary=None, optimizer_def=None, input_depth: int = 512,
                 decode_fn: str = 'beam_search', label_smoothing: float = 0.0, z_loss: float = 0.0, loss_normalizing_factor=None):
        if decode_fn not in self.DECODE_FNS:
            raise ValueError("decode_fn must be 'beam_search' (T5X decoding.beam_search at num_decodes=1), 'greedy' or "
                             "'temperature_sample'")
        if optimizer_def is not None or label_smoothing or z_loss or loss_normalizing_factor is not None:
            raise ValueError('inference only: optimizer / loss arguments are not supported')
        self.module = module
        self.input_vocabulary, self.output_vocabulary = input_vocabulary, output_vocabulary
        self._input_depth = int(input_depth)
        self._decode = self.DECODE_FNS[decode_fn]

    def get_initial_variables(self, rng=None, input_shapes=None, input_types=None):
        """Shape check of the reference's override (models.py:140-152): a rank-2 encoder shape gets the input depth appended,
        a rank-3 one must end in it.  Returns the completed shapes (there are no variables to initialise here)."""
        del rng, input_types
        enc = tuple(input_shapes['encoder_input_tokens'])
        if len(enc) == 2:
            enc = (*enc, self._input_depth)
        else:
            assert enc[-1] == self._input_depth
        return {**dict(input_shapes), 'encoder_input_tokens': enc}

    def _inputs(self, batch: Mapping[str, Any], decoder_params, num_decodes: int):
        if self._decode != 'sample':
            if num_decodes != 1:
                raise ValueError('beam_search and greedy run at num_decodes=1 only (the notebook and infer.gin use the default)')
            if decoder_params and decoder_params.get('decode_rng') is not None:
                raise ValueError('beam_search and greedy are deterministic: decode_rng must be None')
        elif int(num_decodes) != num_decodes or num_decodes < 1:
            raise ValueError('num_decodes must be an int >= 1; got %r' % (num_decodes,))
        x = batch['encoder_input_tokens']
        if x.shape[-1] != self._input_depth:
            raise ValueError('encoder_input_tokens depth %d != input_depth %d' % (x.shape[-1], self._input_depth))
        return x

    def _sample_kw(self, rng, decoder_params) -> Dict[str, Any]:
        """generate's sampling arguments from T5X's rng / decoder_params: the key is `rng` or decoder_params['decode_rng']
        (not both; neither: key 0, T5X's default), an int or a PRNGKey's two uint32 words; temperature, topk and topp
        default to generate's (1.0, 0, 0.0: no filter)."""
        dp = dict(decoder_params or {})
        unknown = set(dp) - {'decode_rng', *self.SAMPLE_PARAMS}
        if unknown:
            raise ValueError('temperature_sample takes decoder_params %s; got %s' % (sorted({'decode_rng', *self.SAMPLE_PARAMS}),
                                                                                   sorted(unknown)))
        key = dp.pop('decode_rng', None)
        if rng is not None:
            if key is not None:
                raise ValueError('pass the key as rng or as decoder_params["decode_rng"], not both')
            key = rng
        return {'seed': 0 if key is None else key, **dp}

    def predict_batch_with_aux(self, params, batch: Mapping[str, Any], rng=None, decoder_params=None, num_decodes: int = 1,
                               return_all_decodes: bool = False, prompt_with_targets: bool = False):
        """tokens int32 [B, max_decode_length] (0 after EOS) and T5X's aux dict {'scores': float32 [B]}: the greedy sequence's
        summed token log-probabilities, or beam_search's length-normalised score.  A module whose `generate` cannot return
        scores (no `return_scores` argument) gives an empty aux dict.  return_all_decodes=True adds T5X's decodes axis:
        tokens [B, 1, max_decode_length], scores [B, 1].  `params` is accepted for signature fidelity: the weights live in
        the module.
        prompt_with_targets=True (T5X): batch['decoder_input_tokens'][:, 1:] is the prompt -- each row's non-zero prefix is
        forced and returned inside the decodes (Transformer.generate's `prompt`).  Column 0 is the BOS 0 of the
        right-shifted targets.
        decode_fn='temperature_sample': `rng` (or decoder_params['decode_rng']) keys the sampling and decoder_params may set
        temperature, topk and topp (_sample_kw).  num_decodes = n > 1 samples n decodes per input (_sample_decodes):
        tokens [B, n, max_decode_length] and scores [B, n] sorted ascending, or the best [B, max_decode_length] / [B]
        without return_all_decodes.  B * n rows must fit the module's max_batch."""
        del params
        x = self._inputs(batch, decoder_params, num_decodes)
        kw = self._sample_kw(rng, decoder_params) if self._decode == 'sample' else {}
        if prompt_with_targets:
            din = np.asarray(batch['decoder_input_tokens'].cpu() if hasattr(batch['decoder_input_tokens'], 'cpu')
                             else batch['decoder_input_tokens'])
            if din.ndim != 2 or din.shape[1] < 1:
                raise ValueError('decoder_input_tokens must be [batch, length >= 1]; got shape %s' % (din.shape,))
            if (din[:, 0] != 0).any():
                raise ValueError('decoder_input_tokens[:, 0] must be BOS 0 (the targets shifted right)')
            kw['prompt'] = np.ascontiguousarray(din[:, 1:])
        if num_decodes > 1:
            return self._sample_decodes(x, kw, num_decodes, return_all_decodes)
        aux = {}
        if 'return_scores' in inspect.signature(self.module.generate).parameters:
            tokens, _, scores = self.module.generate(x, stop_at_eos=True, decode=self._decode, return_scores=True, **kw)
            aux['scores'] = scores[:, None] if return_all_decodes else scores
        else:
            tokens = self.module.generate(x, stop_at_eos=True, decode=self._decode, **kw)
        return (tokens[:, None] if return_all_decodes else tokens), aux

    def _sample_decodes(self, x, kw, n: int, return_all_decodes: bool):
        """num_decodes = n samples per input, as T5X lays them out: input i's are rows i n .. i n + n - 1 of one batch (row
        r draws from stream r), returned sorted by sequence score, ascending (stable on the decode index), best last."""
        import torch
        if 'return_scores' not in inspect.signature(self.module.generate).parameters:
            raise ValueError('num_decodes > 1 ranks the samples by score: the module\'s generate must return scores')
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        b = x.shape[0]
        x = x.repeat_interleave(n, dim=0)
        if 'prompt' in kw:
            kw['prompt'] = np.repeat(kw['prompt'], n, axis=0)
        tokens, _, scores = self.module.generate(x, stop_at_eos=True, decode=self._decode, return_scores=True, **kw)
        tokens, scores = torch.as_tensor(tokens), torch.as_tensor(scores)
        tokens, scores = tokens.reshape(b, n, -1), scores.reshape(b, n)
        order = torch.sort(scores, dim=1, stable=True).indices
        scores = torch.gather(scores, 1, order)
        tokens = torch.gather(tokens, 1, order[..., None].expand_as(tokens))
        if return_all_decodes:
            return tokens, {'scores': scores}
        return tokens[:, -1], {'scores': scores[:, -1]}

    def predict_batch(self, params, batch: Mapping[str, Any], rng=None, decoder_params=None):
        """The tokens of predict_batch_with_aux, without computing scores."""
        del params
        kw = self._sample_kw(rng, decoder_params) if self._decode == 'sample' else {}
        return self.module.generate(self._inputs(batch, decoder_params, 1), stop_at_eos=True, decode=self._decode, **kw)

    def score_batch(self, params, batch: Mapping[str, Any], return_intermediates: bool = False):
        """T5X EncoderDecoderModel.score_batch with z_loss = 0: float32 [B], the sum over positions of
        (log_softmax(logits)[target] * decoder_loss_weights).  `batch` holds the model features of the feature converter
        (encoder_input_tokens, decoder_input_tokens, decoder_target_tokens, decoder_loss_weights), numpy or torch.
        `params` is accepted for signature fidelity: the weights live in the module."""
        del params
        if return_intermediates:
            raise ValueError('return_intermediates=True is not supported: the pass keeps no intermediates')
        import torch
        x = batch['encoder_input_tokens']
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, np.float32))
        if x.shape[-1] != self._input_depth:
            raise ValueError('encoder_input_tokens depth %d != input_depth %d' % (x.shape[-1], self._input_depth))
        encoded = self.module.encode(x.to(self.module.device))
        token_scores = self.module.score(encoded, batch['decoder_input_tokens'], batch['decoder_target_tokens'],
                                         batch.get('decoder_loss_weights'))
        return token_scores.to(torch.float64).sum(-1).to(torch.float32)
