"""InferenceModel: the driver API of the reference's Colab notebook on the H100 path.

The class mirrors `InferenceModel` in mt3/colab/music_transcription_with_transformers.ipynb
(raw JSON lines 170-363; drop-in boundary B1, SURVEY.md 8b): same constructor arguments,
attributes (`batch_size`, `inputs_length`, `outputs_length`, `sequence_length`,
`spectrogram_config`, `codec`, `vocabulary`) and methods (`predict_tokens`, `__call__`,
`audio_to_dataset`, `_audio_to_frames`, `preprocess`, `postprocess`, `_trim_eos`).
tf.data / seqio / T5X are replaced by plain Python lists and the CUDA library:

    audio --host pad/split--> segments --H2D--> log-mel kernel --> encoder + greedy decoder
          --D2H--> token ids --vocabulary.decode_tf--> per-segment predictions

A "dataset" here is a list of example dicts.  Divergences from the notebook, recorded in DESIGN.md:
  * decode='greedy' by default; decode='beam1' runs T5X's beam_search bookkeeping at num_decodes=1, the reference's
    decode_fn (models.py:127) -- the two differ when EOS is among the two best tokens without being decisive;
  * kv_format=KV_P24 by default: the decoder's K/V rows are stored with 24 bits per element (float32 cut to 16
    mantissa bits; all arithmetic stays float32; logit error ~5e-6 of the logit scale against the float64 oracle, the
    level of the float32 arithmetic itself).  kv_format=_lib.KV_F32 keeps float32 rows; _lib.KV_F16 (fp16 rows) is the
    fastest and holds the 5e-4 bar for diffuse attention only -- validate it on the checkpoint first (DESIGN.md section 4);
  * `__call__` returns a NoteSequence stand-in (mt3_b200.note_decoding.NoteSequence), not a note_seq protobuf.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib, gin_lite, models, network, note_decoding, note_encoding, spectrograms, vocabularies, weights

_GIN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gin")


def segment_score_targets(note_sequence, codec, vocabulary, frame_times, inputs_length: int, encoding_spec: str,
                          targets_length: int = 1024) -> Dict[str, np.ndarray]:
    """The decoder features of every audio segment's labels, built the way the transcription tasks and the feature
    converter build them: note_sequence_to_segment_targets per segment of `inputs_length` frames (ties for
    NoteEncodingWithTiesSpec, onsets only for NoteOnsetEncodingSpec), the vocabulary's +3 offset, EOS appended
    (tasks.py:179, seqio's tokenize_and_append_eos), then trimmed or zero-padded to `targets_length` with the decoder input
    shifted right behind a 0 (models.py:77-98).  Returns int32 [S, targets_length] arrays 'decoder_input_tokens',
    'decoder_target_tokens', 'decoder_loss_weights'.  Host only."""
    segs = note_encoding.note_sequence_to_segment_targets(
        note_sequence, codec, frame_times, inputs_length, onsets_only=encoding_spec == 'NoteOnsetEncodingSpec',
        include_ties=encoding_spec == 'NoteEncodingWithTiesSpec')
    conv = models.ContinuousInputsEncDecFeatureConverter()
    keys = ('decoder_input_tokens', 'decoder_target_tokens', 'decoder_loss_weights')
    out = {k: np.zeros((len(segs), targets_length), np.int32) for k in keys}
    for i, toks in enumerate(segs):
        targets = np.asarray(list(vocabulary.encode(toks)) + [1], np.int32)        # EOS = 1 (vocabularies.py:157-159)
        feats = conv.convert_example({'inputs': np.zeros((0, 1), np.float32), 'targets': targets},
                                     {'inputs': 0, 'targets': targets_length})
        for k in keys:
            out[k][i] = feats[k]
    return out


class InferenceModel(object):
    """Wrapper of the H100 model for music transcription."""

    logit_bias = None     # float32 [vocab_size] of programs= / drums=, or None (no restriction)

    def __init__(self, checkpoint_path, model_type='mt3', *, device='cuda:0', batch_size: int = 8,
                 gin_dir: Optional[str] = None, gemm_mode: int = _lib.GEMM_TF32X3, use_graph: bool = True,
                 kv_format: int = _lib.KV_P24, decode: str = 'greedy', sample_params: Optional[Dict] = None,
                 programs: Optional[Sequence[int]] = None, drums: bool = True):
        # Model Constants (notebook :175-185).
        if model_type == 'ismir2021':
            num_velocity_bins = 127
            self.encoding_spec = 'NoteEncodingSpec'
            self.inputs_length = 512
        elif model_type == 'mt3':
            num_velocity_bins = 1
            self.encoding_spec = 'NoteEncodingWithTiesSpec'
            self.inputs_length = 256
        else:
            raise ValueError('unknown model_type: %s' % model_type)
        self.model_type = model_type
        gin_dir = gin_dir or _GIN_DIR
        gin_files = [os.path.join(gin_dir, 'model.gin'), os.path.join(gin_dir, f'{model_type}.gin')]

        self.batch_size = batch_size          # the notebook uses 8 (:190)
        self.outputs_length = 1024
        self.sequence_length = {'inputs': self.inputs_length, 'targets': self.outputs_length}
        self.device = torch.device(device)
        self.use_graph = use_graph
        self._gemm_mode = gemm_mode
        self._kv_format = kv_format
        self.decode = decode              # 'greedy' | 'beam1' (T5X beam_search at num_decodes=1, models.py:127) | 'sample'
        # decode='sample': Transformer.generate's temperature / topk / topp / rescale_log_probs; the seed is per call
        self.sample_params = dict(sample_params or {})
        unknown = set(self.sample_params) - {'temperature', 'topk', 'topp', 'rescale_log_probs'}
        if unknown:
            raise ValueError('sample_params takes temperature, topk, topp and rescale_log_probs; got %s' % sorted(unknown))

        # Build Codecs and Vocabularies (notebook :198-206).
        self.spectrogram_config = spectrograms.SpectrogramConfig()
        self.codec = vocabularies.build_codec(
            vocab_config=vocabularies.VocabularyConfig(num_velocity_bins=num_velocity_bins))
        self.vocabulary = vocabularies.vocabulary_from_codec(self.codec)
        self.output_features = {'inputs': {'dtype': 'float32', 'rank': 2}, 'targets': {'vocabulary': self.vocabulary}}

        self._parse_gin(gin_files)
        # restrict the instruments: the decoder may emit only the program events of `programs` (None: all) and no drum
        # events when drums=False -- a logit bias row (vocabularies.program_logit_bias) that every decode mode applies
        if programs is not None or not drums:
            self.logit_bias = vocabularies.program_logit_bias(self.codec, self._model_config().vocab_size, programs, drums)
        self.model = None
        self.restore_from_checkpoint(checkpoint_path)

    @property
    def input_shapes(self):
        return {
            'encoder_input_tokens': (self.batch_size, self.inputs_length),
            'decoder_input_tokens': (self.batch_size, self.outputs_length)
        }

    def _parse_gin(self, gin_files):
        """Parse gin files used to train the model (notebook :223-233)."""
        gin_bindings = [
            'VOCAB_CONFIG=@vocabularies.VocabularyConfig()',
            'vocabularies.VocabularyConfig.num_velocity_bins=%NUM_VELOCITY_BINS',
        ]
        cfg = gin_lite.parse_config_files_and_bindings(gin_files, gin_bindings)
        self._gin = cfg
        lengths = cfg.macro('TASK_FEATURE_LENGTHS')
        if lengths and lengths.get('inputs') != self.inputs_length:
            raise ValueError('gin TASK_FEATURE_LENGTHS %r disagrees with model_type inputs_length %d'
                             % (lengths, self.inputs_length))
        nvb = cfg.binding('vocabularies.VocabularyConfig', 'num_velocity_bins')
        if nvb is not None and nvb != vocabularies.num_velocity_bins_from_codec(self.codec):
            raise ValueError('gin NUM_VELOCITY_BINS=%r disagrees with the codec' % (nvb,))

    def _model_config(self) -> network.T5Config:
        p = dict(self._gin.params('network.T5Config'))
        vs = p.get('vocab_size')
        if isinstance(vs, gin_lite.Ref) or vs is None:       # @vocabularies.num_embeddings()
            p['vocab_size'] = vocabularies.num_embeddings(self.vocabulary)
        p['mlp_activations'] = tuple(p.get('mlp_activations', ('relu',)))
        p['input_depth'] = spectrograms.input_depth(self.spectrogram_config)
        return network.T5Config(**p)

    def _load_model(self, params: Dict[str, np.ndarray]):
        """Build the Transformer after parsing the gin config (notebook :235-245)."""
        model_config = self._model_config()
        return network.Transformer(model_config, params, device=self.device, max_batch=self.batch_size,
                                   max_input_length=self.inputs_length, max_decode_length=self.outputs_length,
                                   gemm_mode=self._gemm_mode, kv_format=self._kv_format)

    def restore_from_checkpoint(self, checkpoint_path):
        """Restore weights (notebook :247-262).  `checkpoint_path` is a .npz keyed by the Flax tree
        paths (mt3_b200.weights), a {path: array} dict, or 'synthetic[:SEED]' for random weights
        drawn from the reference's initialisers (the published checkpoints are unreachable offline)."""
        from . import distributed as mt3_dist
        rank, world_size = mt3_dist.world()
        params = None
        if rank == 0 or world_size == 1:
            if isinstance(checkpoint_path, dict):
                params = checkpoint_path
            elif isinstance(checkpoint_path, str) and checkpoint_path.startswith('synthetic'):
                seed = int(checkpoint_path.split(':', 1)[1]) if ':' in checkpoint_path else 0
                params = weights.synthetic_params(self._model_config(), seed)
            else:
                params = weights.load(checkpoint_path)
        # data-parallel (one process per GPU): only rank 0 reads the checkpoint; ONE broadcast at load
        params = mt3_dist.broadcast_params(params, self._model_config(), self.device, src=0)
        self.model = self._load_model(params)

    # ---------------------------------------------------------------------------------
    def predict_tokens(self, batch, seed=0):
        """Predict tokens from a preprocessed batch (notebook :277-281).  batch['encoder_input_tokens']
        float32 [B, T, 512] (numpy or torch).  Returns decoded ids np.int32 [B, 1024]: id-3, -1 from
        the first EOS on, -2 for invalid ids.  `seed` keys decode='sample' (row b draws from stream b); greedy and beam1
        ignore it, as decode_rng=None does (:268)."""
        x = batch['encoder_input_tokens']
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(self.device, non_blocking=True)
        prediction = self.model.generate(x, stop_at_eos=True, use_graph=self.use_graph, decode=self.decode, **self._sample_kw(seed, 0),
                                         **self._bias_kw())
        return self.vocabulary.decode_tf(prediction).cpu().numpy()

    def transcribe_segments(self, audio_segments, n_valid_frames=None, num_steps: Optional[int] = None,
                            stop_at_eos: bool = True, decoded: bool = True, return_scores: bool = False, prompts=None, seed=0,
                            segment_offset: int = 0):
        """Hot path end to end for already-cut segments: host float32 [S, inputs_length*hop] ->
        host int32 [S, 1024].  H2D copy, log-mel kernel, encoder, greedy decoder, (vocab decode),
        D2H copy; batches of `batch_size`.  This is the call bench.py's `e2e` times.
        return_scores=True returns (tokens, token_scores float32 [S, 1024], scores float32 [S]) with the same tokens: how sure
        the model was of each emitted token (its log-probability; 0 after EOS) and of each segment (Transformer.generate).
        prompts: host int [S, P], a forced start per segment (Transformer.generate's `prompt`), e.g. the tie section of
        segment_score_targets' decoder_target_tokens: the output rows start with them and decode on from there.
        seed (decode='sample'): segment s draws from stream segment_offset + s, so its tokens do not depend on batch_size,
        nor on how transcribe_segments_sharded splits the segments (it passes each shard's first global index)."""
        a = audio_segments
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(a)
        assert a.dim() == 2 and a.dtype == torch.float32
        if not a.is_cuda and not a.is_pinned():
            a = a.pin_memory()              # so that the per-batch H2D copies below are truly asynchronous
        S = a.shape[0]
        if prompts is not None:
            prompts = np.asarray(prompts)
            if prompts.ndim != 2 or prompts.shape[0] != S:
                raise ValueError('prompts must be [S=%d, P]; got shape %s' % (S, prompts.shape))
        out = torch.empty((S, self.outputs_length), dtype=torch.int32, pin_memory=True)
        if return_scores:
            out_ts = torch.empty((S, self.outputs_length), dtype=torch.float32, pin_memory=True)
            out_sc = torch.empty((S,), dtype=torch.float32, pin_memory=True)
        nv = None
        if n_valid_frames is not None:
            nv = torch.as_tensor(n_valid_frames, dtype=torch.int32).to(self.device)
        for s0 in range(0, S, self.batch_size):
            s1 = min(S, s0 + self.batch_size)
            dev = a[s0:s1].to(self.device, non_blocking=True)
            spec = spectrograms.compute_spectrogram(dev, self.spectrogram_config,
                                                    n_valid_frames=None if nv is None else nv[s0:s1])
            spec = self._pad_inputs(spec)
            toks = self.model.generate(spec, num_steps=num_steps, stop_at_eos=stop_at_eos, use_graph=self.use_graph,
                                       decode=self.decode, return_scores=return_scores,
                                       prompt=None if prompts is None else prompts[s0:s1],
                                       **self._sample_kw(seed, segment_offset + s0), **self._bias_kw())
            if return_scores:
                toks, ts, sc = toks
                out_ts[s0:s1].copy_(ts, non_blocking=True)
                out_sc[s0:s1].copy_(sc, non_blocking=True)
            if decoded:
                toks = self.vocabulary.decode_tf(toks)
            out[s0:s1].copy_(toks, non_blocking=True)
        torch.cuda.synchronize(self.device)
        if return_scores:
            return out.numpy(), out_ts.numpy(), out_sc.numpy()
        return out.numpy()

    def transcribe_segments_sharded(self, audio_segments, **kwargs):
        """Data-parallel transcribe_segments (SURVEY 8e): every rank passes the SAME global segment
        list, transcribes its contiguous shard on its own GPU and receives all token streams
        int32 [S, 1024] in segment order after ONE all-gather (three with return_scores=True: tokens, token scores
        and scores, as transcribe_segments returns them).  Identity with a single process."""
        if kwargs.get('prompts') is not None:
            raise ValueError('transcribe_segments_sharded does not take prompts; call transcribe_segments on each rank\'s segments')
        from . import distributed as mt3_dist
        rank, world_size = mt3_dist.world()
        a = audio_segments
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(a)
        S = a.shape[0]
        if world_size == 1:
            return self.transcribe_segments(a, **kwargs)
        lo, hi = mt3_dist.shard_range(S, rank, world_size)
        nv = kwargs.pop('n_valid_frames', None)
        if nv is not None:
            nv = np.asarray(nv)[lo:hi]
        scored = kwargs.get('return_scores', False)
        if hi > lo:
            local = self.transcribe_segments(a[lo:hi], n_valid_frames=nv, segment_offset=lo, **kwargs)
        else:
            empty = np.zeros((0, self.outputs_length), np.int32)
            local = (empty, empty.astype(np.float32), np.zeros((0,), np.float32)) if scored else empty
        if not scored:
            return mt3_dist.gather_tokens(torch.from_numpy(local).to(self.device), S).cpu().numpy()
        toks, ts, sc = local
        toks, ts, sc = (mt3_dist.gather_tokens(t.to(self.device), S).cpu().numpy()
                        for t in (torch.from_numpy(toks), torch.from_numpy(ts), torch.from_numpy(sc)[:, None]))
        return toks, ts, sc[:, 0]

    def _sample_kw(self, seed, row_offset: int) -> Dict:
        """generate's sampling arguments for a batch whose first row is segment row_offset (none unless decode='sample')"""
        if self.decode != 'sample':
            return {}
        return dict(self.sample_params, seed=seed, row_offset=row_offset)

    def _bias_kw(self) -> Dict:
        """generate's logit_bias argument (none unless programs= or drums=False restrict the instruments)"""
        return {} if self.logit_bias is None else {'logit_bias': self.logit_bias}

    def _pad_inputs(self, spec: torch.Tensor) -> torch.Tensor:
        """Feature converter (models.py:96): trim/pad the frame axis to inputs_length with 0.0."""
        t = spec.shape[1]
        if t == self.inputs_length:
            return spec
        if t > self.inputs_length:
            return spec[:, :self.inputs_length].contiguous()
        pad = torch.zeros((spec.shape[0], self.inputs_length - t, spec.shape[2]), dtype=spec.dtype, device=spec.device)
        return torch.cat([spec, pad], dim=1)

    def __call__(self, audio):
        """Infer note sequence from audio samples (notebook :283-308).

        audio: 1-d numpy array of audio samples (16kHz) for a single example.
        Returns the transcribed NoteSequence (mt3_b200.note_decoding.NoteSequence, the stand-in for
        note_seq's protobuf): segments are decoded on the GPU, their event tokens stitched on the host
        by event_predictions_to_ns exactly as the notebook does (:305-308)."""
        predictions = self.predict_segments(audio)
        result = note_decoding.event_predictions_to_ns(predictions, codec=self.codec, encoding_spec=self.encoding_spec)
        return result['est_ns']

    def predict_segments(self, audio):
        """audio -> list of per-segment predictions {'est_tokens', 'start_time', 'raw_inputs'} (the
        argument of metrics_utils.event_predictions_to_ns)."""
        ds = self.audio_to_dataset(audio)
        ds = self.preprocess(ds)
        hop = self.spectrogram_config.hop_width
        seg_len = self.inputs_length * hop
        segs = np.zeros((len(ds), seg_len), np.float32)
        n_valid = np.zeros((len(ds),), np.int32)
        for i, ex in enumerate(ds):
            flat = np.asarray(ex['inputs'], np.float32).reshape(-1)
            segs[i, :flat.size] = flat
            n_valid[i] = flat.size // hop
        # one process per GPU (torch.distributed initialised): every rank holds the same audio, transcribes its contiguous
        # shard of the segments and receives all token streams after one all-gather; identity with a single process
        tokens = self.transcribe_segments_sharded(segs, n_valid_frames=n_valid)
        return [self.postprocess(t, ex) for t, ex in zip(tokens, ds)]

    def score(self, audio, note_sequence) -> List[Dict]:
        """Log-likelihood of a labelled transcription given the audio, per segment: T5X score_batch over the segments the
        notebook's preprocessing cuts (same audio path as predict_segments: GPU log-mel with the valid-frame count, padding
        to inputs_length, encode; batches of batch_size), with targets from segment_score_targets.  Returns one dict per
        segment: 'start_time' (as postprocess rounds it), 'score' (sum of the token scores), 'num_tokens' (scored
        positions), 'token_scores' float32 [1024]."""
        frames, frame_times = self._audio_to_frames(audio)
        ds = self.preprocess([{'inputs': frames, 'input_times': frame_times}])
        tg = segment_score_targets(note_sequence, self.codec, self.vocabulary, frame_times, self.inputs_length,
                                   self.encoding_spec, self.outputs_length)
        if len(tg['decoder_target_tokens']) != len(ds):
            raise RuntimeError('segment count mismatch: %d target segments, %d audio segments'
                               % (len(tg['decoder_target_tokens']), len(ds)))
        hop = self.spectrogram_config.hop_width
        segs = np.zeros((len(ds), self.inputs_length * hop), np.float32)
        n_valid = np.zeros((len(ds),), np.int32)
        for i, ex in enumerate(ds):
            flat = np.asarray(ex['inputs'], np.float32).reshape(-1)
            segs[i, :flat.size] = flat
            n_valid[i] = flat.size // hop
        scores = np.zeros((len(ds), self.outputs_length), np.float32)
        nv = torch.from_numpy(n_valid).to(self.device)
        for s0 in range(0, len(ds), self.batch_size):
            s1 = min(len(ds), s0 + self.batch_size)
            dev = torch.from_numpy(segs[s0:s1]).to(self.device)
            spec = self._pad_inputs(spectrograms.compute_spectrogram(dev, self.spectrogram_config, n_valid_frames=nv[s0:s1]))
            encoded = self.model.encode(spec)
            ts = self.model.score(encoded, tg['decoder_input_tokens'][s0:s1], tg['decoder_target_tokens'][s0:s1],
                                  tg['decoder_loss_weights'][s0:s1])
            scores[s0:s1] = ts.cpu().numpy()
        out = []
        for i, ex in enumerate(ds):
            start_time = ex['input_times'][0]
            start_time -= start_time % (1 / self.codec.steps_per_second)
            out.append({'start_time': start_time, 'score': float(scores[i].astype(np.float64).sum()),
                        'num_tokens': int(tg['decoder_loss_weights'][i].sum()), 'token_scores': scores[i]})
        return out

    # ---------------------------------------------------------------------------------
    # Batch inference over many recordings (T5X `infer` with gin/infer.gin + inference.write_inferences_to_file)
    # ---------------------------------------------------------------------------------
    def build_infer_dataset(self, records):
        """records: [{'id': str, 'audio': float samples at 16 kHz}, ...] -> (task_ds, segments, n_valid_frames): the
        per-segment examples the reference's inference tasks produce (tasks.py:196-232: unique_id, input_times, the reference
        sequence -- here the id -- on the FIRST segment of a recording only) and the zero-padded audio of ALL segments of all
        recordings in one [S, inputs_length * hop] array, so that decode batches are filled across recordings."""
        hop = self.spectrogram_config.hop_width
        seg_len = self.inputs_length * hop
        task_ds, rows, n_valid = [], [], []
        for rec in records:
            first = True
            for ex in self.preprocess(self.audio_to_dataset(rec['audio'])):
                flat = np.asarray(ex['inputs'], np.float32).reshape(-1)
                row = np.zeros((seg_len,), np.float32)
                row[:flat.size] = flat
                rows.append(row)
                n_valid.append(flat.size // hop)
                task_ds.append({'unique_id': [rec['id']], 'input_times': ex['input_times'], 'raw_inputs': [],
                                'sequence': [rec['id'] if first else '']})
                first = False
        segs = np.stack(rows) if rows else np.zeros((0, seg_len), np.float32)
        return task_ds, segs, np.asarray(n_valid, np.int32)

    def infer_to_file(self, records, path: str) -> int:
        """Transcribe many recordings and write one JSON line of notes per recording ({'id', 'est_notes'}, the reference's
        inference.write_inferences_to_file format).  Segments of all recordings share the decode batches; under
        torch.distributed they are sharded over the GPUs and rank 0 writes.  Returns the number of segments decoded."""
        from . import distributed as mt3_dist
        task_ds, segs, n_valid = self.build_infer_dataset(records)
        if len(task_ds) == 0:
            inferences = np.zeros((0, self.outputs_length), np.int32)
        else:
            inferences = self.transcribe_segments_sharded(segs, n_valid_frames=n_valid, decoded=False)    # raw model ids
        if mt3_dist.world()[0] == 0:
            note_decoding.write_inferences_to_file(
                path, list(inferences), task_ds, 'predict', vocabulary=self.vocabulary,
                vocab_config=vocabularies.VocabularyConfig(num_velocity_bins=vocabularies.num_velocity_bins_from_codec(self.codec)),
                onsets_only=self.encoding_spec == 'NoteOnsetEncodingSpec', use_ties=self.encoding_spec == 'NoteEncodingWithTiesSpec')
        return len(task_ds)

    def audio_to_dataset(self, audio):
        """Create a dataset (list with one example) of frames from input audio (notebook :310-316)."""
        frames, frame_times = self._audio_to_frames(audio)
        return [{'inputs': frames, 'input_times': frame_times}]

    def _audio_to_frames(self, audio):
        """Compute spectrogram frames from audio (notebook :318-326): ALWAYS pads 1..hop samples."""
        frame_size = self.spectrogram_config.hop_width
        audio = np.asarray(audio, np.float32)
        padding = [0, frame_size - len(audio) % frame_size]
        audio = np.pad(audio, padding, mode='constant')
        frames = spectrograms.split_audio(audio, self.spectrogram_config)
        num_frames = len(audio) // frame_size
        times = np.arange(num_frames) / self.spectrogram_config.frames_per_second
        return frames, times

    def preprocess(self, ds):
        """split_tokens_to_inputs_length + add_dummy_targets (notebook :328-344): consecutive,
        non-overlapping chunks of inputs_length frames; the last one may be short.  The
        spectrogram itself is computed on the GPU in transcribe_segments (compute_spectrograms,
        preprocessors.py:613-618, runs per segment there too)."""
        out = []
        for ex in ds:
            frames, times = ex['inputs'], ex['input_times']
            for s in range(0, len(frames), self.inputs_length):
                out.append({'inputs': frames[s:s + self.inputs_length],
                            'input_times': times[s:s + self.inputs_length],
                            'targets': np.zeros((0,), np.int32)})
        return out

    def postprocess(self, tokens, example):
        tokens = self._trim_eos(tokens)
        start_time = example['input_times'][0]
        # Round down to nearest symbolic token step.
        start_time -= start_time % (1 / self.codec.steps_per_second)
        return {
            'est_tokens': tokens,
            'start_time': start_time,
            # Internal MT3 code expects raw inputs, not used here.
            'raw_inputs': []
        }

    @staticmethod
    def _trim_eos(tokens):
        tokens = np.array(tokens, np.int32)
        if vocabularies.DECODED_EOS_ID in tokens:
            tokens = tokens[:np.argmax(tokens == vocabularies.DECODED_EOS_ID)]
        return tokens
