"""Model vocabulary: the token-id contract of the reference's vocabularies.py.

No seqio/t5 here: `GenericTokenVocabulary` keeps the reference's public behaviour
(vocabularies.py:148-277) -- ids shifted by 3 special tokens (0 PAD, 1 EOS, 2 UNK), EOS
sticky on decode, everything outside the regular range decoded as invalid -- for numpy
arrays, torch CPU tensors and (through the CUDA kernel) torch CUDA tensors.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Callable, Optional, Sequence

import numpy as np
import torch

from . import event_codec

DECODED_EOS_ID = -1
DECODED_INVALID_ID = -2

# defaults for vocabulary config (vocabularies.py:34-36)
DEFAULT_STEPS_PER_SECOND = 100
DEFAULT_MAX_SHIFT_SECONDS = 10
DEFAULT_NUM_VELOCITY_BINS = 127

# t5.data.DEFAULT_EXTRA_IDS (third party; used at vocabularies.py:145)
DEFAULT_EXTRA_IDS = 100

# note_seq constants used by build_codec (vocabularies.py:119-140)
MIN_MIDI_PITCH, MAX_MIDI_PITCH = 0, 127
MIN_MIDI_PROGRAM, MAX_MIDI_PROGRAM = 0, 127
MAX_MIDI_VELOCITY = 127

NUM_SPECIAL_TOKENS = 3     # 0=PAD, 1=EOS, 2=UNK: model id = codec index + 3


@dataclasses.dataclass
class VocabularyConfig:
    """Vocabulary configuration parameters (vocabularies.py:39-55)."""
    steps_per_second: int = DEFAULT_STEPS_PER_SECOND
    max_shift_seconds: int = DEFAULT_MAX_SHIFT_SECONDS
    num_velocity_bins: int = DEFAULT_NUM_VELOCITY_BINS

    @property
    def abbrev_str(self):
        s = ''
        if self.steps_per_second != DEFAULT_STEPS_PER_SECOND:
            s += 'ss%d' % self.steps_per_second
        if self.max_shift_seconds != DEFAULT_MAX_SHIFT_SECONDS:
            s += 'ms%d' % self.max_shift_seconds
        if self.num_velocity_bins != DEFAULT_NUM_VELOCITY_BINS:
            s += 'vb%d' % self.num_velocity_bins
        return s


def num_velocity_bins_from_codec(codec: event_codec.Codec):
    lo, hi = codec.event_type_range('velocity')
    return hi - lo


def velocity_to_bin(velocity, num_velocity_bins):
    return 0 if velocity == 0 else math.ceil(num_velocity_bins * velocity / MAX_MIDI_VELOCITY)


def bin_to_velocity(velocity_bin, num_velocity_bins):
    return 0 if velocity_bin == 0 else int(MAX_MIDI_VELOCITY * velocity_bin / num_velocity_bins)


def drop_programs(tokens, codec: event_codec.Codec):
    """Drops program change events from a token sequence (vocabularies.py:77-80)."""
    tokens = np.asarray(tokens)
    lo, hi = codec.event_type_range('program')
    return tokens[(tokens < lo) | (tokens > hi)]


def programs_to_midi_classes(tokens, codec: event_codec.Codec):
    """Program events -> the first program of their MIDI class of 8 (vocabularies.py:83-90)."""
    tokens = np.asarray(tokens)
    lo, hi = codec.event_type_range('program')
    return np.where((tokens >= lo) & (tokens <= hi), lo + 8 * ((tokens - lo) // 8), tokens)


@dataclasses.dataclass
class ProgramGranularity:
    """How programs are collapsed in token streams and in NoteSequences; both maps are idempotent (vocabularies.py:93-97)."""
    tokens_map_fn: Callable
    program_map_fn: Callable[[int], int]


PROGRAM_GRANULARITIES = {
    'flat': ProgramGranularity(tokens_map_fn=drop_programs, program_map_fn=lambda program: 0),            # no program tokens
    'midi_class': ProgramGranularity(tokens_map_fn=programs_to_midi_classes, program_map_fn=lambda program: 8 * (program // 8)),
    'full': ProgramGranularity(tokens_map_fn=lambda tokens, codec: np.asarray(tokens), program_map_fn=lambda program: program),
}


def build_codec(vocab_config: VocabularyConfig):
    """Build event codec (vocabularies.py:119-140): pitch | velocity | tie | program | drum."""
    event_ranges = [
        event_codec.EventRange('pitch', MIN_MIDI_PITCH, MAX_MIDI_PITCH),
        event_codec.EventRange('velocity', 0, vocab_config.num_velocity_bins),   # bin 0 = note-off
        event_codec.EventRange('tie', 0, 0),
        event_codec.EventRange('program', MIN_MIDI_PROGRAM, MAX_MIDI_PROGRAM),
        event_codec.EventRange('drum', MIN_MIDI_PITCH, MAX_MIDI_PITCH),
    ]
    return event_codec.Codec(
        max_shift_steps=vocab_config.steps_per_second * vocab_config.max_shift_seconds,
        steps_per_second=vocab_config.steps_per_second,
        event_ranges=event_ranges)


class GenericTokenVocabulary:
    """Vocabulary with pass-through encoding of tokens (vocabularies.py:148-277)."""

    def __init__(self, regular_ids: int, extra_ids: int = 0):
        self._num_special_tokens = NUM_SPECIAL_TOKENS
        self._num_regular_tokens = regular_ids
        self.extra_ids = extra_ids

    @property
    def pad_id(self) -> int:
        return 0

    @property
    def eos_id(self) -> Optional[int]:
        return 1

    @property
    def unk_id(self) -> Optional[int]:
        return 2

    @property
    def _base_vocab_size(self) -> int:
        return self._num_special_tokens + self._num_regular_tokens

    @property
    def vocab_size(self) -> int:
        return self._base_vocab_size + self.extra_ids

    def encode(self, token_ids: Sequence[int]) -> Sequence[int]:
        out = []
        for t in token_ids:
            if not 0 <= t < self._num_regular_tokens:
                raise ValueError(f'token_id {t} does not fall within valid range of [0, {self._num_regular_tokens})')
            out.append(int(t) + self._num_special_tokens)
        return out

    def decode(self, ids: Sequence[int]) -> Sequence[int]:
        """List form (vocabularies.py:193-217 behind seqio's decode, which cuts at the first EOS):
        ids up to and including the first EOS; EOS -> -1, invalid -> -2."""
        out = []
        for i in ids:
            i = int(i)
            if i == self.eos_id:
                out.append(DECODED_EOS_ID)
                break
            if i < self._num_special_tokens or i >= self._base_vocab_size:
                out.append(DECODED_INVALID_ID)
            else:
                out.append(i - self._num_special_tokens)
        return out

    def decode_tf(self, ids):
        """_decode_tf (vocabularies.py:241-271): elementwise along the last axis, EOS and
        everything after it -> -1, out-of-range -> -2.  CUDA int32 tensors run the kernel."""
        if isinstance(ids, torch.Tensor) and ids.is_cuda:
            from . import _lib
            lib = _lib.load()
            x = ids.to(torch.int32).contiguous()
            flat = x.reshape(-1, x.shape[-1])
            out = torch.empty_like(flat)
            with torch.cuda.device(x.device):
                _lib.check(lib.mt3_vocab_decode(flat.data_ptr(), flat.shape[0], flat.shape[1], self._num_regular_tokens,
                                                out.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream))
            return out.reshape(x.shape)
        a = ids.numpy() if isinstance(ids, torch.Tensor) else np.asarray(ids)
        eos_and_after = np.cumsum((a == self.eos_id).astype(np.int32), axis=-1) > 0
        valid = (a >= self._num_special_tokens) & (a < self._base_vocab_size)
        out = np.where(eos_and_after, DECODED_EOS_ID,
                       np.where(valid, a - self._num_special_tokens, DECODED_INVALID_ID)).astype(np.int32)
        return torch.from_numpy(out) if isinstance(ids, torch.Tensor) else out

    def encode_tf(self, token_ids):
        a = np.asarray(token_ids)
        if (a < 0).any() or (a >= self._num_regular_tokens).any():
            raise ValueError('token ids outside [0, %d)' % self._num_regular_tokens)
        return a + self._num_special_tokens

    def __eq__(self, other):
        return (self.extra_ids == other.extra_ids and self._num_regular_tokens == other._num_regular_tokens)


def vocabulary_from_codec(codec: event_codec.Codec) -> GenericTokenVocabulary:
    return GenericTokenVocabulary(codec.num_classes, extra_ids=DEFAULT_EXTRA_IDS)


def program_logit_bias(codec: event_codec.Codec, vocab_size: int, programs: Optional[Sequence[int]] = None,
                       drums: bool = True) -> np.ndarray:
    """A logit bias float32 [vocab_size] for Transformer.generate that restricts the instruments: 0 everywhere except -inf at
    the model id (codec index + the vocabulary's 3 special ids) of every `program` event whose MIDI program is not in
    `programs` (None: every program allowed), and of the whole `drum` range when drums=False."""
    if vocab_size < codec.num_classes + NUM_SPECIAL_TOKENS:
        raise ValueError(f'vocab_size {vocab_size} is smaller than the codec\'s {codec.num_classes} ids + {NUM_SPECIAL_TOKENS}')
    bias = np.zeros(vocab_size, np.float32)
    if programs is not None:
        programs = [int(p) for p in programs]
        bad = [p for p in programs if not MIN_MIDI_PROGRAM <= p <= MAX_MIDI_PROGRAM]
        if bad:
            raise ValueError(f'programs must lie in [{MIN_MIDI_PROGRAM}, {MAX_MIDI_PROGRAM}]; got {bad}')
        lo, hi = codec.event_type_range('program')
        keep = np.zeros(hi - lo + 1, bool)
        keep[np.asarray(programs, np.int64) - MIN_MIDI_PROGRAM] = True
        bias[lo + NUM_SPECIAL_TOKENS:hi + 1 + NUM_SPECIAL_TOKENS][~keep] = -np.inf
    if not drums:
        lo, hi = codec.event_type_range('drum')
        bias[lo + NUM_SPECIAL_TOKENS:hi + 1 + NUM_SPECIAL_TOKENS] = -np.inf
    return bias


def num_embeddings(vocabulary: GenericTokenVocabulary) -> int:
    """Vocabulary size as a multiple of 128 (vocabularies.py:280-282)."""
    return 128 * math.ceil(vocabulary.vocab_size / 128)
