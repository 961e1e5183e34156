"""Audio file in, MIDI file out: the notebook's three cells (upload audio -> transcribe -> download MIDI,
colab/music_transcription_with_transformers.ipynb) as one command.

    python -m mt3_b200.transcribe input.wav output.mid --checkpoint CKPT [--model mt3|ismir2021]
           [--batch-size 64] [--decode greedy|beam1] [--jsonl notes.jsonl] [--device cuda:0]
           [--programs 0,1,...] [--no-drums]

CKPT is what InferenceModel.restore_from_checkpoint takes: a .npz keyed by the Flax tree paths, a T5X checkpoint
directory (mt3_b200.checkpoints), or 'synthetic[:SEED]' for random weights (plumbing runs only -- the published
checkpoints at gs://mt3/checkpoints are unreachable offline).  Launched under torch.distributed.run the segments are
sharded over the GPUs (InferenceModel.predict_segments) and rank 0 writes the files.  --programs and --no-drums restrict
the instruments the decoder may emit (InferenceModel's programs= and drums=), e.g. `--programs 0 --no-drums` for solo piano.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from typing import List, Optional

SAMPLE_RATE = 16000          # the notebook's SAMPLE_RATE; spectrograms.DEFAULT_SAMPLE_RATE


def _parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog='python -m mt3_b200.transcribe', description=__doc__.split('\n\n')[0])
    ap.add_argument('audio', help='input WAV file (any rate / channel count; resampled to 16 kHz mono)')
    ap.add_argument('midi', help='output Standard MIDI file')
    ap.add_argument('--checkpoint', required=True, help=".npz / T5X checkpoint directory / 'synthetic[:SEED]'")
    ap.add_argument('--model', default='mt3', choices=['mt3', 'ismir2021'])
    ap.add_argument('--batch-size', type=int, default=64, help='segments per decode batch (the notebook uses 8)')
    ap.add_argument('--decode', default='greedy', choices=['greedy', 'beam1'])
    ap.add_argument('--device', default=None, help="default: cuda:LOCAL_RANK")
    ap.add_argument('--jsonl', default=None, help='also write the notes as one JSON line (the T5X-infer style record)')
    ap.add_argument('--programs', type=_programs, default=None,
                    help='comma-separated MIDI programs (0-127) the decoder may emit; default: every program')
    ap.add_argument('--no-drums', dest='drums', action='store_false', help='the decoder emits no drum events')
    return ap


def _programs(text: str) -> List[int]:
    try:
        programs = [int(p) for p in text.split(',')]
    except ValueError:
        raise argparse.ArgumentTypeError('expected comma-separated integers, got %r' % text)
    bad = [p for p in programs if not 0 <= p <= 127]
    if bad:
        raise argparse.ArgumentTypeError('MIDI programs lie in 0..127; got %s' % bad)
    return programs


def main(argv: Optional[List[str]] = None) -> int:
    args = _parser().parse_args(argv)
    from . import audio_io
    try:
        audio = audio_io.load_audio(args.audio, SAMPLE_RATE)
    except (OSError, audio_io.AudioIOError) as e:
        print('transcribe: cannot read %s: %s' % (args.audio, e), file=sys.stderr)
        return 2
    import torch
    if not torch.cuda.is_available():
        print('transcribe: mt3_b200 needs a CUDA device (sm_90a); there is no CPU fallback', file=sys.stderr)
        return 3
    from . import distributed as mt3_dist, inference, note_decoding
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    device = args.device or 'cuda:%d' % local
    torch.cuda.set_device(torch.device(device))
    if world > 1 and not torch.distributed.is_initialized():
        torch.distributed.init_process_group('nccl', device_id=torch.device(device))
    rank, _ = mt3_dist.world()
    model = inference.InferenceModel(args.checkpoint, args.model, device=device, batch_size=args.batch_size, decode=args.decode,
                                     programs=args.programs, drums=args.drums)
    est_ns = model(audio)
    if rank == 0:
        note_decoding.note_sequence_to_midi_file(est_ns, args.midi)
        if args.jsonl:
            with open(args.jsonl, 'w') as f:
                f.write(json.dumps({'id': os.path.basename(args.audio),
                                    'est_notes': [note_decoding.note_to_dict(n) for n in est_ns.notes]}) + '\n')
        # the counts the notebook logs after transcription
        print(json.dumps({'audio_seconds': round(len(audio) / SAMPLE_RATE, 3),
                          'numNotes': sum(1 for n in est_ns.notes if not n.is_drum),
                          'numDrumNotes': sum(1 for n in est_ns.notes if n.is_drum),
                          'numPrograms': len({n.program for n in est_ns.notes if not n.is_drum}),
                          'midi': args.midi}))
    if world > 1:
        torch.distributed.barrier()
    return 0


if __name__ == '__main__':
    sys.exit(main())
