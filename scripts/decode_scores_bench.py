"""Times what decode scores cost: Transformer.generate with and without return_scores at bench.py's configuration (mt3,
B = 64, T = 256, 1024 greedy / beam1 steps without the early stop, TF32X3, 24-bit K/V rows, CUDA graphs).

    python scripts/decode_scores_bench.py [--runs 5] [--warmup 1] [--decode greedy beam1]

Scored and unscored runs alternate in one process (A B A B ...), each after a 256 MB write so that no run starts from the
previous one's L2, with CUDA events around the whole generate (encoder, cross K/V, the decode loop, the finalize and the
copies out).  Reports the median, min and max of each and the median overhead.  The card's name and power limit are read
in the same call (nvidia-smi, read-only query).  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mt3_b200 import _lib, inference, spectrograms  # noqa: E402
from oracle import mt3_oracle as O  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--decode", nargs="+", default=["greedy", "beam1"], choices=["greedy", "beam1"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_scores_bench needs a CUDA device")
    dev = "cuda:0"
    im = inference.InferenceModel('synthetic:0', 'mt3', device=dev, batch_size=args.batch, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format=_lib.KV_P24, use_graph=True)
    audio = np.stack([O.sine_mix(256 * 128, seed=1234 + i) for i in range(args.batch)])
    spec = spectrograms.compute_spectrogram(torch.from_numpy(audio).to(dev), im.spectrogram_config)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    res = {"card": card(), "batch": args.batch, "steps": args.steps, "gemm": "TF32X3", "kv": "p24", "graphs": True}

    def run(decode, scored):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        im.model.generate(spec, num_steps=args.steps, stop_at_eos=False, use_graph=True, decode=decode, return_scores=scored)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for decode in args.decode:
        for _ in range(args.warmup):
            run(decode, False)
            run(decode, True)
        t = {False: [], True: []}
        for _ in range(args.runs):
            for scored in (False, True):
                t[scored].append(run(decode, scored))
        plain, scored = np.median(t[False]), np.median(t[True])
        res[decode] = {"unscored_ms": float(plain), "unscored_ms_min_max": [min(t[False]), max(t[False])],
                       "scored_ms": float(scored), "scored_ms_min_max": [min(t[True]), max(t[True])],
                       "overhead_ms": float(scored - plain), "overhead_pct": float(100 * (scored - plain) / plain)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
