"""Times a 1024-step generate with a logit bias (Transformer.generate(logit_bias=...)) against the same generate without
one, at bench.py's configuration (mt3, B = 64, T = 256, 1024 steps without the early stop, TF32X3, 24-bit K/V rows, CUDA
graphs), for greedy, beam-size-1 and sampled (T = 1) decoding.

    python scripts/logit_bias_bench.py [--runs 5] [--warmup 1]

Per decode mode three settings alternate in one process: unbiased, a zero bias [V], and a program mask (programs 0 and 1,
no drums; vocabularies.program_logit_bias).  Each generate runs after a 256 MB write so that no run starts from the
previous one's L2, with CUDA events around the whole generate; medians, min and max over --runs after --warmup rounds.
A biased generate also copies and checks its bias rows once before the encoder (one kernel and an 8-byte copy back).
Reports the card's name and power limit read in the same call (nvidia-smi, read-only query).  Prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from decode_scores_bench import card  # noqa: E402
from mt3_b200 import _lib, inference, spectrograms, vocabularies  # noqa: E402
from oracle import mt3_oracle as O  # noqa: E402

MODES = {"greedy": dict(decode='greedy'), "beam1": dict(decode='beam1'), "sample": dict(decode='sample', temperature=1.0, seed=7)}


def stats(t):
    return {"median_ms": float(np.median(t)), "min_ms": float(min(t)), "max_ms": float(max(t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logit_bias_bench needs a CUDA device")
    dev = "cuda:0"
    im = inference.InferenceModel('synthetic:0', 'mt3', device=dev, batch_size=args.batch, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format=_lib.KV_P24, use_graph=True)
    m = im.model
    V = m.config.vocab_size
    audio = np.stack([O.sine_mix(256 * 128, seed=1234 + i) for i in range(args.batch)])
    spec = spectrograms.compute_spectrogram(torch.from_numpy(audio).to(dev), im.spectrogram_config)
    biases = {"unbiased": None, "zero": np.zeros(V, np.float32),
              "program_mask": vocabularies.program_logit_bias(im.codec, V, programs=[0, 1], drums=False)}
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)

    def run(kw, bias):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        extra = {} if bias is None else {"logit_bias": bias}
        a.record()
        m.generate(spec, num_steps=args.steps, stop_at_eos=False, use_graph=True, **kw, **extra)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    res = {"card": card(), "batch": args.batch, "steps": args.steps, "gemm": "TF32X3", "kv": "p24", "graphs": True, "runs": args.runs}
    for mode, kw in MODES.items():
        t = {k: [] for k in biases}
        for _ in range(args.warmup):
            for bias in biases.values():
                run(kw, bias)
        for _ in range(args.runs):
            for k, bias in biases.items():
                t[k].append(run(kw, bias))
        r = {k: stats(v) for k, v in t.items()}
        base = r["unbiased"]["median_ms"]
        for k in ("zero", "program_mask"):
            r[k]["vs_unbiased_pct"] = 100.0 * (r[k]["median_ms"] - base) / base
        res[mode] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
