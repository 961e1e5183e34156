"""Times prompted decoding: Transformer.generate with a prompt every row shares against the unprompted generate, at
bench.py's configuration (mt3, B = 64, T = 256, 1024 greedy steps without the early stop, TF32X3, 24-bit K/V rows, CUDA
graphs).

    python scripts/prompt_bench.py [--runs 5] [--warmup 1] [--prompt-lengths 0 16 64 256 768]

The prompts are the first P tokens of a greedy run of the same batch.  For each P three generates alternate in one process
(each after a 256 MB write, so that no run starts from the previous one's L2; CUDA events around the whole generate):
  unprompted   the plain generate;
  prefill      the shared prompt: one teacher-forced pass prefills P positions, the loop runs the rest;
  loop         the same prompt with row 0 emptied: the shared prefix is 0, so every prompt token is forced inside the loop
               (this is the other side of the prefill threshold, at the same number of loop steps per row).
The prefill pass alone is the prompted generate at num_steps = P (encoder, cross K/V, prefill, no loop step) minus the
generate at num_steps = 0.  Reports the median, min and max of each, and the card's name and power limit read in the same
call (nvidia-smi, read-only query).  Prints one JSON line."""
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
from mt3_b200 import _lib, inference, spectrograms  # noqa: E402
from oracle import mt3_oracle as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--prompt-lengths", type=int, nargs="+", default=[0, 16, 64, 256, 768])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prompt_bench needs a CUDA device")
    dev = "cuda:0"
    im = inference.InferenceModel('synthetic:0', 'mt3', device=dev, batch_size=args.batch, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format=_lib.KV_P24, use_graph=True)
    m = im.model
    audio = np.stack([O.sine_mix(256 * 128, seed=1234 + i) for i in range(args.batch)])
    spec = spectrograms.compute_spectrogram(torch.from_numpy(audio).to(dev), im.spectrogram_config)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    g = m.generate(spec, num_steps=args.steps, stop_at_eos=False).cpu().numpy()
    res = {"card": card(), "batch": args.batch, "steps": args.steps, "gemm": "TF32X3", "kv": "p24", "graphs": True,
           "greedy_rows_without_eos": int((~(g == 1).any(1)).sum())}

    def run(steps, prompt):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        m.generate(spec, num_steps=steps, stop_at_eos=False, use_graph=True, prompt=prompt)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    def stats(t):
        return {"median_ms": float(np.median(t)), "min_ms": float(min(t)), "max_ms": float(max(t))}

    for P in args.prompt_lengths:
        shared = np.ascontiguousarray(g[:, :P])
        shared[np.cumsum((shared == 1) | (shared == 0), 1) > 0] = 0     # a row that ended inside P is prompted up to its EOS
        ragged = shared.copy()
        ragged[0] = 0
        kinds = {"unprompted": (args.steps, None), "prefill": (args.steps, shared), "loop": (args.steps, ragged),
                 "prefill_only": (P, shared), "encode_only": (0, None)}
        if P == 0:
            kinds = {k: kinds[k] for k in ("unprompted", "prefill")}
        t = {k: [] for k in kinds}
        for _ in range(args.warmup):
            for k, (steps, prompt) in kinds.items():
                run(steps, prompt)
        for _ in range(args.runs):
            for k, (steps, prompt) in kinds.items():
                t[k].append(run(steps, prompt))
        r = {k: stats(v) for k, v in t.items()}
        if P:
            r["prefill_pass_ms"] = r["prefill_only"]["median_ms"] - r["encode_only"]["median_ms"]
            r["saving_vs_unprompted_ms"] = r["unprompted"]["median_ms"] - r["prefill"]["median_ms"]
            r["prefill_vs_loop_ms"] = r["loop"]["median_ms"] - r["prefill"]["median_ms"]
        res[f"P={P}"] = r
        print(json.dumps({f"P={P}": r}), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
