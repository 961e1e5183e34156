"""Times sampled decoding (Transformer.generate(decode='sample')) against greedy at bench.py's configuration (mt3, B = 64,
T = 256, 1024 steps without the early stop, TF32X3, 24-bit K/V rows, CUDA graphs), and the token pickers alone.

    python scripts/sample_bench.py [--runs 5] [--warmup 1] [--launches 2000]

Greedy and three sampled settings -- (T = 1), (T = 1, topk = 40), (T = 1, topp = 0.9) -- alternate in one process, each
generate after a 256 MB write so that no run starts from the previous one's L2, CUDA events around the whole generate;
medians, min and max over --runs after --warmup rounds.  The pickers alone: argmax_step_kernel and sample_step_kernel
(without filters, top-k 40, top-p 0.9, both) launched back to back through the kernel harness at B = 64, V = 1536, CUDA
events around --launches launches.  Reports the card's name and power limit read in the same call (nvidia-smi, read-only
query).  Prints one JSON line per part and one with everything."""
import argparse
import ctypes as C
import importlib.util
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

SETTINGS = {"greedy": None, "T1": dict(temperature=1.0), "T1_topk40": dict(temperature=1.0, topk=40),
            "T1_topp0.9": dict(temperature=1.0, topp=0.9)}


def stats(t):
    return {"median_ms": float(np.median(t)), "min_ms": float(min(t)), "max_ms": float(max(t))}


def generate_times(args, dev):
    im = inference.InferenceModel('synthetic:0', 'mt3', device=dev, batch_size=args.batch, gemm_mode=_lib.GEMM_TF32X3,
                                  kv_format=_lib.KV_P24, use_graph=True)
    m = im.model
    audio = np.stack([O.sine_mix(256 * 128, seed=1234 + i) for i in range(args.batch)])
    spec = spectrograms.compute_spectrogram(torch.from_numpy(audio).to(dev), im.spectrogram_config)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)

    def run(kw):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        if kw is None:
            m.generate(spec, num_steps=args.steps, stop_at_eos=False, use_graph=True)
        else:
            m.generate(spec, num_steps=args.steps, stop_at_eos=False, use_graph=True, decode='sample', seed=7, **kw)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    t = {k: [] for k in SETTINGS}
    for _ in range(args.warmup):
        for kw in SETTINGS.values():
            run(kw)
    for _ in range(args.runs):
        for k, kw in SETTINGS.items():
            t[k].append(run(kw))
    r = {k: stats(v) for k, v in t.items()}
    g = r["greedy"]["median_ms"]
    for k in SETTINGS:
        if k != "greedy":
            r[k]["vs_greedy_pct"] = 100.0 * (r[k]["median_ms"] - g) / g
            r[k]["extra_us_per_step"] = 1000.0 * (r[k]["median_ms"] - g) / args.steps
    return r


def picker_times(args, dev):
    spec = importlib.util.spec_from_file_location("build_tools", os.path.join(ROOT, "mt3_b200", "csrc", "tools", "build_tools.py"))
    bt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bt)
    if not os.path.exists(bt.HARNESS):
        raise SystemExit(f"{bt.HARNESS} not built: run __graft_entry__.build()")
    lib = C.CDLL(bt.HARNESS)
    P, I, F = C.c_void_p, C.c_int, C.c_float
    lib.kh_argmax_step.argtypes = [P, I, I, P, P, P, I, P, P, I, I, P, P, I, I, P, I]
    lib.kh_sample_step.argtypes = [P, I, I, P, P, P, P, I, P, P, P, I, F, P, P, I, I, P]
    B, V, D, N = args.batch, 1536, 512, args.launches
    rng = np.random.default_rng(0)
    lg = torch.from_numpy((rng.standard_normal((B, V)) * 2).astype(np.float32)).to(dev)
    lg[:, 1] = -float("inf")                                 # no row finishes: every launch does a full pick
    emb = torch.from_numpy(rng.standard_normal((V, D)).astype(np.float32)).to(dev)
    pe = torch.from_numpy(rng.standard_normal((N + 2, D)).astype(np.float32)).to(dev)
    y = torch.empty((B, D), dtype=torch.float32, device=dev)
    cur, fin = torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev)
    tok = torch.zeros((B, N), dtype=torch.int32, device=dev)
    state = torch.zeros(4, dtype=torch.int32, device=dev)

    def params(topk, topp):
        w = np.zeros(7, np.uint32)
        w[0] = np.float32(1.0).view(np.uint32)
        w[1], w[2] = topk, np.float32(topp).view(np.uint32)
        w[3], w[4], w[6] = 0, 7, 1
        return torch.from_numpy(w).to(dev)

    def time(launch):
        for _ in range(2):
            state.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(N):
                assert launch() == 0
            b.record()
            b.synchronize()
        return 1000.0 * a.elapsed_time(b) / N

    r = {"argmax": time(lambda: lib.kh_argmax_step(lg.data_ptr(), V, B, cur.data_ptr(), fin.data_ptr(), tok.data_ptr(), N, None,
                                                   state.data_ptr(), 1, 0, emb.data_ptr(), pe.data_ptr(), N + 2, D, y.data_ptr(), B))}
    for name, k, p in (("sample", 0, 0.0), ("sample_topk40", 40, 0.0), ("sample_topp0.9", 0, 0.9), ("sample_topk40_topp0.9", 40, 0.9)):
        sp = params(k, p)
        r[name] = time(lambda: lib.kh_sample_step(lg.data_ptr(), V, B, cur.data_ptr(), fin.data_ptr(), tok.data_ptr(), None, N,
                                                  None, state.data_ptr(), sp.data_ptr(), k, p, emb.data_ptr(), pe.data_ptr(), N + 2, D,
                                                  y.data_ptr()))
    return {"batch": B, "vocab": V, "launches": N, "us_per_launch": r}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device")
    dev = "cuda:0"
    res = {"card": card(), "batch": args.batch, "steps": args.steps, "gemm": "TF32X3", "kv": "p24", "graphs": True}
    res["pickers"] = picker_times(args, dev)
    print(json.dumps({"pickers": res["pickers"]}), flush=True)
    res["generate"] = generate_times(args, dev)
    print(json.dumps({"generate": res["generate"]}), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
