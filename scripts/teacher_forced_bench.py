"""Times the teacher-forced decoder pass (mt3_decode_teacher_forced: Transformer.decode(decode=False) and
Transformer.score) at B = 64, T = 256, L = 1024 in gemm modes TF32X3 and SIMT, and compares it in the same run with the
step path on the same tokens (teacher_forced_logits: one decode step per position, on an MT3_KV_F32 model).

    python scripts/teacher_forced_bench.py [--iters 5] [--warmup 2]

CUDA events around each pass, warm-up first, a 256 MB write between runs so that no run starts from the previous one's
L2.  The algorithmic work is computed from the shapes (flops()); TFLOP/s are over the measured time and compared with the
H100 SXM data-sheet dense TF32 rate, 495 TFLOP/s, which TF32X3 spends three MMAs per product of (hi.hi + hi.lo + lo.hi).
The card's name and power limit are read in the same call (nvidia-smi, read-only query).  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from mt3_b200 import _lib, network, weights  # noqa: E402

TF32_DENSE_TFLOPS = 495.0          # H100 SXM data sheet, dense TF32 (700 W card)


def flops(B, T, L, D=512, H=6, F=1024, V=1536, layers=8):
    """Algorithmic FLOP of one pass: decoder GEMMs per token, causal self-attention (the lower triangle), cross-attention
    over T keys, and the per-layer cross K/V projection of `encoded`."""
    Q = H * 64
    gemm = B * L * (layers * 2 * (D * 3 * Q + Q * D + D * Q + Q * D + D * 2 * F + F * D) + 2 * D * V)
    self_attn = layers * B * H * 2 * 2 * 64 * (L * (L + 1) / 2)
    cross_attn = layers * B * H * 2 * 2 * 64 * L * T
    cross_kv = layers * 2 * B * T * D * 2 * Q
    return dict(gemm=gemm, self_attn=self_attn, cross_attn=cross_attn, cross_kv=cross_kv,
                total=gemm + self_attn + cross_attn + cross_kv)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_ms(fn, iters, warmup, flush):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--input-length", type=int, default=256)
    ap.add_argument("--length", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("teacher_forced_bench needs a CUDA device")
    B, T, L = args.batch, args.input_length, args.length
    cfg = network.T5Config(vocab_size=1536, emb_dim=512, num_heads=6, num_encoder_layers=8, num_decoder_layers=8, head_dim=64, mlp_dim=1024,
                           mlp_activations=('gelu', 'linear'))
    params = weights.synthetic_params(cfg, 0)
    rng = np.random.default_rng(0)
    dev = "cuda:0"
    enc = torch.from_numpy(rng.standard_normal((B, T, 512)).astype(np.float32)).to(dev)
    tgt = torch.from_numpy(rng.integers(3, 1536, size=(B, L)).astype(np.int32)).to(dev)
    din = torch.cat([torch.zeros((B, 1), dtype=torch.int32, device=dev), tgt[:, :-1]], dim=1).contiguous()
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)
    fl = flops(B, T, L)
    res = {"card": card(), "batch": B, "input_length": T, "length": L, "tflop": fl["total"] / 1e12,
           "tflop_parts": {k: v / 1e12 for k, v in fl.items() if k != "total"}}
    for name, gm in (("tf32x3", _lib.GEMM_TF32X3), ("simt", _lib.GEMM_FP32_SIMT)):
        m = network.Transformer(cfg, params, device=dev, max_batch=B, max_input_length=T, max_decode_length=L, gemm_mode=gm,
                                kv_format=_lib.KV_F32)
        logits_ms = time_ms(lambda: m.decode(enc, None, din, tgt, decode=False), args.iters, args.warmup, flush)
        score_ms = time_ms(lambda: m.score(enc, din, tgt), args.iters, args.warmup, flush)
        r = {"logits_ms": logits_ms[0], "logits_ms_min_max": logits_ms[1:], "score_ms": score_ms[0], "score_ms_min_max": score_ms[1:],
             "tflops": fl["total"] / 1e12 / (score_ms[0] / 1e3)}
        r["fraction_of_tf32_datasheet"] = r["tflops"] / TF32_DENSE_TFLOPS
        if name == "tf32x3":
            r["note"] = "3 tf32 MMAs per product (hi.hi + hi.lo + lo.hi); the rate counts algorithmic FLOP only"
            pass_logits = m.decode(enc, None, din, tgt, decode=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step_logits = m.teacher_forced_logits(enc, din)
            torch.cuda.synchronize()
            r["step_path_ms"] = (time.perf_counter() - t0) * 1e3
            r["step_path_vs_pass_max_rel_dlogit"] = float((pass_logits - step_logits).abs().max() / step_logits.abs().max())
            del pass_logits, step_logits
        res[name] = r
        del m
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
