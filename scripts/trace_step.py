"""Device timeline of one greedy decode step (mt3_debug_trace_step): per graph node start / duration / gap to
the previous node, and the internal phase split of CTA (0,0).  Run on a GPU box:  python scripts/trace_step.py

GEMM phases (us after CTA (0,0) started): PDL wait returned (a node launched under the GEMM before it starts early and waits
there), weights landed and split into hi / lo tiles (tensor modes only, else 0), activations landed, multiply done,
partials exchanged, reduce + epilogue issued.  Attention phases: first K tile landed, pass 1, softmax, pass 2, exit."""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mt3_b200 import _lib, inference  # noqa: E402

SM_GHZ = 1.98      # H100 SXM maximum SM clock
GEMM_WORDS = [6, 7, 2, 3, 4, 5]      # trace words of a GEMM slot in phase order (decode.cuh dec_cluster_body)
ATTN_WORDS = [2, 3, 4, 5, 6, 7]      # attention slot; word 7 is unused


def main():
    B = int(os.environ.get("TRACE_B", "64"))
    dev = torch.device("cuda:0")
    kv = {"f32": _lib.KV_F32, "f16": _lib.KV_F16, "p24": _lib.KV_P24}[os.environ.get("TRACE_KV", "p24")]
    im = inference.InferenceModel("synthetic:0", "mt3", device=dev, batch_size=B, kv_format=kv)
    rng = np.random.default_rng(0)
    audio = torch.from_numpy((0.1 * rng.standard_normal((B, 32768))).astype(np.float32))
    im.transcribe_segments(audio, num_steps=8, stop_at_eos=False)        # encoder state, cross K/V, warm
    lib = _lib.load()
    h = im.model._h
    stream = torch.cuda.current_stream(dev).cuda_stream
    out = np.zeros((256, 16), np.uint64)
    names = C.create_string_buffer(16384)
    n = C.c_int32(0)
    for pos in [int(p) for p in os.environ.get("TRACE_POS", "32,512,1000").split(",")]:
        _lib.check(lib.mt3_debug_trace_step(h, pos, out.ctypes.data_as(C.c_void_p), 256, names, 16384, C.byref(n), stream))
        nm = names.value.decode().split("\n")[:n.value]
        t = out[:n.value].astype(np.int64)
        t0 = t[0, 0]
        print(f"\n== decode step at cache position {pos}: {n.value} traced nodes (B={B})")
        print(f"{'node':18s} {'start':>8s} {'dur':>7s} {'gap':>6s} | CTA(0,0) phases us: "
              "gemm: wait weights loads compute exchange reduce | attn: first-K pass1 softmax pass2 exit -")
        prev_end = t0
        agg = {}
        for i in range(n.value):
            st, en = t[i, 0], t[i, 1]
            ph = t[i, GEMM_WORDS if nm[i].startswith('gemm') else ATTN_WORDS] / (SM_GHZ * 1e3)
            dur, gap = (en - st) / 1e3, (st - prev_end) / 1e3
            a = agg.setdefault(nm[i], [0, 0.0, 0.0, np.zeros(6)])
            a[0] += 1; a[1] += dur; a[2] += gap; a[3] += ph
            if i < 8 and nm[i].startswith('gemm'):
                print(f"{'':18s} SMs of tile 0's cluster (rank 0..7): " + ' '.join(str(int(x)) for x in t[i, 8:16]))
            if i < int(os.environ.get('TRACE_ROWS', '10')) or i >= n.value - 3:
                print(f"{nm[i]:18s} {(st - t0) / 1e3:8.2f} {dur:7.2f} {gap:6.2f} | " + " ".join(f"{x:6.2f}" for x in ph))
            prev_end = en
        total = (t[-1, 1] - t0) / 1e3
        print(f"-- step span (first traced start -> last traced end): {total:.1f} us")
        print(f"{'node':18s} {'count':>5s} {'dur avg':>8s} {'gap avg':>8s} {'dur sum':>8s} {'gap sum':>8s} | mean phases")
        for k, (c, d, g, ph) in agg.items():
            print(f"{k:18s} {c:5d} {d / c:8.2f} {g / c:8.2f} {d:8.1f} {g:8.1f} | " + " ".join(f"{x / c:6.2f}" for x in ph))
        dsum = sum(v[1] for v in agg.values()); gsum = sum(v[2] for v in agg.values())
        print(f"-- sum of node durations {dsum:.1f} us, sum of gaps {gsum:.1f} us")


if __name__ == "__main__":
    main()
