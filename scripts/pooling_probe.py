"""K5 forward time with CLS and with mean pooling, at the shapes mean-pooled models run (one H100).

    python scripts/pooling_probe.py [--iters 20] [--warmup 3]

Prints the card and its power limit, then for all-MiniLM-L6 and e5-large (random weights, bench.random_bert_state) at 256
queries x 32 tokens and 256 /index chunks x 256 tokens (65,536 tokens): the time per krag_embed_dev call from CUDA events on
the consumer stream, CLS and mean alternating on the same inputs after warm-up, and the median of the paired differences.
Then, in a separate profiled pass (torch.profiler, CUDA activity), the mean time of the pooling kernels themselves."""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = {
    "all-MiniLM-L6": dict(num_hidden_layers=6, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522),
    "e5-large": dict(num_hidden_layers=24, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=30522),
}
SHAPES = [(256, 32), (256, 256)]       # (sequences, tokens each)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench
    from kaito_b200 import _native
    if not torch.cuda.is_available():
        raise SystemExit("pooling_probe: no GPU")
    print(f"card: {card()}")
    ctx = _native.Context(0)
    s = torch.cuda.Stream()
    modes = (("cls", _native.POOL_CLS), ("mean", _native.POOL_MEAN))
    cases = []
    for name, cfg in MODELS.items():
        emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"],
                               cfg["intermediate_size"], cfg["vocab_size"])
        emb.load_state_dict(bench.random_bert_state(cfg))
        for B, S in SHAPES:
            g = np.random.default_rng(B * S)
            flat, offs = _native.Embedder.pack([g.integers(1000, 30000, S) for _ in range(B)])
            out = torch.empty((B, cfg["hidden_size"]), dtype=torch.float32, device="cuda")
            for _ in range(args.warmup):
                for _, m in modes:
                    emb.set_pooling(m)
                    emb.embed_dev(flat, offs, out.data_ptr(), cfg["hidden_size"], s.cuda_stream)
            ev = {k: [] for k, _ in modes}
            for _ in range(args.iters):
                for k, m in modes:
                    emb.set_pooling(m)
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(s)
                    emb.embed_dev(flat, offs, out.data_ptr(), cfg["hidden_size"], s.cuda_stream)
                    b.record(s)
                    ev[k].append((a, b))
            s.synchronize()
            ms = {k: np.array([a.elapsed_time(b) for a, b in v]) for k, v in ev.items()}
            diff = ms["mean"] - ms["cls"]
            print(f"{name:14s} {B}x{S:<4d} ({B * S:6d} tok): cls {np.median(ms['cls']):8.3f} ms  mean {np.median(ms['mean']):8.3f} ms"
                  f"  mean - cls median {np.median(diff) * 1e3:+8.1f} us (min {diff.min() * 1e3:+.1f}, max {diff.max() * 1e3:+.1f})")
            cases.append((name, emb, flat, offs, out, cfg["hidden_size"]))
    # profiled pass: kernel times only (tracing slows the host, so no call time is taken here)
    from torch.profiler import ProfilerActivity, profile
    for name, emb, flat, offs, out, d in cases:
        for k, m in modes:
            emb.set_pooling(m)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
                s.synchronize()
            for e in prof.key_averages():
                if "normalize_kernel" in e.key:
                    us = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
                    print(f"kernel {name:14s} {len(offs) - 1}x{(int(offs[-1]) // (len(offs) - 1)):<4d} {k:4s} {e.key[:60]:60s} "
                          f"{us:8.1f} us x {e.count}")
    for c in cases[::len(SHAPES)]:
        c[1].destroy()
    ctx.close()


if __name__ == "__main__":
    main()
