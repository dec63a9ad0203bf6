"""K5 forward time of an MPNet encoder (relative-position bias on every attention score) against the same-shape BERT (one H100).

    python scripts/mpnet_probe.py [--iters 20] [--warmup 3]

Prints the card and its power limit, then for the all-mpnet-base-v2 shape (12 layers x 768, 12 heads, FFN 3072, vocab
30527, 514 positions, mean pooling) and the same-shape BERT (e5-base: vocab 30522, 512 positions, mean pooling), random
weights (bench.random_bert_state; the MPNet table N(0, 1)), at 256 x 32, 256 x 128 and 64 x 384 tokens (384 is
all-mpnet-base-v2's max_seq_length): the time per krag_embed_dev call from CUDA events on the consumer stream (the stream idle
before each call, which returns when the embeddings are written), the two models alternating on the same token ids after
warm-up, and the median of the paired differences.  Then, in a separate
profiled pass (torch.profiler, CUDA activity), the mean time of attention_mma_kernel with REL (MPNet) and without (BERT).
Last, the bar: torch's MPNetModel on the same batches in fp32 and under bf16 autocast (CUDA events, same iterations)."""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPE = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072)
MPNET = dict(SHAPE, vocab_size=30527, max_position_embeddings=514, layer_norm_eps=1e-5)
BERT = dict(SHAPE, vocab_size=30522, max_position_embeddings=512, layer_norm_eps=1e-12)
SHAPES = [(256, 32), (256, 128), (64, 384)]       # (sequences, tokens each)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def mpnet_state(seed=0):
    """K5-named MPNet weights: bench.random_bert_state, 514 position rows, a zero token-type row, a N(0, 1) bias table"""
    import bench
    from kaito_b200.embedding import MPNET_REL_BIAS
    g = np.random.default_rng(seed + 1)
    st = bench.random_bert_state(MPNET, seed)
    d = MPNET["hidden_size"]
    st["embeddings.position_embeddings.weight"] = (0.02 * g.standard_normal((MPNET["max_position_embeddings"], d))).astype(np.float32)
    st["embeddings.token_type_embeddings.weight"] = np.zeros((1, d), np.float32)
    st[MPNET_REL_BIAS] = g.standard_normal((32, MPNET["num_attention_heads"])).astype(np.float32)
    return st


def embedders(ctx):
    import bench
    from kaito_b200 import _native
    out = {}
    for name, cfg in (("mpnet", MPNET), ("bert", BERT)):
        emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                               cfg["vocab_size"], cfg["max_position_embeddings"], 1 if name == "mpnet" else 2, cfg["layer_norm_eps"])
        emb.set_pooling(_native.POOL_MEAN)
        if name == "mpnet":
            emb.set_position_offset(2)
            emb.load_state_dict(mpnet_state())
        else:
            emb.load_state_dict(bench.random_bert_state(cfg))
        out[name] = emb
    return out


def torch_bar(batches, iters, warmup):
    """ms per batch of torch's MPNetModel (eager attention), fp32 and bf16 autocast, on the same token ids"""
    import torch
    from transformers import MPNetConfig, MPNetModel
    from kaito_b200.embedding import _MPNET_NAMES
    m = MPNetModel(MPNetConfig(**MPNET, relative_attention_num_buckets=32), add_pooling_layer=False).cuda().eval()
    inv = tuple((b, a) for a, b in _MPNET_NAMES)
    sd = {}
    for k, v in mpnet_state().items():
        if "token_type" in k:
            continue
        for a, b in inv:
            k = k.replace(a, b)
        sd[k] = torch.from_numpy(v)
    m.load_state_dict(sd, strict=False)
    res = []
    for (B, S), ids in batches:
        x = torch.as_tensor(ids.reshape(B, S).astype(np.int64), device="cuda")
        row = []
        for bf16 in (False, True):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                for _ in range(warmup):
                    m(input_ids=x)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    h = m(input_ids=x).last_hidden_state.mean(1)
                    torch.nn.functional.normalize(h, dim=1)
                b.record()
                b.synchronize()
            row.append(a.elapsed_time(b) / iters)
        res.append(((B, S), row))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from kaito_b200 import _native
    if not torch.cuda.is_available():
        raise SystemExit("mpnet_probe: no GPU")
    print(f"card: {card()}")
    ctx = _native.Context(0)
    s = torch.cuda.Stream()
    embs = embedders(ctx)
    d = SHAPE["hidden_size"]
    batches = []
    for B, S in SHAPES:
        g = np.random.default_rng(B * S)
        flat, offs = _native.Embedder.pack([g.integers(1000, 30000, S) for _ in range(B)])
        out = torch.empty((B, d), dtype=torch.float32, device="cuda")
        for _ in range(args.warmup):
            for emb in embs.values():
                emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
        ms = {k: [] for k in embs}
        for _ in range(args.iters):
            for k, emb in embs.items():
                # each embedder forwards on its own stream: one call at a time, so the two models never overlap
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
                b.record(s)
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
        ms = {k: np.array(v) for k, v in ms.items()}
        diff = ms["mpnet"] - ms["bert"]
        print(f"K5 {B}x{S:<4d} ({B * S:6d} tok): bert {np.median(ms['bert']):8.3f} ms  mpnet {np.median(ms['mpnet']):8.3f} ms"
              f"  mpnet - bert median {np.median(diff) * 1e3:+8.1f} us (min {diff.min() * 1e3:+.1f}, max {diff.max() * 1e3:+.1f})")
        batches.append(((B, S), flat, offs, out))
    # profiled pass: kernel times only (tracing slows the host, so no call time is taken here)
    from torch.profiler import ProfilerActivity, profile
    for (B, S), flat, offs, out in batches:
        for k, emb in embs.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
                s.synchronize()
            for e in prof.key_averages():
                if "attention_mma_kernel" in e.key:
                    us = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
                    rel = "REL" if "true>" in e.key else "   "
                    print(f"kernel {B}x{S:<4d} {k:5s} {rel} {e.key[:70]:70s} {us:8.1f} us x {e.count}")
    for emb in embs.values():
        emb.destroy()
    ctx.close()
    for (B, S), (f32, b16) in torch_bar([((B, S), flat) for (B, S), flat, _, _ in batches], args.iters, args.warmup):
        print(f"torch MPNetModel {B}x{S:<4d}: fp32 {f32:8.3f} ms  bf16 autocast {b16:8.3f} ms")


if __name__ == "__main__":
    main()
