"""K5 forward time of a nomic-embed-text encoder (rotary Q / K in the QKV epilogue, SwiGLU FFN1 epilogue) against the
same-shape BERT (one H100).

    python scripts/nomic_probe.py [--iters 20] [--warmup 3]

Prints the card and its power limit, then for the nomic-embed-text-v1.5 shape (12 layers x 768, 12 heads, FFN 3072, vocab
30528, 8192 positions, mean pooling) and the same-shape BERT (e5-base: vocab 30522, 512 positions, mean pooling), random
weights, at 256 x 32, 256 x 128, 64 x 512 and 4 x 8192 tokens (8192-token sequences: nomic only, BERT stops at 512): the
time per krag_embed_dev call from CUDA events on the consumer stream, the two models alternating on the same token ids
after warm-up, and the median of the paired differences.  Then, in a separate profiled pass (torch.profiler, CUDA
activity), the mean time of each gemm_f16s_kernel / splitk_reduce_kernel instantiation: EP = 1 is the rotary QKV, EP = 2
the gated FFN1, EP = 0 every BERT GEMM.  Last, the bar: torch's NomicBertModel (sdpa attention) on the same batches in fp32
and under bf16 autocast (CUDA events, same iterations)."""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPE = dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072)
NOMIC = dict(SHAPE, vocab_size=30528, max_position_embeddings=8192, type_vocab_size=2, layer_norm_eps=1e-12, rotary_base=1000.0)
BERT = dict(SHAPE, vocab_size=30522, max_position_embeddings=512, layer_norm_eps=1e-12)
SHAPES = [(256, 32), (256, 128), (64, 512), (4, 8192)]       # (sequences, tokens each)


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def nomic_hub_state(seed=0):
    """hub-named nomic weights: embeddings N(0, 0.02), matrices N(0, 0.06), LayerNorm gamma N(1, 0.1)"""
    g = np.random.default_rng(seed)
    d, i = NOMIC["hidden_size"], NOMIC["intermediate_size"]
    n = lambda std, *s, mean=0.0: (mean + std * g.standard_normal(s, dtype=np.float32)).astype(np.float32)   # noqa: E731
    st = {"embeddings.word_embeddings.weight": n(0.02, NOMIC["vocab_size"], d), "embeddings.token_type_embeddings.weight": n(0.02, 2, d),
          "emb_ln.weight": n(0.1, d, mean=1.0), "emb_ln.bias": n(0.05, d)}
    for l in range(NOMIC["num_hidden_layers"]):
        p = f"encoder.layers.{l}."
        st.update({p + "attn.Wqkv.weight": n(0.06, 3 * d, d), p + "attn.out_proj.weight": n(0.06, d, d),
                   p + "mlp.fc11.weight": n(0.06, i, d), p + "mlp.fc12.weight": n(0.06, i, d), p + "mlp.fc2.weight": n(0.06, d, i)})
        for ln in ("norm1", "norm2"):
            st[p + ln + ".weight"], st[p + ln + ".bias"] = n(0.1, d, mean=1.0), n(0.05, d)
    return st


def embedders(ctx):
    import bench
    from kaito_b200 import _native
    from kaito_b200.embedding import nomic_state
    out = {}
    for name, cfg in (("nomic", NOMIC), ("bert", BERT)):
        emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                               cfg["vocab_size"], cfg["max_position_embeddings"], 2, cfg["layer_norm_eps"])
        emb.set_pooling(_native.POOL_MEAN)
        if name == "nomic":
            emb.set_rotary(cfg["rotary_base"])
            emb.load_state_dict(nomic_state(nomic_hub_state(), cfg))
        else:
            emb.load_state_dict(bench.random_bert_state(cfg))
        out[name] = emb
    return out


def torch_bar(batches, iters, warmup):
    """ms per batch of torch's NomicBertModel (sdpa attention), fp32 and bf16 autocast, on the same token ids"""
    import torch
    from transformers import NomicBertConfig, NomicBertModel
    from tests.test_embed_nomic_cpu import native_state
    kw = {k: v for k, v in NOMIC.items() if k != "rotary_base"}
    m = NomicBertModel(NomicBertConfig(**kw, hidden_act="silu", rope_parameters={"rope_type": "default", "rope_theta": 1000.0},
                                       attn_implementation="sdpa")).cuda().eval()
    m.load_state_dict({k: torch.from_numpy(v) for k, v in native_state(nomic_hub_state()).items()}, strict=False)
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
        raise SystemExit("nomic_probe: no GPU")
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
        run = {k: e for k, e in embs.items() if S <= (NOMIC if k == "nomic" else BERT)["max_position_embeddings"]}
        for _ in range(args.warmup):
            for emb in run.values():
                emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
        ms = {k: [] for k in run}
        for _ in range(args.iters):
            for k, emb in run.items():
                # one call at a time on one stream, so the two models never overlap
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
                b.record(s)
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
        ms = {k: np.array(v) for k, v in ms.items()}
        line = f"K5 {B}x{S:<5d} ({B * S:6d} tok): nomic {np.median(ms['nomic']):8.3f} ms"
        if "bert" in ms:
            diff = ms["nomic"] - ms["bert"]
            line += (f"  bert {np.median(ms['bert']):8.3f} ms  nomic / bert {np.median(ms['nomic']) / np.median(ms['bert']):.3f}"
                     f"  nomic - bert median {np.median(diff) * 1e3:+9.1f} us")
        print(line)
        batches.append(((B, S), flat, offs, out, run))
    # profiled pass: kernel times only (tracing slows the host, so no call time is taken here)
    from torch.profiler import ProfilerActivity, profile
    for (B, S), flat, offs, out, run in batches:
        for k, emb in run.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    emb.embed_dev(flat, offs, out.data_ptr(), d, s.cuda_stream)
                s.synchronize()
            for e in prof.key_averages():
                if "gemm_f16s_kernel" in e.key or "splitk_reduce_kernel" in e.key:
                    us = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
                    print(f"kernel {B}x{S:<5d} {k:5s} {e.key[:60]:60s} {us:9.1f} us x {e.count}")
    for emb in embs.values():
        emb.destroy()
    ctx.close()
    for (B, S), (f32, b16) in torch_bar([((B, S), flat) for (B, S), flat, _, _, _ in batches], args.iters, args.warmup):
        print(f"torch NomicBertModel {B}x{S:<5d}: fp32 {f32:8.3f} ms  bf16 autocast {b16:8.3f} ms")


if __name__ == "__main__":
    main()
