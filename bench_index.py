#!/usr/bin/env python
"""bench_index.py -- the /index path (BASELINE.json configs[4], SURVEY.md section 8 a12 / C5): batch-embed chunks with K5
(bge-base shapes, random-init weights), append rows + term lists to the index, commit (postings + tile index).

    python bench_index.py [--chunks N] [--seq S]                               one GPU
    python -m torch.distributed.run --nproc-per-node G ... bench_index.py ...   G GPUs: the chunks are dealt to the ranks
                                                                               (data parallel, one all-reduce of BM25
                                                                               statistics at commit)

Reports chunks/s per stage and end to end (max over ranks, CUDA-synchronised wall clock), the K5 rate, and -- the bar
SURVEY.md section 2.3 sets for K5 -- the same forward through torch's own bf16 BertModel (SDPA attention, cuBLAS GEMMs) on
the same GPU.  Not the /retrieve bench (that is bench.py); prints one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from kaito_b200 import _native  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--chunks", type=int, default=16384, help="chunks over ALL ranks")
ap.add_argument("--seq", type=int, default=256)
ap.add_argument("--model", default="bge-base")
ap.add_argument("--embed-batch", type=int, default=128, help="chunks per K5 call")
ap.add_argument("--no-torch", action="store_true", help="skip the torch bf16 BertModel comparison")
a = ap.parse_args()

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

world, rank, lr = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
cfg = bench.BGE[a.model]
ctx = _native.Context(lr, rank=rank, world_size=world)
emb = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"], cfg["vocab_size"])
emb.load_state_dict(bench.random_bert_state(cfg))
n_local = a.chunks // world + (1 if rank < a.chunks % world else 0)
g = np.random.default_rng(rank)
toks = [g.integers(1000, 30000, a.seq) for _ in range(a.embed_batch)]
emb.embed(toks)                                   # warm-up (graph capture on second use)
emb.embed(toks)


def sync():
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()


def tmax(t):
    if world == 1:
        return t
    x = torch.tensor([t], dtype=torch.float64, device=dev)
    dist.all_reduce(x, op=dist.ReduceOp.MAX)
    return float(x.item())


sync()
t0 = time.perf_counter()
vecs = []
for b0 in range(0, n_local, a.embed_batch):
    vecs.append(emb.embed(toks[: min(a.embed_batch, n_local - b0)]))
torch.cuda.synchronize()
t_embed = tmax(time.perf_counter() - t0)
vecs = np.concatenate(vecs)
# sparse side: ~80 unique terms per chunk from a 2^18 vocabulary (host tokenisation is not timed here)
vocab = 1 << 18
offs = np.arange(0, (n_local + 1) * 80, 80, dtype=np.int64)
tids = g.integers(0, vocab, n_local * 80).astype(np.uint32)
tf = np.ones(n_local * 80, np.uint16)
dl = np.full(n_local, 96, np.uint32)
ix = ctx.create_index("idx", cfg["hidden_size"])
sync()
t0 = time.perf_counter()
ix.add(np.arange(n_local, dtype=np.uint64), vecs, offs, tids, tf, dl)
t_add = tmax(time.perf_counter() - t0)
sync()
t0 = time.perf_counter()
if world > 1:
    from kaito_b200.sharded import NativeStages, ShardedRetriever
    ShardedRetriever(NativeStages(ctx, ix), dev, ix.stats().dim_padded).commit(vocab, n_local)
else:
    ix.commit(vocab)
torch.cuda.synchronize()
t_commit = tmax(time.perf_counter() - t0)

torch_ref = None
if not a.no_torch and rank == 0:
    # The bars for K5 on the same GPU, same shapes, same batch, device tensors in (no host copy).  SURVEY.md section 2.3 names
    # torch + cuBLAS bf16 BertModel (SDPA); bf16 carries 8 mantissa bits (~4e-3 on the embedding), K5 is fp32-accurate
    # (~3e-7), so the same model is also timed in torch's strict fp32 (TF32 off: the arithmetic K5 matches) and in TF32.
    from transformers import BertConfig, BertModel
    ids = torch.from_numpy(np.stack(toks)).to(dev)
    torch_ref = {}
    for label, dtype, tf32 in (("bf16_sdpa", torch.bfloat16, True), ("tf32_sdpa", torch.float32, True), ("fp32_strict_sdpa", torch.float32, False)):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch.backends.cudnn.allow_tf32 = tf32
        m = BertModel(BertConfig(**cfg, attn_implementation="sdpa"), add_pooling_layer=False).to(dev).to(dtype).eval()
        with torch.no_grad():
            for _ in range(2):
                torch.nn.functional.normalize(m(input_ids=ids).last_hidden_state[:, 0].float(), dim=1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            reps = 5
            for _ in range(reps):
                torch.nn.functional.normalize(m(input_ids=ids).last_hidden_state[:, 0].float(), dim=1)
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) / reps
        torch_ref[label] = {"chunks_per_s": a.embed_batch / dt, "ms_per_batch": dt * 1e3,
                            "tflops": bench.bert_flops(cfg, a.seq) * a.embed_batch / dt / 1e12}
        del m
    torch_ref["what"] = "transformers.BertModel + SDPA (cuBLAS / flash kernels) in bf16, TF32 and strict fp32"

if rank == 0:
    fl = bench.bert_flops(cfg, a.seq) * a.chunks
    peaks = json.load(open("MEASURED_PEAKS.json")) if os.path.exists("MEASURED_PEAKS.json") else {}
    f16_peak = float(peaks.get("bf16_tflops_sustained", peaks.get("bf16_tflops", 989.0)))   # else the H100 SXM data sheet (dense bf16)
    k5_rate = a.chunks / t_embed
    print(json.dumps({
        "metric": "index_chunks_per_sec", "unit": "chunks/s", "n_gpus": world, "data": "synthetic", "scaling": "strong",
        "config": {"workload": f"/index: {a.chunks} chunks x {a.seq} tokens, {a.model} shapes (random-init), 80 terms/chunk, vocab 2^18",
                   "embed_batch": a.embed_batch, "parallelism": f"chunks dealt to {world} rank(s); BM25 statistics all-reduced at commit"},
        "value": a.chunks / (t_embed + t_add + t_commit),
        "embed": {"chunks_per_s": k5_rate, "chunks_per_s_per_gpu": k5_rate / world, "tflops_fp32_equivalent": fl / t_embed / 1e12,
                  "tensor_frac_of_f16_peak_per_gpu": 3.0 * fl / t_embed / 1e12 / world / f16_peak,
                  "arithmetic": "split-fp16 operands, 3 fp16 wgmma per step (fp32-accurate); includes D2H of the embeddings",
                  "flops_formula": "L*(24*S*d^2 + 4*S^2*d) per chunk (SURVEY.md 8d)"},
        "torch_same_gpu": torch_ref,
        "k5_vs_torch": None if torch_ref is None else {k: (k5_rate / world) / v["chunks_per_s"] for k, v in torch_ref.items() if isinstance(v, dict)},
        "add_chunks_per_s": a.chunks / t_add, "commit_s": t_commit,
    }), flush=True)
sync()
ix.drop(); emb.destroy(); ctx.close()
if world > 1:
    dist.destroy_process_group()
