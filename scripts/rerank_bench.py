"""Cross-encoder reranking throughput on the GPU: krag_rerank (K5 + classifier head + top-k) at the MiniLM-L6 / L12
cross-encoder shapes, random weights, 256 queries x N candidates, passages of fixed length; and the same pairs through torch
BertForSequenceClassification (padded batches, SDPA) in fp32 and bf16 as the bar.  Prints one JSON line per point (--out:
also the list of them as a JSON file).

  python scripts/rerank_bench.py [--models L6,L12] [--n 10,30,100] [--lens 128,256,480] [--reps 3] [--out file]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = {"L6": 6, "L12": 12}


def flops(cfg, lens):
    """forward FLOPs of the encoder over sequences of the given lengths (GEMMs 24 S d^2 + 4 S^2 d per layer incl. FFN 4d), plus
    the pooler and classifier (2 d^2 + 2 d per pair)"""
    d, i, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    per = sum(L * (2 * s * (4 * d * d + 2 * d * i) + 4 * s * s * d) for s in lens)
    return per + len(lens) * (2 * d * d + 2 * d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="L6,L12")
    ap.add_argument("--n", default="10,30,100")
    ap.add_argument("--lens", default="128,256,480")
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from kaito_b200 import _native
    from kaito_b200.rerank import build_pairs
    from tests.test_gpu_rerank import _encoder, _state
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(device_id=0)
    rows = []
    for mk in a.models.split(","):
        cfg = dict(num_hidden_layers=MODELS[mk], hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522,
                   max_position_embeddings=512)
        state = _state(cfg, "bench")
        enc = _encoder(ctx, cfg, state)
        tm = {}
        if not a.no_torch:
            from transformers import BertConfig, BertForSequenceClassification
            m = BertForSequenceClassification(BertConfig(**cfg, num_labels=1, attn_implementation="sdpa"))
            sd = {(k if k.startswith("classifier.") else "bert." + k): torch.from_numpy(v) for k, v in state.items()}
            m.load_state_dict(sd, strict=False)
            tm = {"fp32": m.cuda().eval(), "bf16": __import__("copy").deepcopy(m).to(torch.bfloat16).cuda().eval()}
        for n in map(int, a.n.split(",")):
            for plen in map(int, a.lens.split(",")):
                g = np.random.default_rng(n + plen)
                qs = [(g.integers(1000, 30000, 12).astype(np.int32), 12) for _ in range(a.queries)]
                ds = [[(g.integers(1000, 30000, plen).astype(np.int32), plen) for _ in range(n)] for _ in range(a.queries)]
                flat, toff, seg, poff = build_pairs(2, 3, qs, ds, 512)
                n_pairs, n_tok = int(poff[-1]), int(toff[-1])
                fl = flops(cfg, np.diff(toff).tolist())
                enc.rerank(poff, flat, toff, seg, 10)                  # warm-up (graphs are captured on the second sight)
                enc.rerank(poff, flat, toff, seg, 10)
                t = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    enc.rerank(poff, flat, toff, seg, 10)              # returns synchronised
                    t.append(time.perf_counter() - t0)
                s = float(np.median(t))
                row = {"model": f"MiniLM-{mk}", "queries": a.queries, "N": n, "passage_tokens": plen, "pairs": n_pairs, "tokens": n_tok,
                       "krag_ms": s * 1e3, "pairs_per_s": n_pairs / s, "tokens_per_s": n_tok / s, "tflops_fp32_equiv": fl / s / 1e12,
                       "gpu": gpu}
                for name, m in tm.items():
                    L = int(np.diff(toff).max())
                    ids = torch.zeros((n_pairs, L), dtype=torch.int64)
                    tt = torch.zeros_like(ids); mask = torch.zeros_like(ids)
                    for p in range(n_pairs):
                        s0, s1 = int(toff[p]), int(toff[p + 1])
                        ids[p, :s1 - s0] = torch.from_numpy(flat[s0:s1].astype(np.int64))
                        tt[p, int(seg[p]):s1 - s0] = 1; mask[p, :s1 - s0] = 1
                    ids, tt, mask = ids.cuda(), tt.cuda(), mask.cuda()
                    bs = max(1, 65536 // L)

                    def run():
                        with torch.no_grad():
                            for b0 in range(0, n_pairs, bs):
                                m(input_ids=ids[b0:b0 + bs], token_type_ids=tt[b0:b0 + bs], attention_mask=mask[b0:b0 + bs])
                    run(); torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.reps):
                        run()
                    e1.record(); torch.cuda.synchronize()
                    row[f"torch_{name}_ms"] = e0.elapsed_time(e1) / a.reps
                print(json.dumps(row), flush=True)
                rows.append(row)
        enc.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
