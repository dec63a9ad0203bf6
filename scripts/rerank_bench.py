"""Cross-encoder reranking throughput on the GPU: krag_rerank (K5 + classifier head + top-k) at the MiniLM-L6 / L12
cross-encoder shapes and the bge-reranker-base / -large (XLM-RoBERTa, vocabulary 250,002) shapes, random weights, 256 queries x
N candidates, passages of fixed length; and the same pairs through torch BertForSequenceClassification (padded batches, SDPA)
in fp32 and bf16, or XLMRobertaForSequenceClassification in fp32 and under bf16 autocast, as the bar.  --tokenize: host time
of the XLM-R Unigram tokeniser on a 256-query batch and on 7,680 passages, native (ASCII) against the Python restatement, on a
tokenizer trained from tests/xlmr_reference's corpus and padded with synthetic pieces to 250,002 entries.  The precision modes of K5 (--precision) are
timed in the same call on the same inputs, alternating, after a warm-up of each; with both, the row also carries the mean
top-10 overlap of their results.  Prints one JSON line per point (--out: also the list of them as a JSON file), each with the
card name and power limit read in this call.  --profile DIR: instead of timing, one call per mode and point under
torch.profiler, per-kernel CUDA times written to DIR/rerank_profile_<mode>.txt.

  python scripts/rerank_bench.py [--models L6,L12,bge-base,bge-large] [--n 10,30,100] [--lens 128,256,480]
                                 [--precision fp32,fp16] [--reps 3] [--out file] [--profile dir] [--tokenize]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MODELS = {"L6": 6, "L12": 12}
XLMR = {"bge-base": "bge-reranker-base", "bge-large": "bge-reranker-large"}


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
    ap.add_argument("--precision", default="fp32,fp16")
    ap.add_argument("--profile", default=None)
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--tokenize", action="store_true")
    a = ap.parse_args()
    modes = a.precision.split(",")
    if not modes or any(m not in ("fp32", "fp16") for m in modes) or a.reps < 1:
        ap.error("--precision takes fp32, fp16 or both; --reps >= 1")
    import torch
    from kaito_b200 import _native
    from kaito_b200.rerank import build_pairs
    from tests.test_gpu_rerank import _encoder, _state
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = _native.Context(device_id=0)
    rows = []
    if a.tokenize:
        rows.append(tokenize_row(gpu))
    for mk in [m for m in a.models.split(",") if m]:
        xlmr = mk in XLMR
        if xlmr:
            from tests import test_gpu_rerank_xlmr as tx, xlmr_reference as xr
            cfg = xr.encoder_config(XLMR[mk])
            state = xr.k5_state(cfg, "random")
            enc = tx._encoder(ctx, cfg, state)
        else:
            cfg = dict(num_hidden_layers=MODELS[mk], hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522,
                       max_position_embeddings=512)
            state = _state(cfg, "bench")
            enc = _encoder(ctx, cfg, state)
        tm = {}
        if xlmr and not a.no_torch and not a.profile:
            from transformers import XLMRobertaConfig, XLMRobertaForSequenceClassification
            m = XLMRobertaForSequenceClassification(XLMRobertaConfig(**cfg, num_labels=1, pad_token_id=1, layer_norm_eps=1e-5,
                                                                     attn_implementation="sdpa"))
            m.load_state_dict({k: torch.from_numpy(v) for k, v in xr.hf_state(state).items()}, strict=False)
            tm = {"fp32": m.cuda().eval(), "bf16_autocast": m}
        elif not a.no_torch and not a.profile:
            from transformers import BertConfig, BertForSequenceClassification
            m = BertForSequenceClassification(BertConfig(**cfg, num_labels=1, attn_implementation="sdpa"))
            sd = {(k if k.startswith("classifier.") else "bert." + k): torch.from_numpy(v) for k, v in state.items()}
            m.load_state_dict(sd, strict=False)
            tm = {"fp32": m.cuda().eval(), "bf16": __import__("copy").deepcopy(m).to(torch.bfloat16).cuda().eval()}
        for n in map(int, a.n.split(",")):
            for plen in map(int, a.lens.split(",")):
                g = np.random.default_rng(n + plen)
                lo, hi = (4, cfg["vocab_size"]) if xlmr else (1000, 30000)
                qs = [(g.integers(lo, hi, 12).astype(np.int32), 12) for _ in range(a.queries)]
                ds = [[(g.integers(lo, hi, plen).astype(np.int32), plen) for _ in range(n)] for _ in range(a.queries)]
                flat, toff, seg, poff = build_pairs(0, 2, qs, ds, 512, 2) if xlmr else build_pairs(2, 3, qs, ds, 512)
                n_pairs, n_tok = int(poff[-1]), int(toff[-1])
                fl = flops(cfg, np.diff(toff).tolist())
                for mode in modes:                                     # warm-up (graphs are captured on the second sight)
                    enc.set_precision(mode)
                    enc.rerank(poff, flat, toff, seg, 10)
                    enc.rerank(poff, flat, toff, seg, 10)
                if a.profile:
                    profile(enc, modes, (poff, flat, toff, seg, 10), a.profile, f"{XLMR.get(mk, 'MiniLM-' + mk)} N={n} passage={plen}")
                    continue
                t, top = {mode: [] for mode in modes}, {}
                for _ in range(a.reps):
                    for mode in modes:                                 # alternating: both modes see the same minutes of the card
                        enc.set_precision(mode)
                        t0 = time.perf_counter()
                        top[mode] = enc.rerank(poff, flat, toff, seg, 10)[0]      # returns synchronised
                        t[mode].append(time.perf_counter() - t0)
                row = {"model": XLMR.get(mk, f"MiniLM-{mk}"), "queries": a.queries, "N": n, "passage_tokens": plen, "pairs": n_pairs, "tokens": n_tok}
                for mode in modes:
                    s = float(np.median(t[mode]))
                    sfx = "" if mode == "fp32" else "_fp16"
                    row.update({f"krag{sfx}_ms": s * 1e3, f"pairs_per_s{sfx}": n_pairs / s, f"tokens_per_s{sfx}": n_tok / s,
                                f"tflops_fp32_equiv{sfx}": fl / s / 1e12})
                if len(modes) == 2:
                    row["top10_overlap"] = float(np.mean([len(set(x.tolist()) & set(y.tolist())) / 10.0
                                                          for x, y in zip(top["fp32"], top["fp16"])]))
                row["gpu"] = gpu
                for name, m in tm.items():
                    L = int(np.diff(toff).max())
                    ids = torch.full((n_pairs, L), 1 if xlmr else 0, dtype=torch.int64)      # XLM-R pads with pad_token_id 1
                    tt = torch.zeros_like(ids); mask = torch.zeros_like(ids)
                    for p in range(n_pairs):
                        s0, s1 = int(toff[p]), int(toff[p + 1])
                        ids[p, :s1 - s0] = torch.from_numpy(flat[s0:s1].astype(np.int64))
                        mask[p, :s1 - s0] = 1
                        if seg is not None:
                            tt[p, int(seg[p]):s1 - s0] = 1
                    ids, tt, mask = ids.cuda(), tt.cuda(), mask.cuda()
                    bs = max(1, 65536 // L)

                    def run():
                        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=name == "bf16_autocast"):
                            for b0 in range(0, n_pairs, bs):
                                if xlmr:
                                    m(input_ids=ids[b0:b0 + bs], attention_mask=mask[b0:b0 + bs])
                                else:
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
    if a.out and not a.profile:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


def tokenize_row(gpu):
    """host seconds of UnigramTokenizer.encode_batch_plain on 256 queries and on 7,680 passages (30 per query): the native
    ASCII path against the Python restatement (median of 3 native calls, one Python pass)"""
    import tempfile
    from kaito_b200.text import UnigramTokenizer, read_unigram_json
    from tests import xlmr_reference as xr
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(xr.train_tokenizer(tmp, seed=0), "tokenizer.json")
        tj = json.load(open(path, encoding="utf-8"))
        g = np.random.default_rng(0)
        have = {p for p, _ in tj["model"]["vocab"]}
        extra = []
        while len(tj["model"]["vocab"]) + len(extra) < xr.VOCAB:
            w = ("▁" if g.random() < 0.5 else "") + "".join(g.choice(list("abcdefghijklmnopqrstuvwxyz"), int(g.integers(2, 9))))
            if w not in have:
                have.add(w)
                extra.append([w, float(g.uniform(-14.0, -8.0))])
        mask = tj["model"]["vocab"].pop()                          # <mask> stays the last id
        tj["model"]["vocab"] += extra + [mask]
        for t in tj["added_tokens"]:
            if t["content"] == "<mask>":
                t["id"] = len(tj["model"]["vocab"]) - 1
        with open(path, "w", encoding="utf-8") as f:
            json.dump(tj, f, ensure_ascii=False)
        tok = UnigramTokenizer(read_unigram_json(path), max_length=512)
    words = ["the", "quick", "brown", "fox", "retrieval", "engine", "query", "passage", "gpu", "token", "kubernetes", "inference"]
    queries = [" ".join(g.choice(words, 12)) + "?" for _ in range(256)]
    passages = [" ".join(g.choice(words, 100)) + "." for _ in range(7680)]
    row = {"tokenizer": f"Unigram, {len(tok.pieces)} pieces", "gpu": gpu}
    for label, texts in (("queries_256", queries), ("passages_7680", passages)):
        for path_name, fn in (("native", tok.encode_batch_plain), ("python", lambda ts: [tok.encode_py(t) for t in ts])):
            ts = []
            for _ in range(3 if path_name == "native" else 1):     # the Python path takes seconds on the passages
                t0 = time.perf_counter()
                fn(texts)
                ts.append(time.perf_counter() - t0)
            row[f"{label}_{path_name}_ms"] = float(np.median(ts)) * 1e3
        assert [x.tolist() for x in tok.encode_batch_plain(texts[:64])] == [tok.encode_py(t) for t in texts[:64]]
    print(json.dumps(row), flush=True)
    return row


def profile(enc, modes, call, out_dir, label):
    """per-kernel CUDA time of one krag_rerank call per mode (tracing slows the host: no end-to-end time is taken here)"""
    from torch.profiler import ProfilerActivity, profile as torch_profile
    os.makedirs(out_dir, exist_ok=True)
    for mode in modes:
        enc.set_precision(mode)
        with torch_profile(activities=[ProfilerActivity.CUDA]) as prof:
            enc.rerank(*call)
        with open(os.path.join(out_dir, f"rerank_profile_{mode}.txt"), "a") as f:
            f.write(f"== {label} {mode}\n{prof.key_averages().table(sort_by='cuda_time_total', row_limit=12, max_name_column_width=60)}\n")


if __name__ == "__main__":
    main()
