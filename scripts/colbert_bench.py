"""Late-interaction (ColBERT) reranking on the GPU: krag_late_rerank at the colbertv2.0 shape (12 x 768, dim 128) and the
answerai-colbert-small shape (12 x 384, dim 96), random weights, 256 queries of 32 rows (12 real tokens, [MASK] expansion,
attend_to_mask_tokens false) x N distinct candidates of a fixed token count (passage rows incl. [CLS] [D] ... [SEP], 15 % of
them on the skiplist).  Per point:
  - krag time per call (host clock around the call, which returns synchronised), both precision modes alternating in one
    process after a warm-up of each, median of --reps;
  - maxsim_kernel alone: torch.profiler CUDA time of the kernel in one call per mode, in a run of its own after the timing;
  - the same computation restated in torch on the same GPU (BertModel with SDPA on padded batches and ColBERT's attention
    mask, projection, F.normalize, masked MaxSim) in fp32 and in bf16 (model weights in bf16), CUDA events, one warm-up;
  - --cross-encoder: the MiniLM-L6 cross-encoder row of scripts/rerank_bench.py (krag_rerank, same queries x N x passage
    tokens, both modes) for reference, in a process of its own.
Every row carries the card's name, power limit and max SM clock read in this call.  Prints one JSON line per point.

  python scripts/colbert_bench.py [--shapes colbertv2.0,answerai-colbert-small] [--n 10,30] [--lens 128,180] [--reps 3]
                                  [--no-torch] [--cross-encoder] [--out file]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

QL, REAL = 32, 12


def inputs(g, n_queries, n, plen):
    """(query ids [n_queries, QL], key counts, passage ids, offsets, keep mask, pair offsets, pair -> passage): every query
    has its own n passages of plen rows"""
    q = np.full((n_queries, QL), 103, np.int32)
    q[:, 0], q[:, 1], q[:, REAL + 2] = 101, 1, 102
    q[:, 2:REAL + 2] = g.integers(1000, 30000, (n_queries, REAL))
    keys = np.full(n_queries, REAL + 3, np.int32)
    n_pass = n_queries * n
    p = g.integers(1000, 30000, (n_pass, plen)).astype(np.int32)
    p[:, 0], p[:, 1], p[:, -1] = 101, 2, 102
    keep = (g.random((n_pass, plen)) > 0.15).astype(np.uint8)
    keep[:, 0] = 1
    d_off = np.arange(0, n_pass * plen + 1, plen, dtype=np.int32)
    poff = np.arange(0, n_pass + 1, n, dtype=np.int32)
    return q, keys, p.reshape(-1), d_off, keep.reshape(-1), poff, np.arange(n_pass, dtype=np.int32)


def maxsim_profile(e, args, modes):
    """CUDA time (ms) of maxsim_kernel in one call per mode, under torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for mode in modes:
        e.set_precision(mode)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.late_rerank(*args)
        us = [getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
              for ev in prof.key_averages() if "maxsim_kernel" in ev.key]
        out[mode] = float(sum(us)) / 1e3 if us else None
    return out


def torch_restatement(cfg, state, w, q, keys, p_ids, keep, n, plen, dtype):
    """ms of one call restated in torch on the GPU: encoder (SDPA, padded; queries with ColBERT's key mask), projection,
    normalisation, masked MaxSim; returns (ms, scores [n_queries, n])"""
    import torch
    from transformers import BertConfig, BertModel
    m = BertModel(BertConfig(**cfg, attn_implementation="sdpa"), add_pooling_layer=False)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()}, strict=False)
    m = m.to(dtype).cuda().eval()
    W = torch.from_numpy(w).to(dtype).cuda()
    qi = torch.from_numpy(q.astype(np.int64)).cuda()
    qm = (torch.arange(QL)[None] < torch.from_numpy(keys.astype(np.int64))[:, None]).long().cuda()
    pi = torch.from_numpy(p_ids.astype(np.int64).reshape(-1, plen)).cuda()
    pk = torch.from_numpy(keep.reshape(-1, plen).astype(bool)).cuda()
    bs = max(1, 65536 // plen)

    def run():
        with torch.no_grad():
            Q = torch.nn.functional.normalize(m(input_ids=qi, attention_mask=qm).last_hidden_state @ W.T, dim=-1)
            D = torch.cat([torch.nn.functional.normalize(m(input_ids=pi[b:b + bs]).last_hidden_state @ W.T, dim=-1)
                           for b in range(0, pi.shape[0], bs)])
            D = D.view(q.shape[0], n, plen, -1)
            s = torch.einsum("qid,qnjd->qnij", Q.float(), D.float())
            s = s.masked_fill(~pk.view(q.shape[0], n, 1, plen), float("-inf"))
            return s.max(dim=-1).values.sum(dim=-1)
    run(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sc = run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    del m
    torch.cuda.empty_cache()
    return ms, sc.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="colbertv2.0,answerai-colbert-small")
    ap.add_argument("--n", default="10,30")
    ap.add_argument("--lens", default="128,180")
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precision", default="fp32,fp16")
    ap.add_argument("--no-torch", action="store_true")
    ap.add_argument("--cross-encoder", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    modes = a.precision.split(",")
    if not modes or any(m not in ("fp32", "fp16") for m in modes) or a.reps < 1:
        ap.error("--precision takes fp32, fp16 or both; --reps >= 1")
    from kaito_b200 import _native
    from tests.test_gpu_colbert import SHAPES, _model, _state
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if not gpu:
        raise SystemExit("colbert_bench: no GPU (nvidia-smi reports none); every number here is a GPU measurement")
    ctx = _native.Context(device_id=0)
    rows = []
    for shape in [s for s in a.shapes.split(",") if s]:
        cfg, state, w = _state(*SHAPES[shape], "bench")
        e = _model(ctx, cfg, state, w)
        for n in map(int, a.n.split(",")):
            for plen in map(int, a.lens.split(",")):
                g = np.random.default_rng(n + plen)
                q, keys, p_ids, d_off, keep, poff, pp = inputs(g, a.queries, n, plen)
                args = (q, keys, p_ids, d_off, keep, poff, pp, 10)
                for mode in modes:                                     # warm-up (graphs are captured on the second sight)
                    e.set_precision(mode)
                    e.late_rerank(*args)
                    e.late_rerank(*args)
                t, top = {mode: [] for mode in modes}, {}
                for _ in range(a.reps):
                    for mode in modes:                                 # alternating: both modes see the same minutes of the card
                        e.set_precision(mode)
                        t0 = time.perf_counter()
                        top[mode] = e.late_rerank(*args)               # returns synchronised
                        t[mode].append(time.perf_counter() - t0)
                ms_maxsim = maxsim_profile(e, args, modes)
                row = {"model": shape, "queries": a.queries, "N": n, "passage_tokens": plen, "pairs": int(poff[-1]),
                       "passage_rows": int(d_off[-1]), "query_rows": a.queries * QL}
                for mode in modes:
                    sfx = "" if mode == "fp32" else "_fp16"
                    row[f"krag{sfx}_ms"] = float(np.median(t[mode])) * 1e3
                    row[f"maxsim_kernel{sfx}_ms"] = ms_maxsim[mode]
                if len(modes) == 2:
                    row["top10_overlap"] = float(np.mean([len(set(x.tolist()) & set(y.tolist())) / 10.0
                                                          for x, y in zip(top["fp32"][0], top["fp16"][0])]))
                if not a.no_torch:
                    import torch
                    ref = None
                    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
                        ms, sc = torch_restatement(cfg, state, w, q, keys, p_ids, keep, n, plen, dt)
                        row[f"torch_{name}_ms"] = ms
                        if ref is None:
                            ref = sc
                    # K5's top-10 against torch fp32's (ties by position)
                    want = np.argsort(-ref, axis=1, kind="stable")[:, :10]
                    row["top10_overlap_vs_torch_fp32"] = float(np.mean([len(set(x.tolist()) & set(y.tolist())) / 10.0
                                                                        for x, y in zip(top["fp32"][0], want)]))
                row["gpu"] = gpu
                print(json.dumps(row), flush=True)
                rows.append(row)
        e.destroy()
    if a.cross_encoder:
        p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "rerank_bench.py"), "--models", "L6", "--n", a.n,
                            "--lens", a.lens, "--queries", str(a.queries), "--reps", str(a.reps), "--precision", a.precision,
                            "--no-torch"], capture_output=True, text=True)
        for line in p.stdout.splitlines():
            if line.startswith("{"):
                row = dict(json.loads(line), reference="cross-encoder (scripts/rerank_bench.py)")
                print(json.dumps(row), flush=True)
                rows.append(row)
        if p.returncode:
            sys.stderr.write(p.stderr)
            raise SystemExit(f"rerank_bench.py exited with {p.returncode}")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
