"""torchrun --nproc-per-node G scripts/sharded_compact_check.py : compaction of the multi-GPU SERVICE on real GPUs.
Rank 0 runs the real VectorStore on a ShardedEngine (NativeStages on every rank, the rows re-dealt over NCCL
all_to_all_single) and the same store on a single-GPU context that compacts with krag_index_compact; with the compaction
threshold lowered, deletes and updates compact both, and /retrieve answers -- ids, order, fp64 scores -- must stay
identical through delete / update / more /index / a second compaction / persist / load."""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, ".")
from kaito_b200 import _native
from kaito_b200 import sharded
from kaito_b200 import sharded_engine as se
from kaito_b200 import vector_store as vs
from kaito_b200.embedding import HashingEmbedding

vs.COMPACT_MIN_DEAD_ROWS = 64
sharded.ShardedRetriever.COMPACT_WINDOW_ROWS = 97        # many windows per compaction, on every rank
rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
ctl = se.init_distributed(rank, world, lr, int(os.environ["MASTER_PORT"]))
ctx = _native.Context(device_id=lr, rank=rank, world_size=world)
eng = se.ShardedEngine(se.native_stages_factory(ctx), torch.device("cuda", lr), None, ctl)
if rank != 0:
    eng.serve()
else:
    g = np.random.default_rng(1)
    words = [f"w{i}" for i in range(400)]
    docs = [{"text": " ".join(g.choice(words, 30)), "metadata": {"area": int(i % 4)}} for i in range(3000)]
    queries = [" ".join(g.choice(words, 4)) for _ in range(64)]
    single_ctx = _native.Context(device_id=lr)
    a, b = vs.VectorStore(HashingEmbedding(96), eng), vs.VectorStore(HashingEmbedding(96), single_ctx)

    def same(name="ix"):
        for k, flt in ((10, None), (5, {"area": 2}), (100, None)):
            ra, rb = a.retrieve_batch(name, queries, k, flt), b.retrieve_batch(name, queries, k, flt)
            for q, x, y in zip(queries, ra, rb):
                assert [(r["doc_id"], r["score"]) for r in x["results"]] == [(r["doc_id"], r["score"]) for r in y["results"]], (q, k, flt)

    def compacted(name="ix"):
        st = a.index_map[name]
        assert st.n_dead == 0 and len(st.nodes) == st.index.n == st.next_key, (st.n_dead, len(st.nodes), st.index.n)
        assert eng.shards[name].rows == -(-len(st.nodes) // world)

    ids = []
    for st in (a, b):
        ids = st.index_documents("ix", docs[:2000]) + st.index_documents("ix", docs[2000:])
    same()
    gone = [ids[i] for i in g.choice(len(ids), 1000, replace=False)]
    for st in (a, b):
        st.delete_documents("ix", gone)
    compacted()
    same()
    left = [i for i in ids if i not in set(gone)]
    upd = [{"doc_id": d, "text": "w1 w2 w3 rewritten " + queries[j % 64], "metadata": {"area": 7}} for j, d in enumerate(left[:50])]
    extra = [{"text": " ".join(g.choice(words, 25)) + f" extra{i}", "metadata": {"area": 1}} for i in range(300)]
    for st in (a, b):
        st.update_documents("ix", upd)
        st.index_documents("ix", extra)
    same()
    for st in (a, b):
        st.delete_documents("ix", left[50:900])
    compacted()
    same()
    with tempfile.TemporaryDirectory() as tmp:
        a.persist("ix", tmp)
        a.load("ix2", tmp)
        assert a.retrieve_batch("ix2", queries, 10) == a.retrieve_batch("ix", queries, 10)
        a.delete_index("ix2")
    print(f"sharded compact check ok: world={world}, {len(a.index_map['ix'].nodes)} live nodes, shard 0 holds "
          f"{eng.shards['ix'].rows} rows", flush=True)
    eng.shutdown()
    single_ctx.close()
for sh in list(eng.shards.values()):
    sh.stages.drop()
ctx.close()
if dist.is_initialized():
    dist.destroy_process_group()
