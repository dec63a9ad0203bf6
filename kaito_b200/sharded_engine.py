"""The engine behind the service when the pod has more than one GPU.

The reference runs one process on one device and a RAGEngine pod is exactly one replica
(pkg/ragengine/manifests/manifests.go:81): all GPUs of the box belong to this one service.  `ShardedEngine` is the object
`VectorStore` talks to instead of a single `_native.Context` -- same interface (create_index / load_index; an index with add,
remove, commit, retrieve, search_dense, persist, drop) -- and spreads every index over G ranks, one process per GPU:

  rank 0   the HTTP host (kaito_b200.service): docstore, tokenisation, request coalescing; owns shard 0
  rank r   `python -m kaito_b200.sharded_engine` worker: owns shard r, executes the commands rank 0 broadcasts

Nodes are dealt round-robin: global ordinal o lives on shard o % G at local row o // G (krag_index_set_ordinal_map(base = r,
stride = G)), so ordinals -- and with them every tie-break of the merge and fuse kernels -- are exactly the single-GPU
insertion order, and shards stay balanced under appends and deletes.  BM25 statistics (N, avgdl, df) are all-reduced at
commit.  A coalesced /retrieve batch is ONE broadcast of (query vectors, term ids, k, filter bitmap); every rank runs its
local dense + BM25 candidate kernels, the candidate lists are exchanged over NVLink peer memory (krag_p2p_*) or one NCCL
all-gather, merged and fused on every rank, and rank 0 answers (kaito_b200/sharded.py).

Control messages travel over a gloo group (pickled dicts, a few hundred microseconds per batch); the data path between
GPUs never touches the host.  The stage objects are injected (`stages_factory`) so that the whole protocol runs on CPU
with oracle-backed stand-ins in tests/test_sharded_engine_cpu.py; the product always uses NativeStages.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.distributed as dist

from .sharded import ShardedRetriever


class _Shard:
    def __init__(self, stages, sr, dim):
        self.stages, self.sr, self.dim, self.rows, self.vocab = stages, sr, dim, 0, 0


class ShardedEngine:
    def __init__(self, stages_factory, device: torch.device, data_group=None, ctl_group=None):
        """stages_factory(name, dim, load_path=None) -> stages object of THIS rank (NativeStages in production)"""
        self.factory, self.device = stages_factory, device
        self.data_group, self.ctl = data_group, ctl_group
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.shards: dict[str, _Shard] = {}
        import threading
        self._cmd_mu = threading.Lock()
        # the only CPU-side torch work of these processes is staging a few hundred KB per batch into pinned buffers; spread
        # over an OpenMP team (one thread per core by default) each of those copies waits for threads the HTTP workers and
        # clients keep descheduling -- tens of milliseconds per batch on a loaded box
        torch.set_num_threads(1)

    # ------------------------------------------------------------------ control plane
    def _bcast(self, cmd: dict | None) -> dict:
        box = [cmd]
        dist.broadcast_object_list(box, src=0, group=self.ctl)
        return box[0]

    def _run(self, cmd: dict, ack: bool = True):
        """rank 0: broadcast `cmd`, execute it locally, collect the workers' status"""
        assert self.rank == 0
        with self._cmd_mu:               # one command at a time: the ranks execute the broadcast sequence in lock step
            self._bcast(cmd)
            err, out = None, None
            try:
                out = self._exec(cmd)
            except Exception as e:           # still take part in the status gather, then raise
                err = e
            if ack:
                errs = [None] * self.world
                dist.gather_object(None if err is None else f"rank 0: {err}", errs, dst=0, group=self.ctl)
                bad = [e for e in errs if e]
                if err is not None:
                    raise err
                if bad:
                    raise RuntimeError("; ".join(bad))
            elif err is not None:
                raise err
            return out

    def serve(self):
        """worker loop (ranks > 0)"""
        assert self.rank != 0
        while True:
            cmd = self._bcast(None)
            if cmd["op"] == "shutdown":
                break
            err = None
            try:
                self._exec(cmd)
            except Exception as e:
                err = f"rank {self.rank}: {type(e).__name__}: {e}"
            if cmd.get("ack", True):
                dist.gather_object(err, None, dst=0, group=self.ctl)

    def shutdown(self):
        """rank 0: tell the workers to leave their loops, then tear the process groups down on this side too (the workers'
        destroy_process_group() waits for every rank)"""
        if self.rank == 0 and self.world > 1:
            self._bcast({"op": "shutdown"})
            try:
                dist.destroy_process_group()
            except Exception:
                pass

    # ------------------------------------------------------------------ commands (every rank)
    def _exec(self, cmd: dict):
        op = cmd["op"]
        if op == "create" or op == "load":
            name, dim = cmd["name"], cmd["dim"]
            path = None if op == "create" else os.path.join(cmd["path"], f"shard_{self.rank}_of_{self.world}")
            stages = self.factory(name, dim, path)
            stages.set_ordinal_map(self.rank, self.world)
            sh = _Shard(stages, ShardedRetriever(stages, self.device, stages.dim_padded(), self.data_group), dim)
            sh.rows = stages.n_rows()
            self.shards[name] = sh
            if op == "load" and cmd.get("vocab", 0) > 0:
                sh.vocab = cmd["vocab"]
                sh.sr.commit(sh.vocab, sh.rows, ordinal_base=self.rank)
            return None
        if op == "synth":
            # load-test corpora (scripts/http_load.py): every rank generates its share of a synthetic index on the device
            name, dim, n_total = cmd["name"], cmd["dim"], cmd["n"]
            stages = self.factory(name, dim, None)
            per = n_total // self.world + (1 if self.rank < n_total % self.world else 0)
            stages.index.synth_fill(per, row_base=self.rank * (n_total // self.world + 1), seed=cmd["seed"], vocab=cmd["vocab"])
            stages.set_ordinal_map(self.rank, self.world)
            sh = _Shard(stages, ShardedRetriever(stages, self.device, stages.dim_padded(), self.data_group), dim)
            sh.rows, sh.vocab = per, cmd["vocab"]
            self.shards[name] = sh
            if cmd["vocab"] > 0:
                sh.sr.commit(sh.vocab, sh.rows, ordinal_base=self.rank)
            return None
        if op == "adopt":
            old = self.shards.pop(cmd["to"], None)
            self.shards[cmd["to"]] = self.shards.pop(cmd["name"])
            if old is not None:
                old.stages.drop()
            return None
        if op == "drop":
            sh = self.shards.pop(cmd["name"], None)
            if sh is not None:
                sh.stages.drop()
            return None
        sh = self.shards[cmd["name"]]
        if op == "add":
            ords = cmd["ordinals"]
            mine = np.nonzero(ords % self.world == self.rank)[0]
            if len(mine):
                rows = (ords[mine] // self.world).astype(np.int64)
                if rows[0] != sh.rows or not np.array_equal(rows, np.arange(sh.rows, sh.rows + len(mine))):
                    raise RuntimeError(f"round-robin invariant broken: shard {self.rank} holds {sh.rows} rows, got rows {rows[:3]}..")
                off = cmd["term_offsets"]
                if off is not None:
                    lens = np.diff(off)[mine]
                    noff = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
                    take = np.concatenate([np.arange(off[i], off[i + 1]) for i in mine]) if lens.sum() else np.zeros(0, np.int64)
                    sh.stages.add(ords[mine].astype(np.uint64), cmd["vecs"][mine], noff, cmd["term_ids"][take], cmd["term_tf"][take],
                                  cmd["doc_len"][mine])
                else:
                    sh.stages.add(ords[mine].astype(np.uint64), cmd["vecs"][mine])
                sh.rows += len(mine)
            return None
        if op == "remove":
            ords = cmd["ordinals"]
            mine = ords[ords % self.world == self.rank]
            if len(mine):
                sh.stages.remove(mine.astype(np.uint64))
            return None
        if op == "compact":
            kw = {"window_rows": cmd["window_rows"]} if cmd.get("window_rows") else {}
            reclaimed, sh.rows = sh.sr.compact(sh.vocab, **kw)
            return reclaimed
        if op == "commit":
            sh.vocab = cmd["vocab"]
            sh.sr.commit(sh.vocab, sh.rows, ordinal_base=self.rank)
            return None
        if op == "retrieve":
            return sh.sr.retrieve(cmd["q"], cmd["terms"], cmd["k"], allow_bitmap=cmd["allow"], cand_mult=cmd["cand_mult"],
                                  vector_weight=cmd["vw"], text_weight=cmd["tw"], mode=cmd["mode"])
        if op == "persist":
            p = os.path.join(cmd["path"], f"shard_{self.rank}_of_{self.world}")
            os.makedirs(p, exist_ok=True)
            sh.stages.persist(p)
            return None
        raise ValueError(f"unknown command {op}")

    # ------------------------------------------------------------------ engine interface (rank 0, what VectorStore calls)
    def create_index(self, name: str, dim: int) -> "ShardedIndex":
        self._run({"op": "create", "name": name, "dim": dim})
        return ShardedIndex(self, name, dim)

    def synth_index(self, name: str, dim: int, n: int, vocab: int, seed: int = 20260921) -> "ShardedIndex":
        """load tests: a synthetic corpus of n rows generated on the devices (not on the product path)"""
        self._run({"op": "synth", "name": name, "dim": dim, "n": int(n), "vocab": int(vocab), "seed": int(seed)})
        ix = ShardedIndex(self, name, dim)
        ix.n, ix.vocab = int(n), int(vocab)
        return ix

    def load_index(self, name: str, path: str) -> "ShardedIndex":
        import json
        with open(os.path.join(path, "sharded.json")) as f:
            meta = json.load(f)
        if meta["world"] != self.world:
            raise RuntimeError(f"snapshot was written by {meta['world']} shards, this service runs {self.world}")
        tmp = name + "\x00loading"          # loaded beside a live index of that name, swapped in only on success
        try:
            self._run({"op": "load", "name": tmp, "dim": meta["dim"], "path": path, "vocab": meta["vocab"]})
        except Exception:
            self._run({"op": "drop", "name": tmp})
            raise
        self._run({"op": "adopt", "name": tmp, "to": name})
        ix = ShardedIndex(self, name, meta["dim"])
        ix.n, ix.vocab = meta["n"], meta["vocab"]
        return ix


class ShardedIndex:
    """index handle on rank 0: every call is one broadcast command executed by all ranks"""

    def __init__(self, eng: ShardedEngine, name: str, dim: int):
        self.eng, self.name, self.dim = eng, name, dim
        self.n = 0            # global ordinals handed out so far

    def add(self, node_ids, vecs, term_offsets=None, term_ids=None, term_tf=None, doc_len=None):
        ords = np.asarray(node_ids, np.int64)
        if len(ords) and (ords[0] != self.n or not np.array_equal(ords, np.arange(self.n, self.n + len(ords)))):
            raise ValueError("sharded index: node ids must be the consecutive global ordinals")
        self.eng._run({"op": "add", "name": self.name, "ordinals": ords, "vecs": np.ascontiguousarray(vecs, np.float32).reshape(len(ords), self.dim),
                       "term_offsets": None if term_offsets is None else np.asarray(term_offsets, np.int64),
                       "term_ids": None if term_ids is None else np.asarray(term_ids, np.uint32),
                       "term_tf": None if term_tf is None else np.asarray(term_tf, np.uint16),
                       "doc_len": None if doc_len is None else np.asarray(doc_len, np.uint32)})
        self.n += len(ords)

    def remove(self, node_ids) -> int:
        ords = np.asarray(node_ids, np.int64)
        self.eng._run({"op": "remove", "name": self.name, "ordinals": ords})
        return len(ords)

    # node ids are the global ordinals, so a compaction renumbers them with the ordinals (VectorStore follows)
    compact_renumbers_keys = True

    def compact(self, window_rows: int | None = None) -> int:
        """remove the dead rows of every shard (ShardedRetriever.compact on every rank); the live nodes keep their order and
        get the ordinals 0 .. n_live-1.  Returns the rows reclaimed."""
        reclaimed = int(self.eng._run({"op": "compact", "name": self.name, "window_rows": window_rows}))
        self.n -= reclaimed
        return reclaimed

    def commit(self, vocab: int):
        self.vocab = vocab
        self.eng._run({"op": "commit", "name": self.name, "vocab": int(vocab)})

    def retrieve(self, q, q_terms_list, k: int, cand_mult: float = 3.0, vector_weight: float = 0.7, text_weight: float = 0.3,
                 fusion_mode: int = 0, keyword_allow_bitmap=None):
        if fusion_mode & 0x100:
            raise RuntimeError("filter pushdown is a single-GPU mode; the sharded service applies the reference's keyword-side filter")
        q = np.ascontiguousarray(q, np.float32).reshape(-1, self.dim)
        terms = None if q_terms_list is None else [np.asarray(t, np.uint32) for t in q_terms_list]
        return self.eng._run({"op": "retrieve", "name": self.name, "q": q, "terms": terms, "k": int(k), "cand_mult": float(cand_mult),
                              "vw": float(vector_weight), "tw": float(text_weight), "mode": int(fusion_mode),
                              "allow": None if keyword_allow_bitmap is None else np.asarray(keyword_allow_bitmap, np.uint32), "ack": False},
                             ack=False)

    def search_dense(self, q, k: int):
        out = self.retrieve(q, None, k, cand_mult=1.0)
        dist_, ordn = out["final"].astype(np.float32), out["ordinal"].copy()
        for b in range(len(ordn)):
            c = int(out["count"][b])
            dist_[b, c:] = np.inf; ordn[b, c:] = -1
        return dist_, ordn

    def persist(self, path: str):
        import json
        os.makedirs(path, exist_ok=True)
        self.eng._run({"op": "persist", "name": self.name, "path": path})
        with open(os.path.join(path, "sharded.json"), "w") as f:
            json.dump({"world": self.eng.world, "dim": self.dim, "vocab": int(getattr(self, "vocab", 0)), "n": self.n}, f)

    def drop(self):
        self.eng._run({"op": "drop", "name": self.name})


def native_stages_factory(ctx):
    """production: a krag_index per shard on this rank's GPU"""
    from .sharded import NativeStages

    def make(name, dim, load_path=None):
        ix = ctx.load_index(name, load_path) if load_path else ctx.create_index(name, dim)
        return NativeStages(ctx, ix)
    return make


def init_distributed(rank: int, world: int, local_rank: int, master_port: int, backend: str = "nccl"):
    """one process group for the GPU data path (NCCL) and one for control messages (gloo)"""
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ["MASTER_PORT"] = str(master_port)
    if backend == "nccl":
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local_rank))
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    return dist.new_group(backend="gloo")


def worker_main():
    """`python -m kaito_b200.sharded_engine`: shard worker of the multi-GPU service (ranks 1..G-1), spawned by service.main()"""
    from . import _native
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    ctl = init_distributed(rank, world, local_rank, int(os.environ["MASTER_PORT"]))
    ctx = _native.Context(device_id=local_rank, rank=rank, world_size=world, row_storage=_native.row_storage_from_env())
    eng = ShardedEngine(native_stages_factory(ctx), torch.device("cuda", local_rank), None, ctl)
    try:
        eng.serve()
    finally:
        try:
            for sh in list(eng.shards.values()):
                sh.stages.drop()
            ctx.close()
            dist.destroy_process_group()
        finally:
            os._exit(0)        # never linger behind a half-torn-down NCCL communicator


def spawn_workers(world: int, master_port: int):
    """rank 0 side: start the workers (one per extra GPU) and join the process groups"""
    import subprocess
    procs = []
    for r in range(1, world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(master_port))
        procs.append(subprocess.Popen([sys.executable, "-m", "kaito_b200.sharded_engine"], env=env))
    return procs


if __name__ == "__main__":
    worker_main()
