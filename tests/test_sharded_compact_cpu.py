"""Compaction of the multi-GPU service's round-robin shards (ShardedRetriever.compact, the redeal protocol of
kaito_rag.h krag_redeal_begin) without a GPU: the protocol over gloo with 2 and 3 processes and a numpy stage double that
packs and unpacks rows with the same plan tables, driven through VectorStore on ShardedEngine and compared with the
single-process store that compacts; and a numpy check of the window schedule's in-place invariant."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.oracle_engine import OracleShardStages


# ------------------------------------------------------------------------------------------------ the plan, in numpy
def _ceil_rows(R, s, G):
    """rows j of shard s with j * G + s < R"""
    return (R - s + G - 1) // G if R > s else 0


def redeal_plan(alive_all, s, window_rows, lens):
    """What krag_redeal_begin computes for shard s from the gathered bitmaps [G, words]: new ordinals, windows, the send
    order (grouped by window and destination, ascending rank) and the [n_windows, G] tables.  lens: term-list lengths of
    shard s's rows."""
    G = alive_all.shape[0]
    bits = np.unpackbits(np.ascontiguousarray(alive_all, np.uint32).view(np.uint8), bitorder="little").reshape(G, -1).astype(bool)
    live = bits.T.reshape(-1)                          # by ordinal m * G + t
    rank = np.cumsum(live) - 1                         # live ordinals below
    n_live = int(live.sum())
    dead = np.flatnonzero(~live)
    first = min(int(dead[0]) if dead.size else live.size, n_live)
    W = -(-(n_live - first) // window_rows) if n_live > first else 0
    mine = np.flatnonzero(bits[s])
    r = rank[mine * G + s]
    moving, rm = mine[r >= first], r[r >= first]
    key = ((rm - first) // window_rows) * G + rm % G
    order = np.lexsort((rm, key))
    o_all = np.flatnonzero(live)
    ro = rank[o_all]
    sel = (ro >= first) & (ro % G == s)
    lens = np.asarray(lens, np.int64)
    return {
        "G": G, "s": s, "n_live": n_live, "first": first, "n_windows": W, "n_new": _ceil_rows(n_live, s, G),
        "j_first": _ceil_rows(first, s, G), "send": moving[order], "key": key[order], "dst": rm[order] // G,
        "send_rows": np.bincount(key, minlength=W * G).reshape(W, G).astype(np.int64),
        "send_ents": np.bincount(key, weights=lens[moving], minlength=W * G).reshape(W, G).astype(np.int64),
        "recv_rows": np.bincount(((ro[sel] - first) // window_rows) * G + o_all[sel] % G, minlength=W * G).reshape(W, G).astype(np.int64),
    }


def _bitmap(live):
    live = np.asarray(live, bool)
    return np.packbits(np.concatenate([live, np.zeros((-len(live)) % 32, bool)]), bitorder="little").view(np.uint32).copy()


ENT = np.dtype([("tid", "<u4"), ("tf", "<u4")])


class RedealOracleStages(OracleShardStages):
    """OracleShardStages plus the redeal steps: pack and unpack in numpy, with the plan tables of redeal_plan"""

    def _row_dtype(self):
        return np.dtype([("dst", "<i8"), ("len", "<i8"), ("dl", "<u4"), ("pad", "<u4"), ("x", "<f4", (self.dim,))])

    def alive_bitmap(self):
        ix = self.ix
        return _bitmap([i not in ix.dead for i in range(len(ix.ids))])

    def redeal_begin(self, alive_all, window_rows):
        p = self._plan = redeal_plan(alive_all, self.base, window_rows, np.diff(self.ix.off))
        assert p["G"] == self.stride
        self._new = {}
        return p["n_windows"], p["n_live"], self._row_dtype().itemsize, p["send_rows"], p["send_ents"], p["recv_rows"]

    def redeal_prepare(self, recv_entries):
        self._plan["recv_ents"] = np.asarray(recv_entries, np.int64)

    def redeal_pack(self, k, rows, entries):
        p, ix, G = self._plan, self.ix, self.stride
        idx = np.flatnonzero(p["key"] // G == k)
        src = p["send"][idx]
        R = np.zeros(len(idx), self._row_dtype())
        R["dst"], R["len"], R["dl"], R["x"] = p["dst"][idx], ix.off[src + 1] - ix.off[src], ix.dl[src], ix.x[src]
        take = np.concatenate([np.arange(ix.off[r], ix.off[r + 1]) for r in src]) if len(src) else np.zeros(0, np.int64)
        E = np.zeros(len(take), ENT)
        E["tid"], E["tf"] = ix.tid[take], ix.tf[take]
        rows[:R.nbytes].copy_(torch.from_numpy(np.frombuffer(R.tobytes(), np.uint8).copy()))
        entries[:E.nbytes].copy_(torch.from_numpy(np.frombuffer(E.tobytes(), np.uint8).copy()))

    def redeal_unpack(self, k, rows, entries):
        p, dt = self._plan, self._row_dtype()
        n, ne = int(p["recv_rows"][k].sum()), int(p["recv_ents"][k].sum())
        R = np.frombuffer(rows[:n * dt.itemsize].numpy().tobytes(), dt)
        E = np.frombuffer(entries[:ne * ENT.itemsize].numpy().tobytes(), ENT)
        pos = 0                                  # rows and entries both come grouped by sender, in ascending rank
        for r in R:
            ln = int(r["len"])
            assert int(r["dst"]) not in self._new
            self._new[int(r["dst"])] = (r["x"].copy(), int(r["dl"]), E["tid"][pos:pos + ln].copy(), E["tf"][pos:pos + ln].astype(np.uint16))
            pos += ln
        assert pos == ne

    def redeal_finish(self):
        p, ix, G, s = self._plan, self.ix, self.stride, self.base
        jf, n = p["j_first"], p["n_new"]
        assert sorted(self._new) == list(range(jf, n))
        x, dl, tid, tf, off = list(ix.x[:jf]), list(ix.dl[:jf]), [ix.tid[:ix.off[jf]]], [ix.tf[:ix.off[jf]]], list(ix.off[:jf + 1])
        for j in range(jf, n):
            xv, d, t, f = self._new[j]
            x.append(xv); dl.append(d); tid.append(t); tf.append(f); off.append(off[-1] + len(t))
        ix.x = np.asarray(x, np.float32).reshape(n, self.dim)
        ix.dl, ix.off = np.asarray(dl, np.uint32), np.asarray(off, np.int64)
        ix.tid, ix.tf = np.concatenate(tid).astype(np.uint32), np.concatenate(tf).astype(np.uint16)
        ix.ids = (s + np.arange(n, dtype=np.int64) * G).astype(np.uint64)
        ix.dead, ix.post = set(), None
        self._plan = self._new = None
        return n

    def redeal_abort(self):
        self._plan = self._new = None


# ----------------------------------------------------------------------------------------- the service over gloo
WORDS = ("retrieval engine kernel tensor tomato basil vector index search cluster node pod operator memory gpu cache "
         "token query answer model latency batch shard commit delete update snapshot disk text score").split()
QUERIES = ["retrieval engine", "tomato basil", "gpu kernel latency", "snapshot disk delete", "vector search index", "zebra"]


def _docs(n, seed):
    rng = np.random.default_rng(seed)
    return [{"text": f"doc {seed}-{i}: " + " ".join(rng.choice(WORDS, size=int(rng.integers(4, 12)))),
             "metadata": {"tag": "a" if i % 3 else "b"}} for i in range(n)]


def _run(rank, world, port, tmp, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    eng = None
    try:
        from oracle import oracle as o
        from kaito_b200 import sharded
        from kaito_b200 import vector_store as vs
        from kaito_b200.embedding import HashingEmbedding
        from kaito_b200.sharded_engine import ShardedEngine, init_distributed
        from tests.oracle_engine import OracleEngine
        from tests.test_compact_cpu import CompactingOracleEngine
        sharded.ShardedRetriever.COMPACT_WINDOW_ROWS = 5          # many windows on every compaction
        vs.COMPACT_MIN_DEAD_ROWS = 4

        def load(name, dim, path):
            st = RedealOracleStages(o, name, dim)
            st.ix = OracleEngine(o).load_index(name, path)
            st.ix.post = None
            return st
        ctl = init_distributed(rank, world, rank, port, backend="gloo")
        eng = ShardedEngine(lambda name, dim, path=None: RedealOracleStages(o, name, dim) if path is None else load(name, dim, path),
                            torch.device("cpu"), None, ctl)
        if rank != 0:
            eng.serve()
            ret[rank] = "ok"
            return
        a, b = vs.VectorStore(HashingEmbedding(48), eng), vs.VectorStore(HashingEmbedding(48), CompactingOracleEngine(o))

        def same(name="ix"):
            for q in QUERIES:
                for kw in ({"max_node_count": 7}, {"max_node_count": 12, "metadata_filter": {"tag": "b"}}):
                    ra, rb = a.retrieve(name, q, **kw), b.retrieve(name, q, **kw)
                    assert [(r["doc_id"], r["text"], r["score"]) for r in ra["results"]] == \
                           [(r["doc_id"], r["text"], r["score"]) for r in rb["results"]], (q, kw)
            assert [n.node_id for n, _ in a.dense_candidates(name, QUERIES[2], 20)] == \
                   [n.node_id for n, _ in b.dense_candidates(name, QUERIES[2], 20)]

        def compacted(name="ix"):
            st = a.index_map[name]
            assert st.n_dead == 0 and len(st.nodes) == st.index.n == st.next_key
            assert [n.ordinal for n in st.nodes] == [n.key for n in st.nodes] == list(range(len(st.nodes)))
            assert eng.shards[name].rows == -(-len(st.nodes) // world)        # shard 0's rows: the fresh deal of the live nodes

        ids = []
        for s in (a, b):
            ids = s.index_documents("ix", _docs(40, 1)) + s.index_documents("ix", _docs(25, 2))
        same()
        rng = np.random.default_rng(3)
        gone = [ids[i] for i in rng.choice(len(ids), 20, replace=False)]
        for s in (a, b):
            s.delete_documents("ix", gone)
        compacted()
        same()
        left = [i for i in ids if i not in gone]
        upd = [{"doc_id": d, "text": "rewritten about tomato basil and gpu latency " + d[:6], "metadata": {"tag": "b"}} for d in left[:4]]
        for s in (a, b):
            assert s.update_documents("ix", upd)["updated_documents"]
            s.index_documents("ix", _docs(9, 4))
        same()
        for s in (a, b):                            # the first nodes: every row moves, and a second compaction
            s.delete_documents("ix", left[4:20])
        compacted()
        same()
        for s in (a, b):
            s.delete_documents("ix", [left[25]])      # a delete after the compaction removes exactly its rows
            s.index_documents("ix", _docs(3, 5))
        same()
        a.persist("ix", os.path.join(tmp, "snap"))
        a.load("ix2", os.path.join(tmp, "snap"))
        b.persist("ix", os.path.join(tmp, "snap_b"))
        b.load("ix2", os.path.join(tmp, "snap_b"))
        same("ix2")
        for s in (a, b):
            s.delete_documents("ix2", left[26:40])
        compacted("ix2")
        same("ix2")
        eng.shutdown()
        ret[rank] = "ok"
    except Exception:
        import traceback
        ret[rank] = traceback.format_exc()
        try:
            if rank == 0 and eng is not None:
                eng.shutdown()
        except Exception:
            pass
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_compaction_equals_single_process(world, tmp_path):
    from oracle import oracle as o
    o.build()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_run, args=(world, _free_port(), str(tmp_path), ret), nprocs=world, join=True)
    for r in range(world):
        assert ret.get(r) == "ok", ret.get(r)


# ------------------------------------------------------------------------------------ the window schedule, in numpy
def _patterns(n, G, rng):
    o = np.arange(n)
    return {"random30": rng.random(n) >= 0.3, "shard0": o % G != 0, "leading": o >= n // 3, "tail": o < n - 37,
            "none": np.ones(n, bool), "all": np.zeros(n, bool), "sparse": rng.random(n) < 0.05, "first": o != 0}


@pytest.mark.parametrize("G", [2, 3, 8])
def test_window_schedule_reads_every_row_before_it_is_overwritten(G):
    """every shard packs window k (reads) before any shard unpacks it (writes), windows ascending, in place: no row is read
    after it was overwritten, and the result is the fresh deal of the live rows"""
    rng = np.random.default_rng(G)
    for n in (1, 7, 300, 1001):
        for name, live in _patterns(n, G, rng).items():
            rows = [np.arange(s, n, G) for s in range(G)]                    # old ordinals of each shard's rows
            alive = [live[r] for r in rows]
            words = max(1, max((len(r) + 31) // 32 for r in rows))
            alive_all = np.zeros((G, words), np.uint32)
            for s in range(G):
                bm = _bitmap(alive[s])
                alive_all[s, :len(bm)] = bm
            for wr in (1, 3, 64):
                plans = [redeal_plan(alive_all, s, wr, np.ones(len(rows[s]), np.int64)) for s in range(G)]
                mem = [r.copy() for r in rows]                               # what each row slot holds (an old ordinal)
                W = plans[0]["n_windows"]
                for k in range(W):
                    sent = {}
                    for s, p in enumerate(plans):
                        idx = np.flatnonzero(p["key"] // G == k)
                        assert np.array_equal(mem[s][p["send"][idx]], rows[s][p["send"][idx]]), (name, n, wr, k, s)
                        for d in range(G):
                            seg = idx[p["key"][idx] % G == d]
                            sent[(s, d)] = list(zip(p["dst"][seg], rows[s][p["send"][seg]]))
                            assert len(seg) == p["send_rows"][k, d] == plans[d]["recv_rows"][k, s]
                    for d in range(G):
                        for s in range(G):
                            for j, o_old in sent[(s, d)]:
                                mem[d][j] = o_old
                live_ords = np.flatnonzero(live)
                for s, p in enumerate(plans):
                    assert p["n_new"] == len(range(s, len(live_ords), G)), (name, n, wr)
                    assert np.array_equal(mem[s][:p["n_new"]], live_ords[s::G]), (name, n, wr, s)
