"""Compaction (krag_index_compact) without a GPU: the service's delete / update paths over an oracle engine that compacts,
checked against a store that never does, and a numpy model of the engine's in-place window schedule."""
import json
import os

import numpy as np
import pytest

from kaito_b200 import vector_store as vs
from kaito_b200.embedding import HashingEmbedding
from tests.oracle_engine import OracleEngine, OracleIndex


class CompactingOracleIndex(OracleIndex):
    """OracleIndex plus compact(): dead rows leave, live rows keep their order.  The service compacts right after a commit,
    so re-committing over the live rows reproduces the statistics of that commit."""

    def compact(self):
        n = len(self.ids)
        live = np.array([i not in self.dead for i in range(n)], bool)
        if live.all():
            return 0
        lens = np.diff(self.off)
        keep = np.repeat(live, lens)
        self.x, self.ids, self.dl = self.x[live], self.ids[live], self.dl[live]
        self.tid, self.tf = self.tid[keep], self.tf[keep]
        self.off = np.concatenate([[0], np.cumsum(lens[live])]).astype(np.int64)
        self.dead = set()
        if self.post is not None:
            self.commit(self.vocab)
        return int((~live).sum())


class CompactingOracleEngine(OracleEngine):
    def create_index(self, name, dim):
        return CompactingOracleIndex(self.o, name, dim)

    def load_index(self, name, path):
        ix = super().load_index(name, path)
        ix.__class__ = CompactingOracleIndex
        return ix


WORDS = ("retrieval engine kernel tensor tomato basil vector index search cluster node pod operator memory gpu cache "
         "token query answer model latency batch shard commit delete update snapshot disk text score").split()


def _docs(n, seed):
    rng = np.random.default_rng(seed)
    return [{"text": f"doc {seed}-{i}: " + " ".join(rng.choice(WORDS, size=int(rng.integers(4, 12)))),
             "metadata": {"tag": "a" if i % 3 else "b"}} for i in range(n)]


QUERIES = ["retrieval engine", "tomato basil", "gpu kernel latency", "snapshot disk delete", "vector search index"]


def _answers(store, name="ix"):
    out = []
    for q in QUERIES:
        for flt in (None, {"tag": "b"}):
            r = store.retrieve(name, q, max_node_count=7, metadata_filter=flt)
            out.append([(x["doc_id"], x["text"], x["score"]) for x in r["results"]])
    return out


@pytest.fixture
def low_policy(monkeypatch):
    monkeypatch.setattr(vs, "COMPACT_MIN_DEAD_ROWS", 4)
    monkeypatch.setattr(vs, "COMPACT_DEAD_FRACTION", 0.25)


def _pair(oracle):
    a = vs.VectorStore(HashingEmbedding(64), CompactingOracleEngine(oracle))
    b = vs.VectorStore(HashingEmbedding(64), OracleEngine(oracle))     # no compact(): keeps its tombstones
    return a, b


def test_churn_matches_a_store_that_never_compacts(oracle, low_policy):
    a, b = _pair(oracle)
    docs = _docs(40, 1)
    ids = [s.index_documents("ix", docs) for s in (a, b)][0]
    rng = np.random.default_rng(7)
    for step in range(6):
        gone = [ids[i] for i in rng.choice(len(ids), size=5, replace=False)]
        ids = [i for i in ids if i not in gone]
        assert a.delete_documents("ix", gone) == b.delete_documents("ix", gone)
        upd = [{"doc_id": d, "text": f"updated {step} {d[:8]} " + " ".join(rng.choice(WORDS, size=6)), "metadata": {"tag": "b"}}
               for d in ids[:3]]
        assert a.update_documents("ix", upd) == b.update_documents("ix", upd)
        new = _docs(6, 100 + step)
        ids += [s.index_documents("ix", new) for s in (a, b)][0]
        assert _answers(a) == _answers(b)
        sa = a.index_map["ix"]
        assert [n.ordinal for n in sa.nodes] == list(range(len(sa.nodes)))
        assert len(sa.index.ids) == len(sa.nodes)
        assert [int(k) for k in sa.index.ids] == [n.key for n in sa.nodes]
    sa, sb = a.index_map["ix"], b.index_map["ix"]
    assert len(sa.nodes) == sum(n.alive for n in sb.nodes) + sa.n_dead < len(sb.nodes)


def test_mutations_after_a_compaction_hit_the_right_documents(oracle, low_policy):
    a, b = _pair(oracle)
    docs = _docs(30, 2)
    ids = [s.index_documents("ix", docs) for s in (a, b)][0]
    for s in (a, b):
        s.delete_documents("ix", ids[:12])
    st = a.index_map["ix"]
    assert st.n_dead == 0 and all(n.alive for n in st.nodes) and len(st.nodes) == 18
    assert any(n.key != n.ordinal for n in st.nodes)
    # a delete and an update by doc id after the compaction
    victim, target = ids[20], ids[25]
    upd = [{"doc_id": target, "text": "replacement text about tomato basil soup", "metadata": {}}]
    for s in (a, b):
        s.delete_documents("ix", [victim])
        s.update_documents("ix", upd)
    assert _answers(a) == _answers(b)
    texts = {n.text for n in st.nodes if n.alive}
    assert docs[20]["text"] not in texts and docs[25]["text"] not in texts
    assert "replacement text about tomato basil soup" in texts
    assert [st.nodes[o].text for o in st.ref_docs[target]["nodes"]] == ["replacement text about tomato basil soup"]
    assert [n.text for n in st.nodes if n.ref_doc_id == target and n.alive] == ["replacement text about tomato basil soup"]
    listed = {d["doc_id"] for d in a.list_documents_in_index("ix", limit=100)["documents"]}
    assert victim not in listed and target in listed and not (set(ids[:12]) & listed)


def test_persist_load_after_a_compaction(oracle, low_policy, tmp_path):
    a, b = _pair(oracle)
    docs = _docs(24, 3)
    ids = [s.index_documents("ix", docs) for s in (a, b)][0]
    for s in (a, b):
        s.delete_documents("ix", ids[:10])
    path = str(tmp_path / "snap")
    a.persist("ix", path)
    ds = json.load(open(os.path.join(path, "docstore.json")))
    assert ds["version"] == 1 and len(ds["nodes"]) == 14 and "keys" in ds
    raw = open(os.path.join(path, "docstore.json")).read()
    for d in docs[:10]:
        assert json.dumps(d["text"])[1:-1] not in raw
    c = vs.VectorStore(HashingEmbedding(64), CompactingOracleEngine(oracle))
    c.load("ix", path)
    assert _answers(c) == _answers(b)
    sc = c.index_map["ix"]
    assert [n.key for n in sc.nodes] == ds["keys"] and sc.next_key == max(ds["keys"]) + 1
    for s in (b, c):                       # keys survive the round trip: a delete after the load removes the right rows
        s.delete_documents("ix", [ids[15]])
    assert _answers(c) == _answers(b)


def test_snapshot_without_keys_loads_unchanged(oracle, tmp_path):
    b = vs.VectorStore(HashingEmbedding(64), OracleEngine(oracle))
    ids = b.index_documents("ix", _docs(12, 4))
    b.delete_documents("ix", ids[:3])
    path = str(tmp_path / "old")
    b.persist("ix", path)
    ds = json.load(open(os.path.join(path, "docstore.json")))
    assert "keys" not in ds and len(ds["nodes"]) == 12 and sum(1 for n in ds["nodes"] if not n[4]) == 3
    c = vs.VectorStore(HashingEmbedding(64), OracleEngine(oracle))
    c.load("ix", path)
    sc = c.index_map["ix"]
    assert [n.key for n in sc.nodes] == list(range(12)) and sc.next_key == 12 and sc.n_dead == 3
    assert _answers(c) == _answers(b)
    new = _docs(2, 5)
    for s in (b, c):
        s.index_documents("ix", new)
        s.delete_documents("ix", [ids[5]])
    assert _answers(c) == _answers(b)
    assert [n.key for n in sc.nodes] == list(range(len(sc.nodes)))


def test_default_policy_leaves_small_indexes_alone(oracle):
    a = vs.VectorStore(HashingEmbedding(64), CompactingOracleEngine(oracle))
    ids = a.index_documents("ix", _docs(20, 6))
    a.delete_documents("ix", ids[:15])
    st = a.index_map["ix"]
    assert len(st.nodes) == 20 and st.n_dead == 15


# ---------------------------------------------------------------- numpy model of compact.cu's window schedule
STAGE_BYTES = 32 << 20      # COMPACT_STAGE_BYTES
TERM_BYTES = 6              # COMPACT_TERM_BYTES


def _first_moving(src):
    moved = np.flatnonzero(src != np.arange(len(src)))
    return int(moved[0]) if moved.size else len(src)


def _row_windows(src, W):
    """compact_rows: windows of W destination rows from the first dead row; direct iff the window ends at or below its
    first source row"""
    for d0 in range(_first_moving(src), len(src), W):
        d1 = min(len(src), d0 + W)
        yield d0, d1, d1 <= src[d0]


def _term_windows(src, to, tn, cap):
    """compact_terms: the longest run of destination rows whose entries fit the staging buffer (at least one row)"""
    d0, n = _first_moving(src), len(src)
    while d0 < n:
        d1 = int(np.searchsorted(tn, tn[d0] + cap, side="right")) - 1
        d1 = min(n, max(d1, d0 + 1))
        yield d0, d1, tn[d1] <= to[src[d0]]
        d0 = d1


def _simulate(n_units, moves):
    """moves: per window (reads, writes, direct), unit indices in the destination order.  Checks that every unit read still
    holds its original content and that a direct window reads nothing it writes; returns the final memory."""
    mem = np.arange(n_units)
    for reads, writes, direct in moves:
        assert np.array_equal(mem[reads], reads), "a source unit was overwritten before it was read"
        if direct and reads.size:
            assert writes.max() < reads.min(), "a direct window writes over its own sources"
        mem[writes] = mem[reads]
    return mem


def _patterns(n, W):
    rng = np.random.default_rng(11)
    every_other = np.arange(n) % 2 == 0
    runs = np.ones(n, bool)
    for a in (30, W - 3, 2 * W - 40, 3 * W + 31):
        runs[a:a + 45] = False
    last = np.ones(n, bool)
    last[-37:] = False
    row0 = np.ones(n, bool)
    row0[0] = False
    return {"none": np.ones(n, bool), "all": np.zeros(n, bool), "row0": row0, "last": last, "every_other": every_other,
            "runs": runs, "random30": rng.random(n) >= 0.3, "contiguous50": np.arange(n) >= n // 2}


@pytest.mark.parametrize("row_bytes", [4, 2 * 768, 4 * 768])
def test_row_window_schedule_reads_before_it_writes(row_bytes):
    W = STAGE_BYTES // row_bytes
    scale = max(1, W // 64)                 # simulate W/scale-row windows over 5 windows' worth of rows
    W //= scale
    n = 5 * W + 17
    for name, alive in _patterns(n, W).items():
        src = np.flatnonzero(alive)
        moves = [(src[d0:d1], np.arange(d0, d1), direct) for d0, d1, direct in _row_windows(src, W)]
        mem = _simulate(n, moves)
        assert np.array_equal(mem[:len(src)], src), name
        if name == "row0":
            assert moves and not any(d for _, _, d in moves)      # every row shifts by one: all staged
        if name == "none":
            assert moves == []


def test_term_window_schedule_reads_before_it_writes():
    rng = np.random.default_rng(5)
    n = 900
    lens = rng.integers(0, 9, size=n)
    lens[123] = 300                           # one list longer than the staging buffer below
    to = np.concatenate([[0], np.cumsum(lens)])
    cap = 200
    for name, alive in _patterns(n, 64).items():
        src = np.flatnonzero(alive)
        tn = np.concatenate([[0], np.cumsum(lens[src])])
        cap_w = max(cap, int(np.diff(tn).max(initial=0)))
        moves = []
        for d0, d1, direct in _term_windows(src, to, tn, cap_w):
            reads = np.concatenate([np.arange(to[s], to[s + 1]) for s in src[d0:d1]])
            writes = np.arange(tn[d0], tn[d1])
            assert writes.size == reads.size and writes.size <= cap_w
            moves.append((reads, writes, direct))
        mem = _simulate(int(to[-1]), moves)
        expect = np.concatenate([np.arange(to[s], to[s + 1]) for s in src]) if src.size else np.zeros(0, int)
        assert np.array_equal(mem[:tn[-1]], expect), name
