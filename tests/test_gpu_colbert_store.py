"""GPU tests of the ColBERT passage vector store (krag_late_store_*, krag_late_rerank_stored): stored rows against
krag_debug_late_vectors of each passage alone, stored and mixed scores against krag_late_rerank, the shared budget, compaction,
truncation, the refusals, and /retrieve through VectorStore with the store on against the store off.  Every float comparison
is ==: the store must give exactly the per-call path's bits.  Random weights (no checkpoints offline)."""
import json

import numpy as np
import pytest

from tests.test_gpu_colbert import SHAPES, _model, _passage, _query, _state

PRECISIONS = ("fp32", "fp16")


def _emb(ctx, shape, precision, layers=2, seed=0):
    base, dim = SHAPES[shape]
    cfg, st, w = _state(dict(base, num_hidden_layers=layers) if layers else base, dim, "bench", seed)
    return _model(ctx, cfg, st, w, precision)


def _pack(docs):
    off = np.concatenate([[0], np.cumsum([len(d[0]) for d in docs])]).astype(np.int32)
    return np.concatenate([d[0] for d in docs]), off, np.concatenate([d[1] for d in docs])


def _alone_rows(e, doc):
    ids, keep = doc
    return e.debug_late_vectors(ids, np.array([0, len(ids)], np.int32))[keep != 0]


def _append(store, docs):
    return store.append(*_pack(docs))


def _check_rows(e, store, docs, ordinals):
    for o, d in zip(ordinals, docs):
        want = _alone_rows(e, d)
        got = store.debug_vectors(o, len(want))
        assert np.array_equal(got, want), o           # bit for bit (array_equal is ==)


def _queries(g, n):
    qs, qk = zip(*[_query(g, int(g.integers(0, 40))) for _ in range(n)])
    return np.stack(qs), np.asarray(qk, np.int32)


def _rerank_both(e, store, q, qk, docs, cands, stored_of, top_k):
    """krag_late_rerank over every candidate encoded in the call, and krag_late_rerank_stored with the stored ones named by
    ordinal (stored_of[j]: the ordinal of passage j, or -1 when it is not stored) and the others encoded in the call"""
    poff = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.int32)
    pp = np.concatenate([np.asarray(c, np.int32) for c in cands]) if poff[-1] else np.zeros(0, np.int32)
    tok, off, keep = _pack(docs)
    a = e.late_rerank(q, qk, tok, off, keep, poff, pp, top_k)
    call = sorted({int(j) for j in pp if stored_of[j] < 0})
    where = {j: i for i, j in enumerate(call)}
    src = np.array([stored_of[j] if stored_of[j] >= 0 else ~where[int(j)] for j in pp], np.int32)
    if call:
        ctok, coff, ckeep = _pack([docs[j] for j in call])
    else:
        ctok, coff, ckeep = np.zeros(0, np.int32), np.zeros(1, np.int32), np.zeros(0, np.uint8)
    b = e.late_rerank_stored(store, q, qk, ctok, coff, ckeep, poff, src, top_k)
    return a, b


def _same(a, b):
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1], b[1], equal_nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_stored_rows_are_the_kept_rows_of_each_passage_alone(ctx, shape, precision):
    from kaito_b200 import _native
    e = _emb(ctx, shape, precision)
    e.set_store_budget(1 << 30)
    s = _native.LateStore(e)
    g = np.random.default_rng(7)
    lens = [0, 1, 5, 31, 32, 33, 64, 100, 177]                       # 3 tokens ([CLS] [D] [SEP]) up to doc_maxlen 180
    docs = [_passage(g, n) for n in lens]
    one = _passage(g, 50)
    one = (one[0], np.zeros_like(one[1]))
    one[1][17] = 1                                                    # a single kept row
    docs.append(one)
    assert _append(s, docs).all()
    _check_rows(e, s, docs, range(len(docs)))
    n0 = len(docs)
    # appends of different sizes, one of them over 65,536 tokens (two forwards): 1, 7 and 400 passages of 180 tokens
    for k in (1, 7, 400):
        more = [_passage(g, 177) for _ in range(k)]
        assert _append(s, more).all()
        pick = range(k) if k < 400 else (0, 1, 363, 364, 365, 398, 399)  # 364 x 180 tokens fill the first forward
        _check_rows(e, s, [more[i] for i in pick], [n0 + i for i in pick])
        n0 += k
    st = s.stats()
    assert st["ordinals"] == n0 and st["stored"] == n0
    s.destroy(); e.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_full_depth_rows_and_scores(ctx, shape, precision):
    from kaito_b200 import _native
    e = _emb(ctx, shape, precision, layers=None)
    e.set_store_budget(1 << 30)
    s = _native.LateStore(e)
    g = np.random.default_rng(8)
    docs = [_passage(g, int(n)) for n in g.integers(0, 178, 24)]
    assert _append(s, docs).all()
    _check_rows(e, s, docs, range(len(docs)))
    q, qk = _queries(g, 16)
    cands = [list(g.choice(len(docs), 10, replace=False)) for _ in range(16)]
    _same(*_rerank_both(e, s, q, qk, docs, cands, list(range(len(docs))), 10))
    s.destroy(); e.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_stored_scores_equal_per_call_scores(ctx, shape, precision):
    from kaito_b200 import _native
    e = _emb(ctx, shape, precision)
    e.set_store_budget(1 << 30)
    s = _native.LateStore(e)
    g = np.random.default_rng(9)
    docs = [_passage(g, 177) for _ in range(300)]
    docs[5] = docs[4]                                                  # a tie: the same passage under two ordinals
    assert _append(s, docs).all()
    every = list(range(len(docs)))
    # the bench's call: 256 queries x 30 candidates
    q, qk = _queries(g, 256)
    cands = [list(g.choice(300, 30, replace=False)) for _ in range(256)]
    _same(*_rerank_both(e, s, q, qk, docs, cands, every, 30))
    # 300 candidates, a query with none, shared candidates and the tie, top_k 1 / 7 / 300
    q, qk = _queries(g, 5)
    cands = [every, [], [4, 5, 4, 5], [0, 1, 2] * 3, list(g.permutation(300)[:77])]
    for k in (1, 7, 300):
        a, b = _rerank_both(e, s, q, qk, docs, cands, every, k)
        _same(a, b)
    # mixed: every third passage encoded in the call, the others from the store
    mixed = [-1 if j % 3 == 0 else j for j in every]
    q, qk = _queries(g, 64)
    cands = [list(g.choice(300, 30, replace=False)) for _ in range(64)]
    _same(*_rerank_both(e, s, q, qk, docs, cands, mixed, 30))
    s.destroy(); e.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
def test_budget_is_shared_and_exact(ctx, precision):
    from kaito_b200 import _native
    e = _emb(ctx, "answerai-colbert-small", precision)
    g = np.random.default_rng(10)
    docs = []
    for _ in range(40):                                               # 40 passages of exactly 150 kept rows each
        ids, keep = _passage(g, 177)
        keep = np.zeros_like(keep); keep[:150] = 1
        docs.append((ids, keep))
    per = 150 * 96 * 4
    bytes0 = _native.device_bytes()
    e.set_store_budget(25 * per)
    a, b = _native.LateStore(e), _native.LateStore(e)
    assert _append(a, docs[:18]).all()                               # a's first slab takes what the budget allows: 25 passages
    assert a.stats()["device_bytes"] == 25 * per
    assert _native.device_bytes() - bytes0 >= 25 * per
    assert _append(b, docs[:4]).tolist() == [0] * 4                  # the budget is spent: b holds nothing
    assert b.stats() == {"ordinals": 4, "stored": 0, "rows": 0, "device_bytes": 0}
    assert _append(a, docs[18:27]).tolist() == [1] * 7 + [0] * 2    # a's slab fills up to exactly 25 passages
    sa = a.stats()
    assert sa == {"ordinals": 27, "stored": 25, "rows": 25 * 150, "device_bytes": 25 * per}
    q, qk = _queries(g, 12)
    cands = [list(range(i, i + 16)) for i in range(12)]
    stored_of = list(range(25)) + [-1] * 15
    _same(*_rerank_both(e, a, q, qk, docs, [[c + 11 for c in x] for x in cands], stored_of, 10))   # ordinals 11 .. 37
    a.destroy()                                                       # its slab returns to the budget
    assert _append(b, docs[:3]).all()
    assert b.stats()["device_bytes"] == 25 * per
    b.destroy(); e.destroy()


@pytest.mark.gpu
def test_compaction_and_truncation(ctx):
    from kaito_b200 import _native
    e = _emb(ctx, "answerai-colbert-small", "fp32")
    e.set_store_budget(2 << 30)
    s = _native.LateStore(e)
    g = np.random.default_rng(11)
    # over one 256 MB slab: 6,000 passages of 150 to 180 tokens, about 140 kept rows of 384 bytes each
    docs = [_passage(g, int(n)) for n in g.integers(147, 178, 6000)]
    assert _append(s, docs).all()
    st0 = s.stats()
    assert st0["device_bytes"] > 256 << 20
    probe = list(range(0, 6000, 97)) + [5999]
    want = {o: s.debug_vectors(o, int(docs[o][1].sum())) for o in probe}
    # truncate rollback: an append, then back to 6,000 ordinals
    extra = [_passage(g, 177) for _ in range(900)]
    _append(s, extra)
    s.truncate(6000)
    assert s.stats() == st0
    # compact away a random 40 %
    alive = g.random(6000) >= 0.4
    s.compact(alive)
    st1 = s.stats()
    assert st1["ordinals"] == int(alive.sum()) and st1["device_bytes"] < st0["device_bytes"]
    new = np.cumsum(alive) - 1
    for o in probe:
        if alive[o]:
            assert np.array_equal(s.debug_vectors(int(new[o]), int(docs[o][1].sum())), want[o]), o
    live = [d for d, a in zip(docs, alive) if a]
    _check_rows(e, s, [live[i] for i in range(0, len(live), 41)], range(0, len(live), 41))
    assert _append(s, extra[:3]).all()                                 # appends continue after the compacted rows
    _check_rows(e, s, extra[:3], range(len(live), len(live) + 3))
    s.destroy(); e.destroy()


@pytest.mark.gpu
def test_refusals(ctx):
    from kaito_b200 import _native
    e = _emb(ctx, "answerai-colbert-small", "fp32", layers=1)
    with pytest.raises(_native.KragError, match="budget") as ex:
        e.set_store_budget(-1)
    assert ex.value.code == _native.KRAG_E_INVALID
    e.set_store_budget(200 * 96 * 4)                                   # room for one passage
    s = _native.LateStore(e)
    g = np.random.default_rng(12)
    docs = [_passage(g, 150), _passage(g, 150)]
    assert _append(s, docs).tolist() == [1, 0]
    q, qk = _queries(g, 1)
    tok0, off0, keep0 = np.zeros(0, np.int32), np.zeros(1, np.int32), np.zeros(0, np.uint8)
    for src, what in (([1], "does not hold"), ([2], "does not hold"), ([~0], "passage index")):
        with pytest.raises(_native.KragError, match=what) as ex:
            e.late_rerank_stored(s, q, qk, tok0, off0, keep0, np.array([0, 1]), np.array(src), 1)
        assert ex.value.code == _native.KRAG_E_INVALID
    with pytest.raises(_native.KragError, match="destroy its passage vector stores") as ex:
        e.destroy()
    e.set_precision("fp16")
    for call in (lambda: _append(s, docs[:1]),
                 lambda: e.late_rerank_stored(s, q, qk, tok0, off0, keep0, np.array([0, 1]), np.array([0]), 1)):
        with pytest.raises(_native.KragError, match="precision") as ex:
            call()
        assert ex.value.code == _native.KRAG_E_INVALID
    e.set_precision("fp32")
    e.late_rerank_stored(s, q, qk, tok0, off0, keep0, np.array([0, 1]), np.array([0]), 1)    # the valid call
    s.destroy(); e.destroy()
    cfg, st, _ = _state(dict(SHAPES["answerai-colbert-small"][0], num_hidden_layers=1), 96, "bench")
    plain = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                             cfg["vocab_size"], cfg["max_position_embeddings"])
    plain.load_state_dict(st)
    with pytest.raises(_native.KragError, match="late-interaction embedder") as ex:
        _native.LateStore(plain)
    assert ex.value.code == _native.KRAG_E_INVALID
    plain.destroy()


def _colbert_dir(tmp_path):
    from tests import st_snapshot as sts
    vocab = sts.VOCAB + ["[unused0]", "[unused1]"]
    base = dict(SHAPES["answerai-colbert-small"][0], num_hidden_layers=4, vocab_size=len(vocab))
    cfg, st, w = _state(base, 96, "bench", seed=5)
    disk = {"bert." + k: v for k, v in st.items()}
    disk["linear.weight"] = w
    sts.write(tmp_path, {"config.json": dict(sts.BGE_SMALL, **base, architectures=["HF_ColBERT"]),
                         "tokenizer_config.json": {"do_lower_case": True}}, vocab=vocab, state=disk)
    with open(tmp_path / "artifact.metadata", "w") as f:
        json.dump({"query_maxlen": 32, "doc_maxlen": 180, "dim": 96, "mask_punctuation": True, "attend_to_mask_tokens": False,
                   "query_token_id": "[unused0]", "doc_token_id": "[unused1]", "similarity": "cosine"}, f)
    return str(tmp_path), [x for x in sts.VOCAB if not x.startswith("[") and not x.startswith("##")]


@pytest.mark.gpu
def test_service_with_the_store_answers_as_without(ctx, tmp_path, monkeypatch):
    from kaito_b200 import vector_store as vs
    from kaito_b200.embedding import HashingEmbedding
    from kaito_b200.rerank import GpuLateInteractionReranker
    monkeypatch.setattr(vs, "COMPACT_MIN_DEAD_ROWS", 16)
    monkeypatch.setattr(vs, "COMPACT_DEAD_FRACTION", 0.25)
    d, words = _colbert_dir(tmp_path / "model")
    on_rr = GpuLateInteractionReranker.from_pretrained(ctx, d, store_bytes=1 << 30)
    off_rr = GpuLateInteractionReranker.from_pretrained(ctx, d)
    on = vs.VectorStore(HashingEmbedding(384), ctx, reranker=on_rr)
    off = vs.VectorStore(HashingEmbedding(384), ctx, reranker=off_rr)
    g = np.random.default_rng(3)
    docs = [{"text": " ".join(g.choice(words, int(g.integers(5, 90)))), "metadata": {"n": str(i % 3)}} for i in range(240)]
    queries = ["quick brown fox", "gpu token search passage", "the the the", "model index retrieval"]

    def same(step, a="ix_on", b="ix_off"):
        for k in (3, 10):
            x = on.retrieve_batch_bytes(a, queries, max_node_count=k)
            y = off.retrieve_batch_bytes(b, queries, max_node_count=k)
            assert [r[0] for r in x] == [r[0] for r in y], step

    ids = on.index_documents("ix_on", docs); off.index_documents("ix_off", docs)
    st = on.index_map["ix_on"]
    assert st.late_store.stored.all() and len(st.late_store) == len(st.nodes)
    same("index")
    assert not st._pair_cache                                        # every candidate stored: no passage was tokenised or encoded
    bytes_full = st.late_store.stats()["device_bytes"]
    dead = ids[::2]
    on.delete_documents("ix_on", dead); off.delete_documents("ix_off", dead)
    assert st.n_dead == 0 and len(st.late_store) == len(st.nodes)    # compacted
    same("delete + compact")
    upd = [{"doc_id": ids[1], "text": "replaced quick brown fox passage", "metadata": {"n": "9"}}]
    on.update_documents("ix_on", upd); off.update_documents("ix_off", upd)
    same("update")
    on.persist("ix_on", str(tmp_path / "snap_on")); off.persist("ix_off", str(tmp_path / "snap_off"))
    first = ((on, "ix_on"), (off, "ix_off"))
    on = vs.VectorStore(HashingEmbedding(384), ctx, reranker=on_rr)       # fresh stores: `same` now reads these
    off = vs.VectorStore(HashingEmbedding(384), ctx, reranker=off_rr)
    on.load("ix_on2", str(tmp_path / "snap_on")); off.load("ix_off2", str(tmp_path / "snap_off"))
    st2 = on.index_map["ix_on2"]
    assert st2.late_store.stored.all() and len(st2.late_store) == len(st2.nodes)
    same("load", "ix_on2", "ix_off2")
    assert not st2._pair_cache
    assert st2.late_store.stats()["device_bytes"] <= bytes_full
    for store, name in first + ((on, "ix_on2"), (off, "ix_off2")):
        store.delete_index(name)
    on_rr._emb.destroy(); off_rr._emb.destroy()                          # refused if a store were left


@pytest.mark.gpu
def test_compaction_skips_a_small_slab_between_full_ones(ctx):
    """slabs differ in size: one opened when the budget was nearly spent is small.  Its passage is compacted away and the
    next passage, which does not fit that small slab, stays in its own later slab; the emptied small slab is freed"""
    from kaito_b200 import _native
    e = _emb(ctx, "answerai-colbert-small", "fp32")
    g = np.random.default_rng(13)
    row = 96 * 4

    def rows(r):                                                      # a 180-token passage with exactly r kept rows
        ids, keep = _passage(g, 177)
        keep = np.zeros_like(keep); keep[:r] = 1
        return ids, keep
    first = [rows(150) for _ in range(9)]
    small, big, tail = rows(160), rows(175), rows(40)
    e.set_store_budget(10 * 150 * row)                                # slab 0: 10 passages of 150 rows; 9 stored
    s = _native.LateStore(e)
    assert _append(s, first).all()
    e.set_store_budget(10 * 150 * row + 170 * row)                   # slab 1: a leftover of 170 rows, for the 160-row passage
    assert _append(s, [small]).all()
    e.set_store_budget(1 << 30)                                       # slab 2 (256 MB): the 175-row passage, then 40 rows
    assert _append(s, [big, tail]).all()
    before = s.stats()
    assert before["device_bytes"] == 10 * 150 * row + 170 * row + (256 << 20)
    alive = np.ones(12, bool); alive[9] = False                       # drop the small slab's passage
    s.compact(alive)
    after = s.stats()
    assert after == {"ordinals": 11, "stored": 11, "rows": 9 * 150 + 175 + 40, "device_bytes": before["device_bytes"] - 170 * row}
    _check_rows(e, s, first + [big, tail], range(11))
    # appends go on after the last stored passage, in the big slab
    more = [rows(100) for _ in range(3)]
    assert _append(s, more).all()
    _check_rows(e, s, more, range(11, 14))
    assert s.stats()["device_bytes"] == after["device_bytes"]
    # and a compaction that moves passages down across slabs: drop the first 150-row passage, the big one moves into slab 0
    alive = np.ones(14, bool); alive[0] = False
    s.compact(alive)
    live = first[1:] + [big, tail] + more
    _check_rows(e, s, live, range(len(live)))
    assert s.stats()["rows"] == sum(int(d[1].sum()) for d in live)
    # a move that overlaps its own source: a 100-row passage shifts down by the 20 rows of the one dropped before it
    short, long_ = rows(20), rows(100)
    assert _append(s, [short, long_]).all()
    alive = np.ones(len(live) + 2, bool); alive[len(live)] = False
    s.compact(alive)
    live = live + [long_]
    _check_rows(e, s, live, range(len(live)))
    s.destroy(); e.destroy()
