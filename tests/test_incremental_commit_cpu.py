"""The incremental commit's merge rule, restated in numpy and checked against a sort-based rebuild over random histories of
adds, removes, commits and compactions (no GPU needed).

Rule: a term's new list is its base list without the rows that are dead now, in base order, followed by the live rows added
since the base, ascending; df = survivors + delta.  A compaction renumbers the survivors to their ranks among the live rows
and keeps the rows below the old base boundary as the new base."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def full_build(term_lists, alive, vocab):
    """postings by a stable sort of (term, row) over the live rows: off [vocab + 1], doc [nnz]"""
    rows = [r for r in range(len(term_lists)) if alive[r]]
    t = np.concatenate([term_lists[r] for r in rows] + [np.zeros(0, np.int64)]).astype(np.int64)
    d = np.concatenate([np.full(len(term_lists[r]), r) for r in rows] + [np.zeros(0, np.int64)]).astype(np.int64)
    order = np.lexsort((d, t))
    off = np.concatenate([[0], np.cumsum(np.bincount(t, minlength=vocab))])
    return off, d[order]


def merge(base_off, base_doc, base_rows, term_lists, alive, vocab):
    """survivor counts per term from fixed blocks of base postings, their scan, then survivors followed by the delta"""
    nb = len(base_doc)
    term_of = np.searchsorted(base_off, np.arange(nb), side="right") - 1          # largest t with off[t] <= p
    ok = alive[base_doc] if nb else np.zeros(0, bool)
    block = 2048
    block_cnt = np.array([ok[i:i + block].sum() for i in range(0, nb, block)], np.int64)
    block_off = np.concatenate([[0], np.cumsum(block_cnt)])[:-1]
    surv = np.bincount(term_of[ok], minlength=vocab)[:vocab]
    before = np.concatenate([[0], np.cumsum(surv)])
    # delta: live rows >= base_rows, sorted by (term, row)
    new_rows = [r for r in range(base_rows, len(term_lists)) if alive[r]]
    dt = np.concatenate([term_lists[r] for r in new_rows] + [np.zeros(0, np.int64)]).astype(np.int64)
    dd = np.concatenate([np.full(len(term_lists[r]), r) for r in new_rows] + [np.zeros(0, np.int64)]).astype(np.int64)
    order = np.lexsort((dd, dt))
    dt, dd = dt[order], dd[order]
    delta = np.bincount(dt, minlength=vocab)
    delta_off = np.concatenate([[0], np.cumsum(delta)])
    df = surv + delta
    off = np.concatenate([[0], np.cumsum(df)])
    doc = np.full(off[-1], -1, np.int64)
    for p in range(nb):                                                           # survivor k of t -> off[t] + k
        if ok[p]:
            s = block_off[p // block] + ok[(p // block) * block:p].sum()
            t = term_of[p]
            doc[off[t] + (s - before[t])] = base_doc[p]
    for q in range(len(dt)):                                                      # then the delta
        t = dt[q]
        doc[off[t] + surv[t] + (q - delta_off[t])] = dd[q]
    assert (doc >= 0).all()
    return off, doc, df


def compact(base_off, base_doc, base_rows, term_lists, alive):
    """live rows move down to their ranks; the base keeps its survivors renumbered"""
    rank = np.cumsum(alive) - 1
    ok = alive[base_doc] if len(base_doc) else np.zeros(0, bool)
    term_of = np.searchsorted(base_off, np.arange(len(base_doc)), side="right") - 1
    surv = np.bincount(term_of[ok], minlength=len(base_off) - 1)
    off = np.concatenate([[0], np.cumsum(surv)])
    doc = rank[base_doc[ok]]
    new_lists = [term_lists[r] for r in range(len(term_lists)) if alive[r]]
    new_base_rows = int(alive[:base_rows].sum())
    return off, doc, new_base_rows, new_lists, np.ones(len(new_lists), bool)


def test_merge_rule_matches_sort_rebuild_over_random_histories():
    rng = np.random.default_rng(0)
    for trial in range(40):
        vocab = int(rng.integers(3, 60))
        lists, alive = [], np.zeros(0, bool)
        base = None          # (off, doc, base_rows)
        for step in range(int(rng.integers(3, 12))):
            op = rng.choice(["add", "remove", "commit", "compact"], p=[0.4, 0.25, 0.25, 0.1])
            if op == "add":
                for _ in range(int(rng.integers(1, 300))):
                    k = int(rng.integers(0, min(vocab, 8)))
                    lists.append(np.unique(rng.integers(0, vocab, k)))
                alive = np.concatenate([alive, np.ones(len(lists) - len(alive), bool)])
            elif op == "remove" and len(lists):
                alive[rng.random(len(lists)) < rng.random() * 0.5] = False
            elif op == "compact" and len(lists):
                if base is not None:
                    o, d, br, lists, alive = compact(base[0], base[1], base[2], lists, alive)
                    base = (o, d, br)
                else:
                    lists = [lists[r] for r in range(len(lists)) if alive[r]]
                    alive = np.ones(len(lists), bool)
            elif op == "commit":
                ref_off, ref_doc = full_build(lists, alive, vocab)
                if base is None:
                    base = (ref_off, ref_doc, len(lists))
                    continue
                off, doc, df = merge(base[0], base[1], base[2], lists, alive, vocab)
                assert np.array_equal(off, ref_off) and np.array_equal(doc, ref_doc), (trial, step)
                assert np.array_equal(df, np.diff(ref_off))
                base = (off, doc, len(lists))


def test_block_straddles_terms_and_long_terms():
    """one term over many blocks, and blocks over many terms, with removals inside"""
    rng = np.random.default_rng(1)
    lists = [np.array([0] + ([int(rng.integers(1, 40))] if r % 3 else []), np.int64) for r in range(9000)]
    alive = np.ones(9000, bool)
    off, doc = full_build(lists, alive, 40)
    alive[rng.random(9000) < 0.2] = False
    lists += [np.array([0, 5]), np.array([], np.int64), np.array([39])]
    alive = np.concatenate([alive, [True, True, False]])
    m_off, m_doc, _ = merge(off, doc, 9000, lists, alive, 41)
    r_off, r_doc = full_build(lists, alive, 41)
    assert np.array_equal(m_off, r_off) and np.array_equal(m_doc, r_doc)


def test_last_commit_is_declared_and_bound():
    from kaito_b200 import _native
    assert "krag_last_commit" in _native.SYMBOLS
    assert "krag_last_commit(" in open(os.path.join(ROOT, "include", "kaito_rag.h")).read()
    L = _native.load()
    assert getattr(L, "krag_last_commit") is not None
