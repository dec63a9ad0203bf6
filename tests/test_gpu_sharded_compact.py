"""Compaction of the multi-GPU service's round-robin shards on one GPU: G shard indexes in one context, each driven by the
production ShardedRetriever.compact (the krag_redeal_* session: plan, all_to_all_single windows, pack / unpack kernels,
collective commit) with one thread per rank through an in-process stand-in for torch.distributed.

Every case is compared with one index holding every row, given the same removals, then commit + krag_index_compact: bit
for bit, ids, ordinals, fp64 finals, dense and sparse scores, ranks, tie order.  The layout is checked row by row (shard s,
row j holds live row j * G + s; node ids are the new ordinals), the postings against the oracle's build of each shard's
rows under the global statistics, and the results against the oracle pipeline over the live rows renumbered.
KRAG_P2P=0 keeps the query data path on all-gather -> krag_dev_merge."""
import numpy as np
import pytest
import torch

from tests.test_gpu_shards_one_device import (Loopback, OracleRef, assert_same, bitmap, global_stats, run_ranks,
                                              special_queries, sub_csr)

pytestmark = pytest.mark.gpu

KRAG_E_STATE = -6


class LoopbackA2A(Loopback):
    """the loopback plus all_to_all_single: rank r's output is, sender by sender, the sender's input segment for r"""

    @staticmethod
    def all_to_all_single(out, inp, output_split_sizes=None, input_split_sizes=None, group=None):
        sh = group.shared
        sh.slots[group.rank] = (inp, [int(x) for x in input_split_sizes])
        sh.barrier.wait()
        o = 0
        for t in range(sh.world):
            tin, splits = sh.slots[t]
            a, n = sum(splits[:group.rank]), splits[group.rank]
            assert n == int(output_split_sizes[t])
            if n:
                out[o:o + n].copy_(tin[a:a + n])
            o += n
        sh.barrier.wait()


@pytest.fixture
def loopback(monkeypatch):
    from kaito_b200 import sharded
    monkeypatch.setattr(sharded, "dist", LoopbackA2A)
    monkeypatch.setenv("KRAG_P2P", "0")
    return sharded


class RR:
    """G round-robin shards of a corpus (ordinal o -> shard o % G, row o // G; node id = ordinal) with their retrievers"""

    def __init__(self, sharded, ctx, name, x, csr, vocab, G, id_offset=None):
        from kaito_b200.sharded import NativeStages
        self.G, self.vocab, self.n = G, vocab, len(x)
        self.ix, self.sr = [], [None] * G
        for s in range(G):
            r = np.arange(s, len(x), G)
            ix = ctx.create_index(f"{name}_{s}", x.shape[1])
            if len(r):
                ids = r + (id_offset[s] if id_offset else 0)
                ix.add(ids.astype(np.uint64), x[r], *sub_csr(csr, r))
            ix.set_ordinal_map(s, G)
            self.ix.append(ix)
        dpad = self.ix[0].stats().dim_padded

        def mk(rank, group):
            self.sr[rank] = sharded.ShardedRetriever(NativeStages(ctx, self.ix[rank]), torch.device("cuda", 0), dpad, group=group)
        run_ranks(G, mk)

    def each(self, fn, catch=False):
        def body(rank, group):
            self.sr[rank].group = group
            if not catch:
                return fn(rank)
            try:
                return fn(rank)
            except Exception as e:       # every rank's own outcome (the peers still finish the collective protocol)
                return e
        return run_ranks(self.G, body)

    def commit(self):
        return self.each(lambda r: self.sr[r].commit(self.vocab, int(self.ix[r].stats().n_rows), ordinal_base=r))

    def compact(self, window_rows=None, catch=False):
        return self.each(lambda r: self.sr[r].compact(self.vocab, window_rows=window_rows), catch)

    def remove(self, ords):
        ords = np.asarray(ords, np.int64)
        for s, ix in enumerate(self.ix):
            mine = ords[ords % self.G == s]
            if len(mine):
                assert ix.remove(mine.astype(np.uint64)) == len(mine)

    def add(self, x, csr):
        """append rows with the next ordinals, dealt round robin"""
        o = self.n + np.arange(len(x))
        for s, ix in enumerate(self.ix):
            i = np.nonzero(o % self.G == s)[0]
            if len(i):
                ix.add(o[i].astype(np.uint64), x[i], *sub_csr(csr, i))
        self.n += len(x)

    def retrieve(self, q, qs, k, **kw):
        outs = self.each(lambda r: self.sr[r].retrieve(q, qs, k, **kw))
        for o in outs[1:]:
            for name in o:
                assert np.array_equal(o[name], outs[0][name], equal_nan=True), name
        return outs[0]

    def snapshot(self):
        return [(ix.stats().n_rows, ix.stats().n_live, ix.alive_bitmap().copy(), ix.read_rows(0, int(ix.stats().n_rows)))
                for ix in self.ix]

    def drop(self):
        for ix in self.ix:
            ix.drop()


def single_compacted(ctx, name, x, csr, vocab, dead):
    """one index of every row, the same removals, commit, then krag_index_compact"""
    ix = ctx.create_index(name, x.shape[1])
    ix.add(np.arange(len(x), dtype=np.uint64), x, *csr)
    ix.commit(vocab)
    if len(dead):
        ix.remove(np.asarray(dead, np.uint64))
    ix.commit(vocab)
    ix.compact()
    return ix


def check_layout(sh, x, live_ords):
    G = sh.G
    for s, ix in enumerate(sh.ix):
        mine = live_ords[s::G]
        st = ix.stats()
        assert st.n_rows == st.n_live == len(mine), (s, st.n_rows, len(mine))
        if len(mine):
            assert np.array_equal(ix.read_rows(0, len(mine)), x[mine]), s
            ords = s + G * np.arange(len(mine), dtype=np.int64)
            assert np.array_equal(ix.node_ids(ords), ords.astype(np.uint64)), s


def check_postings(o, sh, csr_new, vocab, terms):
    """each shard's postings bitwise against the oracle's build of its rows under the global statistics"""
    n_live = len(csr_new[3])
    df, _, total = global_stats(csr_new, np.ones(n_live, bool), vocab)
    for s, ix in enumerate(sh.ix):
        rows = np.arange(s, n_live, sh.G)
        if not len(rows):
            continue
        st = ix.stats()
        assert (st.n_docs_global, st.total_len_global) == (n_live, total), s
        post = o.bm25_build(*sub_csr(csr_new, rows), vocab, df, n_live, total)
        for t in terms:
            docs, scores, cnt = ix.read_postings(int(t), cap=len(rows) + 1)
            sl = slice(post.off[t], post.off[t + 1])
            assert cnt == post.off[t + 1] - post.off[t], (s, t)
            assert np.array_equal(docs, post.doc[sl]) and np.array_equal(scores.view(np.uint32), post.score[sl].view(np.uint32)), (s, t)


# (K3 kernel, k, fusion mode, allow-bitmap density)
COMBOS = [("warp", 300, 0, None), ("legacy", 10, 1, 0.3), ("legacy", 1, 0, None), ("warp", 10, 1, None)]


def check_retrieve(sh, single, q, qs, n_live, monkeypatch, ref=None, combos=COMBOS):
    for kern, k, mode, dens in combos:
        monkeypatch.setenv("KRAG_BM25_KERNEL", kern)
        bm = bitmap(np.random.default_rng(k + mode).random(n_live) < dens) if dens else None
        got = sh.retrieve(q, qs, k, mode=mode, allow_bitmap=bm)
        assert_same(got, single.retrieve(q, qs, k, fusion_mode=mode, keyword_allow_bitmap=bm), (kern, k, mode, dens))
        if ref is not None:
            ref.check(got, k, 3 * k, 0.7, 0.3, mode, allow=bm, what=(kern, k, mode, dens))


# --------------------------------------------------------------------------------------------------- service shapes
N_SVC, D_SVC, V_SVC, B_SVC = 600_001, 128, 30_000, 64
PATTERNS = ["scattered30", "shard0", "leading", "tail", "none", "all"]


def dead_ordinals(pattern, n, G):
    o = np.arange(n)
    return {"scattered30": np.random.default_rng(81).random(n) < 0.3, "shard0": o % G == 0, "leading": o < n // 4,
            "tail": o >= n - 5000, "none": np.zeros(n, bool), "all": np.ones(n, bool)}[pattern]


@pytest.fixture(scope="module")
def svc(oracle):
    from kaito_b200 import _native
    o = oracle
    x = o.synth_dense(N_SVC, D_SVC, 91)
    csr = o.synth_sparse(N_SVC, V_SVC, 92, mean_len=48.0)
    q = o.synth_queries(x, B_SVC, 93)
    qs = special_queries(csr, V_SVC, o.synth_query_terms(V_SVC, B_SVC, 94, rank_offset=30), np.random.default_rng(95))
    ctx = _native.Context(0)
    state = {"x": x, "csr": csr, "q": q, "qs": qs, "ctx": ctx, "singles": {}, "refs": {}}
    yield state
    for ix in state["singles"].values():
        ix.drop()
    ctx.close()


def _reference(svc, o, key, dead):
    """the compacted single index and the oracle pipeline over the live rows renumbered, per removal set"""
    if key not in svc["singles"]:
        x, csr = svc["x"], svc["csr"]
        live_ords = np.flatnonzero(~dead)
        svc["singles"][key] = single_compacted(svc["ctx"], f"single_{key}", x, csr, V_SVC, np.flatnonzero(dead))
        svc["refs"][key] = OracleRef(o, x[live_ords], sub_csr(csr, live_ords), V_SVC, svc["q"], svc["qs"],
                                     np.ones(len(live_ords), bool), 900) if len(live_ords) else None
    return svc["singles"][key], svc["refs"][key]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("G", [2, 3, 8])
def test_service_shapes(svc, oracle, loopback, monkeypatch, G, pattern):
    from kaito_b200 import _native
    x, csr, q, qs = svc["x"], svc["csr"], svc["q"], svc["qs"]
    dead = dead_ordinals(pattern, N_SVC, G)
    live_ords = np.flatnonzero(~dead)
    n_live = len(live_ords)
    single, ref = _reference(svc, oracle, (pattern, G) if pattern == "shard0" else pattern, dead)
    csr_new = sub_csr(csr, live_ords)
    first = int(np.flatnonzero(dead)[0]) if dead.any() else N_SVC
    moving = n_live - min(first, n_live)
    terms = np.unique(np.concatenate([np.arange(12), np.random.default_rng(G).integers(0, V_SVC, 30), np.concatenate(qs[5:9])]))
    for wr in (None, max(1, moving // 300)):      # the production width, then hundreds of windows
        sh = RR(loopback, svc["ctx"], f"rr{G}_{pattern}", x, csr, V_SVC, G)
        try:
            sh.commit()
            sh.remove(np.flatnonzero(dead))
            sh.commit()
            res = sh.compact(window_rows=wr)
            assert [r[0] for r in res] == [N_SVC - n_live] * G
            assert [r[1] for r in res] == [len(live_ords[s::G]) for s in range(G)]
            assert _native.last_compact()["postings_ms"] == 0.0        # the redeal's report (the rebuild is the commit's)
            check_layout(sh, x, live_ords)
            if wr is None:
                check_postings(oracle, sh, csr_new, V_SVC, terms)
                check_retrieve(sh, single, q, qs, n_live, monkeypatch, ref if n_live else None)
            else:
                check_retrieve(sh, single, q, qs, n_live, monkeypatch, combos=COMBOS[:2])
        finally:
            sh.drop()


def test_grow_remove_and_compact_again(svc, oracle, loopback, monkeypatch):
    """after a compaction: more rows, removals, an incremental commit, a second compaction -- still the single index"""
    from kaito_b200 import _native
    o, G = oracle, 3
    x, csr, q, qs = svc["x"], svc["csr"], svc["q"], svc["qs"]
    rng = np.random.default_rng(101)
    dead = rng.random(N_SVC) < 0.3
    sh = RR(loopback, svc["ctx"], "again", x, csr, V_SVC, G)
    single = single_compacted(svc["ctx"], "again_single", x, csr, V_SVC, np.flatnonzero(dead))
    try:
        sh.commit()
        sh.remove(np.flatnonzero(dead))
        sh.commit()
        sh.compact(window_rows=2000)
        n1 = int((~dead).sum())
        xa = o.synth_dense(40_000, D_SVC, 102)
        ca = o.synth_sparse(40_000, V_SVC, 103, mean_len=48.0)
        sh.n = n1
        sh.add(xa, ca)
        single.add(N_SVC + np.arange(40_000, dtype=np.uint64), xa, *ca)
        n2 = n1 + 40_000
        rm = np.flatnonzero(rng.random(n2) < 0.3)                # new ordinals, old and new rows alike
        sh.remove(rm)
        single.remove(single.node_ids(rm))
        sh.commit()
        assert _native.last_commit()["merged"] == 1
        single.commit(V_SVC)
        check_retrieve(sh, single, q, qs, n2, monkeypatch, combos=COMBOS[:2])
        res = sh.compact(window_rows=977)
        single.compact()
        assert [r[0] for r in res] == [len(rm)] * G
        n3 = n2 - len(rm)
        keep = np.setdiff1d(np.arange(n2), rm)
        x2 = np.concatenate([x[~dead], xa])[keep]
        check_layout(sh, x2, np.arange(n3))
        c2 = sub_csr((np.concatenate([csr[0][:-1], csr[0][-1] + ca[0]]), np.concatenate([csr[1], ca[1]]),
                      np.concatenate([csr[2], ca[2]]), np.concatenate([csr[3], ca[3]])),
                     np.concatenate([np.flatnonzero(~dead), N_SVC + np.arange(40_000)])[keep])
        check_postings(o, sh, c2, V_SVC, np.unique(np.concatenate([np.arange(20), np.concatenate(qs[5:9])])))
        ref = OracleRef(o, x2, c2, V_SVC, q, qs, np.ones(n3, bool), 900)
        check_retrieve(sh, single, q, qs, n3, monkeypatch, ref)
        sh.commit()
        assert _native.last_commit()["merged"] == 1               # a commit after the compaction merges again
    finally:
        sh.drop()
        single.drop()


# ---------------------------------------------------------------------------- the bf16 copy and host-resident rows
@pytest.mark.parametrize("mode", ["bf16_shadow", "host_rows"])
def test_moved_arrays_equal_a_fresh_deal(oracle, loopback, monkeypatch, mode):
    """Xh (bf16 shadow / host rows' device copy), xres and the pinned host rows (through the mapped pointer) move with the
    rows: the compacted shards equal shards freshly built from the live rows in their new order -- rows, device bytes,
    results and the K2 counters that depend on the bf16 rows and xres"""
    from kaito_b200 import _native
    o, G, n, d, vocab = oracle, 2, 800_001, 128, 20_000
    x = o.synth_dense(n, d, 111)
    csr = o.synth_sparse(n, vocab, 112, mean_len=24.0)
    q = o.synth_queries(x, 64, 113)
    qs = o.synth_query_terms(vocab, 64, 114, rank_offset=20)
    kw = {"dense_mode": _native.DENSE_TC_BF16} if mode == "bf16_shadow" else {"row_storage": _native.ROWS_HOST}
    ctx = _native.Context(0, **kw)
    dead = np.random.default_rng(115).random(n) < 0.3
    live_ords = np.flatnonzero(~dead)
    sh = RR(loopback, ctx, "moved", x, csr, vocab, G)
    fresh = RR(loopback, ctx, "fresh", x[live_ords], sub_csr(csr, live_ords), vocab, G)
    try:
        sh.commit()
        sh.remove(np.flatnonzero(dead))
        sh.commit()
        pinned0 = _native.host_pinned_bytes()
        sh.compact(window_rows=3000)
        if mode == "host_rows":
            assert _native.host_pinned_bytes() < pinned0
        fresh.commit()
        check_layout(sh, x, live_ords)
        for a, b in zip(sh.ix, fresh.ix):
            assert a.stats().device_bytes == b.stats().device_bytes
            assert np.array_equal(a.alive_bitmap(), b.alive_bitmap())
        for k in (10, 300):
            c0 = (_native.load().krag_tc_fallback_queries(), _native.host_rows_fetched())
            got = sh.retrieve(q, qs, k)
            c1 = (_native.load().krag_tc_fallback_queries(), _native.host_rows_fetched())
            exp = fresh.retrieve(q, qs, k)
            c2 = (_native.load().krag_tc_fallback_queries(), _native.host_rows_fetched())
            assert_same(got, exp, (mode, k))
            assert (c1[0] - c0[0], c1[1] - c0[1]) == (c2[0] - c1[0], c2[1] - c1[1]), (mode, k)
            if mode == "host_rows":
                assert c1[1] > c0[1]                            # the K2 host path ran: bf16 prune, host rescoring
            else:
                assert _native.last_dense_kernel()[1] == 4        # K2 on the bf16 shadow
    finally:
        sh.drop()
        fresh.drop()
        ctx.close()


# ------------------------------------------------------------------------------------------------------------ refusals
@pytest.fixture
def small(oracle):
    from kaito_b200 import _native
    n, d, vocab = 3001, 64, 500
    x = oracle.synth_dense(n, d, 121)
    csr = oracle.synth_sparse(n, vocab, 122, mean_len=16.0)
    ctx = _native.Context(0)
    yield {"x": x, "csr": csr, "vocab": vocab, "ctx": ctx, "q": oracle.synth_queries(x, 8, 123),
           "qs": oracle.synth_query_terms(vocab, 8, 124, rank_offset=5)}
    ctx.close()


def _same_snapshot(a, b):
    for (n0, l0, al0, x0), (n1, l1, al1, x1) in zip(a, b):
        assert (n0, l0) == (n1, l1) and np.array_equal(al0, al1) and np.array_equal(x0, x1)


@pytest.mark.parametrize("change", ["add", "remove", "node_id"])
def test_refusals_leave_every_shard_unchanged(small, loopback, change):
    from kaito_b200 import _native
    G, x, csr = 3, small["x"], small["csr"]
    n = len(x) - 30
    sh = RR(loopback, small["ctx"], f"ref_{change}", x[:n], sub_csr(csr, np.arange(n)), small["vocab"], G,
            id_offset=[0, 10 ** 6, 0] if change == "node_id" else None)
    try:
        sh.commit()
        rm = np.arange(0, n, 7)
        sh.remove(rm[rm % G != 1] if change == "node_id" else rm)
        sh.commit()
        if change == "add":
            sh.add(x[n:], sub_csr(csr, np.arange(n, len(x))))
        elif change == "remove":
            sh.remove([1, 2, 4])
        before = sh.snapshot()
        errs = sh.compact(window_rows=50, catch=True)
        assert all(isinstance(e, Exception) for e in errs), errs
        assert KRAG_E_STATE in {getattr(e, "code", None) for e in errs}, errs
        assert all(isinstance(e, _native.KragError) or "refused on another rank" in str(e) for e in errs), errs
        _same_snapshot(before, sh.snapshot())          # and no session is left open: every call works again
        if change != "node_id":
            sh.commit()
            res = sh.compact(window_rows=50)
            assert res[0][0] > 0 and all(ix.stats().n_rows == ix.stats().n_live for ix in sh.ix)
    finally:
        sh.drop()


def test_calls_are_refused_while_a_session_is_open(small, loopback):
    from kaito_b200 import _native
    G, x, csr, q, qs = 2, small["x"], small["csr"], small["q"], small["qs"]
    sh = RR(loopback, small["ctx"], "open", x, csr, small["vocab"], G)
    try:
        sh.commit()
        ix = sh.ix[0]
        expect = ix.retrieve(q, qs, 10)
        bms = [i.alive_bitmap() for i in sh.ix]
        words = max(len(b) for b in bms)
        alive_all = np.zeros((G, words), np.uint32)
        for s, b in enumerate(bms):
            alive_all[s, :len(b)] = b
        ix.redeal_begin(alive_all, 100)
        for call in (lambda: ix.retrieve(q, qs, 10), lambda: ix.search_dense(q, 5), lambda: ix.stats(),
                     lambda: ix.add(np.array([10 ** 7], np.uint64), x[:1], *sub_csr(csr, [0])), lambda: ix.remove([0]),
                     lambda: ix.commit(small["vocab"]), lambda: ix.compact(), lambda: ix.redeal_begin(alive_all, 100)):
            with pytest.raises(_native.KragError) as e:
                call()
            assert e.value.code == KRAG_E_STATE
        ix.redeal_abort()
        got = ix.retrieve(q, qs, 10)
        for name in expect:
            assert np.array_equal(got[name], expect[name], equal_nan=True), name
        with pytest.raises(_native.KragError) as e:
            ix.redeal_abort()
        assert e.value.code == KRAG_E_STATE
    finally:
        sh.drop()


# --------------------------------------------------------------------------------------------------------- large shape
def test_large_shape(oracle, loopback, monkeypatch):
    """4M x 768 over G = 4 shards, 30 % removed, against the compacted single index on 256 queries"""
    from kaito_b200 import _native
    monkeypatch.delenv("KRAG_BM25_KERNEL", raising=False)
    o, G, n, d, vocab, chunk = oracle, 4, 4_000_000, 768, 1 << 18, 500_000
    ctx = _native.Context(0)
    single = ctx.create_index("large_single", d)
    single.reserve(n)
    sh = None
    try:
        sh = RR(loopback, ctx, "large", np.zeros((0, d), np.float32), (np.zeros(1, np.int64), np.zeros(0, np.uint32),
                np.zeros(0, np.uint16), np.zeros(0, np.uint32)), vocab, G)
        for ix in sh.ix:
            ix.reserve(n // G + 1)
        qrows = []
        for c in range(0, n, chunk):
            xc = o.synth_dense(chunk, d, 131 + c)
            cc = o.synth_sparse(chunk, vocab, 132 + c, mean_len=24.0)
            single.add(c + np.arange(chunk, dtype=np.uint64), xc, *cc)
            sh.add(xc, cc)
            qrows.append(xc[:32])
        single.commit(vocab)
        sh.commit()
        dead = np.flatnonzero(np.random.default_rng(133).random(n) < 0.3)
        single.remove(dead.astype(np.uint64))
        single.commit(vocab)
        single.compact()
        sh.remove(dead)
        sh.commit()
        res = sh.compact()
        assert [r[0] for r in res] == [len(dead)] * G
        rng = np.random.default_rng(134)
        qx = np.concatenate(qrows)[:128]
        q = np.concatenate([qx + 0.05 * rng.standard_normal(qx.shape).astype(np.float32),
                            rng.standard_normal((128, d)).astype(np.float32)])
        q = np.ascontiguousarray(q / np.linalg.norm(q, axis=1, keepdims=True), np.float32)
        qs = o.synth_query_terms(vocab, 256, 135, rank_offset=50)
        for k in (10, 300):
            assert_same(sh.retrieve(q, qs, k), single.retrieve(q, qs, k), k)
        print(f"\nlarge shape: {_native.device_bytes() / 2**30:.1f} GiB of device memory after the compactions; "
              f"last redeal moved {_native.last_compact()['bytes_moved'] / 2**30:.2f} GiB from one shard")
    finally:
        if sh is not None:
            sh.drop()
        single.drop()
        ctx.close()
