"""Concurrent searches on one index against serial results, and the ordering the device stage API promises
(include/kaito_rag.h): work a stage call leaves queued on the caller's stream is finished before its search slot serves
another call and before the index is mutated.

The kernels are deterministic, so concurrency may not change a single bit: every comparison is on the bytes of ids and
scores.  Threads run a fixed number of rounds; the only waiting on the GPU is a bounded torch.cuda._sleep that holds a
stream while the host goes on."""
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N, D, VOCAB, K = 300_000, 128, 5000, 10
SLEEP_CYCLES = 200_000_000          # about 100 ms at H100 clocks (an estimate, not a measurement)


def same(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes() for x, y in zip(a, b))


def run_threads(n, fn):
    """fn(i) on n threads started together; the first exception is raised after every thread has ended"""
    errs, go = [], threading.Barrier(n, timeout=600)

    def body(i):
        try:
            go.wait()
            fn(i)
        except BaseException as e:        # noqa: BLE001 -- re-raised below
            errs.append(e)

    ts = [threading.Thread(target=body, args=(i,)) for i in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errs:
        raise errs[0]


def _retrieve(ix, *a, **kw):
    out = ix.retrieve(*a, **kw)
    return tuple(out[key] for key in ("final", "dense", "sparse", "rank", "ordinal", "count"))


class Corpus:
    """the seeded hybrid corpus, its tombstones and queries, and the oracle over its live rows"""

    def __init__(self, o, n=N, d=D, vocab=VOCAB, seed=41):
        self.n, self.d, self.vocab = n, d, vocab
        self.x = o.synth_dense(n, d, seed)
        self.csr = o.synth_sparse(n, vocab, seed + 1)
        self.dead = np.arange(5, n, 29, dtype=np.int64)            # ~3.4 %: alive_ptr is non-null in every kernel
        self.q = o.synth_queries(self.x, 256, seed + 2)
        self.qs = o.synth_query_terms(vocab, 256, seed + 3, rank_offset=30)
        rng = np.random.default_rng(seed + 4)
        self.allow = np.packbits(rng.random(((n + 31) // 32) * 32) < 0.3, bitorder="little").view(np.uint32)
        self.alive = o.alive_bitmap(n, self.dead)

    def build(self, ctx, name):
        ix = ctx.create_index(name, self.d)
        ix.add(np.arange(self.n, dtype=np.uint64), self.x, *self.csr)
        ix.remove(self.dead.astype(np.uint64))
        ix.commit(self.vocab)
        return ix

    def live_postings(self, o):
        off, ids, tf, dl = self.csr
        live = np.ones(self.n, bool)
        live[self.dead] = False
        keep = np.repeat(live, np.diff(off))
        off2 = np.concatenate([[0], np.cumsum(np.where(live, np.diff(off), 0))]).astype(np.int64)
        df = np.bincount(ids[keep], minlength=self.vocab).astype(np.uint32)
        return o.bm25_build(off2, ids[keep], tf[keep], dl, self.vocab, df, int(live.sum()), int(dl[live].astype(np.int64).sum()))


def call_mix(c):
    """name -> call on an index: every synchronous entry point at the shapes that pick K1, K2 (NQ 64 and 256) and K3"""
    from kaito_b200 import _native
    return {
        "retrieve": lambda ix: _retrieve(ix, c.q[:8], c.qs[:8], K),
        "retrieve_allow": lambda ix: _retrieve(ix, c.q[8:12], c.qs[8:12], K, keyword_allow_bitmap=c.allow),
        "retrieve_pushdown": lambda ix: _retrieve(ix, c.q[12:16], c.qs[12:16], K, fusion_mode=_native.FILTER_PUSHDOWN,
                                                  keyword_allow_bitmap=c.allow),
        "dense_1": lambda ix: ix.search_dense(c.q[:1], 30),
        "dense_16": lambda ix: ix.search_dense(c.q[16:32], 30),
        "dense_256": lambda ix: ix.search_dense(c.q, 30),
        "bm25_30": lambda ix: ix.search_bm25(c.qs[:16], 30),
        "bm25_900": lambda ix: ix.search_bm25(c.qs[16:20], 900),
    }


@pytest.fixture(scope="module")
def corpus(oracle):
    return Corpus(oracle)


@pytest.fixture(scope="module")
def indexes(corpus):
    """(row storage, search_slots) -> (context, index over the corpus), built on first use"""
    from kaito_b200 import _native
    made = {}

    def get(storage, slots):
        if (storage, slots) not in made:
            ctx = _native.Context(0, search_slots=slots, row_storage=storage)
            made[(storage, slots)] = (ctx, corpus.build(ctx, f"conc_{storage}_{slots}"))
        return made[(storage, slots)]

    yield get
    for ctx, ix in made.values():
        ix.drop()
        ctx.close()


@pytest.fixture(scope="module")
def serial(corpus, indexes, oracle):
    """row storage -> the call mix's results run one at a time, a sample of them anchored to the oracle"""
    from kaito_b200 import _native
    o, c = oracle, corpus
    post = c.live_postings(o)
    P = o.pool_size(K)
    res = {}
    for storage in (_native.ROWS_DEVICE, _native.ROWS_HOST):
        _, ix = indexes(storage, 8)
        r = {name: fn(ix) for name, fn in call_mix(c).items()}
        dd, do = o.dense_topk(c.x, c.q[:3], 30, c.alive)
        assert np.array_equal(r["dense_256"][0][:3], dd) and np.array_equal(r["dense_256"][1][:3], do)
        assert same(r["dense_1"], (dd[:1], do[:1]))
        dd, do = o.dense_topk(c.x, c.q[16:18], 30, c.alive)
        assert np.array_equal(r["dense_16"][0][:2], dd) and np.array_equal(r["dense_16"][1][:2], do)
        for b in range(2):
            rs, ro = o.bm25_query(post, c.qs[b], 30, c.alive)
            assert np.array_equal(r["bm25_30"][0][b], rs) and np.array_equal(r["bm25_30"][1][b], ro)
            rs, ro = o.bm25_query(post, c.qs[16 + b], 900, c.alive)
            assert np.array_equal(r["bm25_900"][0][b], rs) and np.array_equal(r["bm25_900"][1][b], ro)
            dd, do = o.dense_topk(c.x, c.q[b:b + 1], P, c.alive)
            bs, bo = o.bm25_query(post, c.qs[b], P, c.alive)
            fin, de, sp, rk, od = o.fuse(dd[0], do[0], bs, bo, K)
            final, _, _, rank, ordn, count = r["retrieve"]
            assert count[b] == len(od) and np.array_equal(ordn[b, :count[b]], od)
            assert np.array_equal(final[b, :count[b]], fin) and np.array_equal(rank[b, :count[b]], rk)
            elig = c.allow & c.alive
            dd, do = o.dense_topk(c.x, c.q[12 + b:13 + b], P, elig)
            bs, bo = o.bm25_query(post, c.qs[12 + b], P, elig)
            fin, de, sp, rk, od = o.fuse(dd[0], do[0], bs, bo, K)
            final, _, _, rank, ordn, count = r["retrieve_pushdown"]
            assert count[b] == len(od) and np.array_equal(ordn[b, :count[b]], od) and np.array_equal(final[b, :count[b]], fin)
        res[storage] = r
    return res


# ------------------------------------------------------------------------------ (a) concurrent synchronous calls
ROUNDS = 3


def _configs():
    from kaito_b200 import _native
    out = []
    for slots in (1, 2, 8):
        out.append(pytest.param(_native.ROWS_DEVICE, slots, _native.DENSE_AUTO, id=f"device-auto-slots{slots}"))
        out.append(pytest.param(_native.ROWS_DEVICE, slots, _native.DENSE_TC_BF16, id=f"device-bf16-slots{slots}"))
        out.append(pytest.param(_native.ROWS_HOST, slots, _native.DENSE_AUTO, id=f"host-slots{slots}"))
    return out


@pytest.mark.parametrize("kernel", ["warp", "legacy"])
@pytest.mark.parametrize("storage,slots,mode", _configs())
def test_concurrent_sync_calls_equal_serial(corpus, indexes, serial, monkeypatch, storage, slots, mode, kernel):
    from kaito_b200 import _native
    monkeypatch.setenv("KRAG_BM25_KERNEL", kernel)
    _, ix = indexes(storage, slots)
    ix.set_dense_mode(mode)
    try:
        calls = list(call_mix(corpus).items())
        bad = []

        def thread(i):
            for r in range(ROUNDS):
                for j in range(len(calls)):
                    name, fn = calls[(i + r + j) % len(calls)]
                    if not same(fn(ix), serial[storage][name]):
                        bad.append((i, r, name))

        run_threads(8, thread)
        assert not bad, bad[:10]
    finally:
        ix.set_dense_mode(_native.DENSE_AUTO)


# ------------------------------------------------------------------------------ (b) stage calls on their own streams
class StageInputs:
    """device copies of the corpus queries for the stage API, and the output tensors of one caller"""

    def __init__(self, c, ix, B):
        dpad = int(ix.stats().dim_padded)
        q = np.zeros((B, dpad), np.float32)
        q[:, :c.d] = c.q[:B]
        flat, offs = ix._pack_terms(c.qs[:B])
        self.B, self.P, self.h_toff = B, 30, offs
        self.q = torch.from_numpy(q).cuda()
        self.terms = torch.from_numpy(flat.view(np.int32)).cuda()
        self.toff = torch.from_numpy(offs).cuda()

    def outputs(self):
        B, P = self.B, self.P
        e = lambda shape, dt: torch.empty(shape, dtype=dt, device="cuda")
        return {"dense": e((B, P), torch.int64), "bm25": e((B, P), torch.int64), "merged": e((B, P), torch.int64),
                "final": e((B, K), torch.float64), "dense_s": e((B, K), torch.float32), "sparse": e((B, K), torch.float32),
                "rank": e((B, K), torch.int32), "ordinal": e((B, K), torch.int64), "count": e((B,), torch.int32)}


def issue_stages(ctx, ix, inp, out, stream):
    """candidate stages, merge and fuse of one batch on `stream`; returns without synchronising"""
    B, P = inp.B, inp.P
    ix.dev_dense_candidates(B, inp.q.data_ptr(), P, out["dense"].data_ptr(), stream)
    ix.dev_bm25_candidates(B, inp.terms.data_ptr(), inp.toff.data_ptr(), P, out["bm25"].data_ptr(), stream, inp.h_toff)
    ctx.dev_merge(1, B, P, out["dense"].data_ptr(), out["merged"].data_ptr(), stream)
    ctx.dev_fuse(B, P, K, out["dense"].data_ptr(), out["bm25"].data_ptr(), 0.7, 0.3, 0, None, out["final"].data_ptr(),
                 out["dense_s"].data_ptr(), out["sparse"].data_ptr(), out["rank"].data_ptr(), out["ordinal"].data_ptr(),
                 out["count"].data_ptr(), stream)


def host(out):
    return {key: t.cpu().numpy() for key, t in out.items()}


@pytest.mark.parametrize("slots", [1, 8])
@pytest.mark.parametrize("storage", ["device", "host"])
def test_stage_calls_on_own_streams_equal_serial(corpus, indexes, serial, storage, slots):
    from kaito_b200 import _native
    storage = _native.ROWS_HOST if storage == "host" else _native.ROWS_DEVICE
    ctx, ix = indexes(storage, slots)
    shapes = [StageInputs(corpus, ix, B) for B in (4, 16)]       # K1, and K2 at NQ 64 on device rows
    ref = []
    s0 = torch.cuda.Stream()
    for inp in shapes:
        out = inp.outputs()
        issue_stages(ctx, ix, inp, out, s0.cuda_stream)
        s0.synchronize()
        ref.append(host(out))
    for inp, r in zip(shapes, ref):         # anchors: the stage pipeline is the host-buffer retrieve, key for key
        want = _retrieve(ix, corpus.q[:inp.B], corpus.qs[:inp.B], K)
        assert same((r["final"], r["dense_s"], r["sparse"], r["rank"], r["ordinal"], r["count"]), want)
        _, ordn = ix.search_dense(corpus.q[:inp.B], inp.P)
        assert np.array_equal(r["dense"].view(np.uint64) & np.uint64(0xFFFFFFFF), ordn.astype(np.uint64))
        assert np.array_equal(r["merged"], r["dense"])

    n_stage, rounds = 4, 4
    streams = [torch.cuda.Stream() for _ in range(n_stage)]
    outs = [[[inp.outputs() for inp in shapes] for _ in range(rounds)] for _ in range(n_stage)]
    torch.cuda.synchronize()
    calls = list(call_mix(corpus).items())
    bad = []

    def thread(i):
        if i < n_stage:
            for r in range(rounds):
                for j, inp in enumerate(shapes):
                    issue_stages(ctx, ix, inp, outs[i][r][j], streams[i].cuda_stream)
        else:
            for r in range(2):
                for j in range(len(calls)):
                    name, fn = calls[(i + r + j) % len(calls)]
                    if not same(fn(ix), serial[storage][name]):
                        bad.append(("sync", i, r, name))

    run_threads(2 * n_stage, thread)
    for s in streams:
        s.synchronize()
    for i in range(n_stage):
        for r in range(rounds):
            for j in range(len(shapes)):
                got = host(outs[i][r][j])
                for key in got:
                    if got[key].tobytes() != ref[j][key].tobytes():
                        bad.append(("stage", i, r, j, key))
    assert not bad, bad[:10]


# ------------------------------------------------------------------ (c), (d) stage work queued behind a sleeping stream
@pytest.fixture(params=["device", "host"])
def small(request, oracle):
    """one search slot, an index of 50k rows with tombstones (K1, or the streamed scan for host rows: no host
    synchronisation inside the stage calls), its corpus and the stage inputs"""
    from kaito_b200 import _native
    storage = _native.ROWS_HOST if request.param == "host" else _native.ROWS_DEVICE
    c = Corpus(oracle, n=50_000, vocab=3000, seed=51)
    ctx = _native.Context(0, search_slots=1, row_storage=storage)
    ix = c.build(ctx, "queued")
    yield ctx, ix, c
    ix.drop()
    ctx.close()


def test_stage_call_keeps_its_slot_until_its_stream_is_done(small, oracle):
    ctx, ix, c = small
    inp = StageInputs(c, ix, 4)
    A = torch.cuda.Stream()
    out = inp.outputs()
    ix.dev_dense_candidates(inp.B, inp.q.data_ptr(), inp.P, out["dense"].data_ptr(), A.cuda_stream)
    ix.dev_bm25_candidates(inp.B, inp.terms.data_ptr(), inp.toff.data_ptr(), inp.P, out["bm25"].data_ptr(), A.cuda_stream, inp.h_toff)
    A.synchronize()
    ref = host(out)
    q2 = c.q[100:108]
    ref2 = ix.search_dense(q2, 30)                       # also grows every buffer of the slot to these shapes
    dd, do = oracle.dense_topk(c.x, q2, 30, c.alive)
    assert same(ref2, (dd, do))

    out = inp.outputs()
    torch.cuda.synchronize()
    with torch.cuda.stream(A):
        torch.cuda._sleep(SLEEP_CYCLES)
    ix.dev_dense_candidates(inp.B, inp.q.data_ptr(), inp.P, out["dense"].data_ptr(), A.cuda_stream)
    ix.dev_bm25_candidates(inp.B, inp.terms.data_ptr(), inp.toff.data_ptr(), inp.P, out["bm25"].data_ptr(), A.cuda_stream, inp.h_toff)
    issued = torch.cuda.Event()
    issued.record(A)
    got2 = ix.search_dense(q2, 30)
    finished = issued.query()
    A.synchronize()
    assert finished, "search_dense returned while stage work that used its only slot was still queued"
    assert same(got2, ref2)
    got = host(out)
    assert got["dense"].tobytes() == ref["dense"].tobytes() and got["bm25"].tobytes() == ref["bm25"].tobytes()


def test_mutation_waits_for_issued_stage_work(small):
    ctx, ix, c = small
    inp = StageInputs(c, ix, 4)
    A = torch.cuda.Stream()
    out = inp.outputs()
    ix.dev_dense_candidates(inp.B, inp.q.data_ptr(), inp.P, out["dense"].data_ptr(), A.cuda_stream)
    A.synchronize()
    ref = out["dense"].cpu().numpy()
    top1 = int(ref[0, 0]) & 0xFFFFFFFF                   # ordinal == node id here
    out["dense"].fill_(0)
    torch.cuda.synchronize()
    with torch.cuda.stream(A):
        torch.cuda._sleep(SLEEP_CYCLES)
    ix.dev_dense_candidates(inp.B, inp.q.data_ptr(), inp.P, out["dense"].data_ptr(), A.cuda_stream)
    assert ix.remove(np.array([top1], np.uint64)) == 1
    A.synchronize()
    assert out["dense"].cpu().numpy().tobytes() == ref.tobytes(), "queued search saw a tombstone written after it was issued"
    _, ordn = ix.search_dense(c.q[:1], 30)               # and the removal is in place for what follows
    assert top1 not in ordn[0].tolist()


def test_sharded_retrieve_dev_then_remove(small, oracle):
    """the same ordering through the production ShardedRetriever (one shard): retrieve_dev leaves every stage queued on
    the current stream and returns; a removal that follows must not reach the queued kernels"""
    from kaito_b200.sharded import NativeStages, ShardedRetriever
    ctx, ix, c = small
    stages = NativeStages(ctx, ix)
    sr = ShardedRetriever(stages, torch.device("cuda", 0), stages.dim_padded())
    sr.commit(c.vocab, stages.n_rows())
    inp = StageInputs(c, ix, 4)
    ref = host(sr.retrieve_dev(inp.q, inp.terms, inp.toff, K, toff_host=inp.h_toff))
    assert same(tuple(ref[key] for key in ("final", "dense", "sparse", "rank", "ordinal", "count")),
                _retrieve(ix, c.q[:4], c.qs[:4], K))
    top1 = int(ref["ordinal"][0, 0])
    torch.cuda.synchronize()
    A = torch.cuda.Stream()
    with torch.cuda.stream(A):
        torch.cuda._sleep(SLEEP_CYCLES)
        out = sr.retrieve_dev(inp.q, inp.terms, inp.toff, K, toff_host=inp.h_toff)
    assert stages.remove(np.array([top1], np.uint64)) == 1
    A.synchronize()
    got = host(out)
    for key in ref:
        assert got[key].tobytes() == ref[key].tobytes(), key


# ------------------------------------------------------------------------------ (e) searches beside a writer
def test_searches_interleaved_with_writer_see_one_state_or_the_next(oracle):
    """one writer runs remove, add (into reserved space), commit, remove, compact; four readers search meanwhile.  Each
    reader result equals the serial result of one state of the sequence -- computed on a twin that replays it -- and a
    reader never sees an earlier state after a later one."""
    from kaito_b200 import _native
    c = Corpus(oracle, n=60_000, d=64, vocab=2000, seed=61)
    extra = Corpus(oracle, n=3000, d=64, vocab=2000, seed=62)
    rng = np.random.default_rng(63)
    rm1 = rng.choice(np.setdiff1d(np.arange(c.n), c.dead), 500, replace=False).astype(np.uint64)
    rm2 = np.concatenate([rng.choice(np.setdiff1d(np.arange(c.n), np.concatenate([c.dead, rm1])), 500, replace=False),
                          c.n + np.arange(0, extra.n, 7)]).astype(np.uint64)
    ops = [lambda ix: ix.remove(rm1),
           lambda ix: ix.add(c.n + np.arange(extra.n, dtype=np.uint64), extra.x, *extra.csr),
           lambda ix: ix.commit(c.vocab),
           lambda ix: ix.remove(rm2),
           lambda ix: ix.compact()]
    q, qs = c.q[:4], c.qs[:4]
    reads = {"retrieve": lambda ix: _retrieve(ix, q, qs, K), "dense": lambda ix: ix.search_dense(q, 30),
             "bm25": lambda ix: ix.search_bm25(qs, 30)}

    def read(ix, name):
        try:
            return reads[name](ix)
        except _native.KragError as e:         # after the add and before the commit the index has no postings
            assert e.code == _native.KRAG_E_STATE and name == "bm25"
            return (np.array([e.code]),)

    ctx = _native.Context(0, search_slots=8)
    try:
        twin = c.build(ctx, "twin")
        states = []
        for i in range(len(ops) + 1):
            states.append({name: read(twin, name) for name in reads})
            if i < len(ops):
                ops[i](twin)
        twin.drop()
        assert not same(states[0]["dense"], states[-1]["dense"])

        ix = c.build(ctx, "live")
        ix.reserve(c.n + extra.n, int(c.csr[0][-1] + extra.csr[0][-1]))
        seen, stop = [[] for _ in range(4)], threading.Event()

        def thread(i):
            if i == 4:
                for op in ops:
                    time.sleep(0.05)
                    op(ix)
                time.sleep(0.05)
                stop.set()
                return
            names = list(reads)
            r = 0
            while r < 400 and not (stop.is_set() and r > 20):
                name = names[(i + r) % len(names)]
                got = read(ix, name)
                seen[i].append((name, [s for s, st in enumerate(states) if same(got, st[name])]))
                r += 1

        run_threads(5, thread)
        for i in range(4):
            lo = 0
            for name, match in seen[i]:
                assert match, (i, name, "matches no state of the sequence")
                assert max(match) >= lo, (i, name, match, lo)
                lo = max(lo, min(m for m in match if m >= lo))
        ix.drop()
    finally:
        ctx.close()
