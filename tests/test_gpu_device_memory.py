"""Every device allocation of libkaito_rag has one owner, DevArray (kaito_b200/csrc/engine.h), which keeps a process-wide
count of the bytes it holds (krag_device_bytes).  The GPU tests below run each object's life cycle, including the failure
paths that used to leak, on a Context of their own and check that the count comes back to where it started.  They never
fill device memory: the out-of-memory paths are left to reading the code."""
import contextlib
import glob
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kaito_b200", "csrc")


def test_only_devarray_calls_cuda_malloc_and_free():
    """a raw cudaMalloc / cudaFree anywhere else is an allocation without an owner"""
    alloc = re.compile(r"\bcuda(Malloc|Free)\b")
    engine = open(os.path.join(CSRC, "engine.h")).read()
    start = engine.index("struct DevArray {")
    depth, end = 0, start
    for end in range(start, len(engine)):
        depth += {"{": 1, "}": -1}.get(engine[end], 0)
        if depth == 0 and engine[end] == "}":
            break
    assert alloc.search(engine[start:end]), "DevArray no longer allocates: update this test"
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*"))):
        if not path.endswith((".cu", ".cuh", ".h", ".cpp")):
            continue
        txt = open(path).read()
        for m in alloc.finditer(txt):
            if not (path.endswith("engine.h") and start < m.start() < end):
                found.append(f"{os.path.basename(path)}:{txt.count(chr(10), 0, m.start()) + 1}")
    assert not found, found


@contextlib.contextmanager
def own_context():
    """a Context of the test's own; closing it must bring the device byte count back to where it was before"""
    from kaito_b200 import _native
    before = _native.device_bytes()
    c = _native.Context(device_id=0)
    try:
        yield c
    finally:
        c.close()
    assert _native.device_bytes() == before


def _corpus(n=300, dim=64, vocab=500, seed=0):
    g = np.random.default_rng(seed)
    vecs = g.standard_normal((n, dim)).astype(np.float32)
    lens = g.integers(1, 12, n)
    offs = np.zeros(n + 1, np.int64)
    offs[1:] = np.cumsum(lens)
    ids = g.integers(0, vocab, int(offs[-1])).astype(np.uint32)
    tf = g.integers(1, 4, int(offs[-1])).astype(np.uint16)
    return np.arange(n, dtype=np.uint64), vecs, offs, ids, tf, lens.astype(np.uint32)


def _hybrid_index(c, name, dim=64, vocab=500):
    node_ids, vecs, offs, ids, tf, dl = _corpus(dim=dim, vocab=vocab)
    ix = c.create_index(name, dim)
    ix.add(node_ids, vecs, offs, ids, tf, dl)
    return ix, vecs, int(ids.max())


@pytest.mark.gpu
def test_index_round_trip_frees_everything():
    from kaito_b200 import _native
    with own_context() as c:
        base = _native.device_bytes()
        ix, vecs, _ = _hybrid_index(c, "mem-round-trip")
        ix.commit(500)
        d, o = ix.search_dense(vecs[:4], 10)
        assert (o[:, 0] == np.arange(4)).all()
        ix.search_bm25([[1, 2, 3], [7]], 10)
        out = ix.retrieve(vecs[:4], [[1, 2], [3], [4, 5, 6], [9]], 5)
        assert (out["count"] >= 1).all()
        assert _native.device_bytes() > base
        ix.drop()
        # what is left are the search workspaces the queries grew: they belong to the context and go with close()


@pytest.mark.gpu
def test_rejected_commit_leaves_nothing_behind():
    from kaito_b200 import _native
    with own_context() as c:
        base = _native.device_bytes()
        ix, _, max_id = _hybrid_index(c, "mem-rejected")
        for commit in (ix.commit, ix.commit_local):
            with pytest.raises(_native.KragError) as e:
                commit(max_id)          # vocab must exceed the largest term id
            assert e.value.code == _native.KRAG_E_INVALID
        ix.drop()
        assert _native.device_bytes() == base


@pytest.mark.gpu
def test_truncated_snapshot_leaves_nothing_behind(tmp_path):
    from kaito_b200 import _native
    with own_context() as c:
        ix, _, _ = _hybrid_index(c, "mem-snapshot")
        ix.commit(500)
        ix.persist(str(tmp_path))
        ix.drop()
        base = _native.device_bytes()
        path = tmp_path / "krag_index.bin"
        data = path.read_bytes()
        path.write_bytes(data[: len(data) - 64])
        with pytest.raises(_native.KragError) as e:
            c.load_index("mem-snapshot-2", str(tmp_path))
        assert e.value.code == _native.KRAG_E_IO
        assert _native.device_bytes() == base


def _bert_state(layers=1, hidden=128, inter=512, vocab=100, max_pos=64, seed=0):
    g = np.random.default_rng(seed)

    def r(*shape):
        return (0.05 * g.standard_normal(shape)).astype(np.float32)

    st = {"embeddings.word_embeddings.weight": r(vocab, hidden), "embeddings.position_embeddings.weight": r(max_pos, hidden),
          "embeddings.token_type_embeddings.weight": r(2, hidden), "embeddings.LayerNorm.weight": 1 + r(hidden),
          "embeddings.LayerNorm.bias": r(hidden)}
    for l in range(layers):
        p = f"encoder.layer.{l}."
        for m in ("query", "key", "value"):
            st[p + f"attention.self.{m}.weight"], st[p + f"attention.self.{m}.bias"] = r(hidden, hidden), r(hidden)
        st[p + "attention.output.dense.weight"], st[p + "attention.output.dense.bias"] = r(hidden, hidden), r(hidden)
        st[p + "attention.output.LayerNorm.weight"], st[p + "attention.output.LayerNorm.bias"] = 1 + r(hidden), r(hidden)
        st[p + "intermediate.dense.weight"], st[p + "intermediate.dense.bias"] = r(inter, hidden), r(inter)
        st[p + "output.dense.weight"], st[p + "output.dense.bias"] = r(hidden, inter), r(hidden)
        st[p + "output.LayerNorm.weight"], st[p + "output.LayerNorm.bias"] = 1 + r(hidden), r(hidden)
    return st


@pytest.mark.gpu
def test_embedder_frees_everything():
    from kaito_b200 import _native
    state = _bert_state()
    with own_context() as c:
        base = _native.device_bytes()
        emb = _native.Embedder(c, 1, 128, 2, 512, 100, 64)
        try:
            emb.load_state_dict(state)
            small = emb.embed([[1, 2, 3]])
            again = emb.embed([[1, 2, 3]])          # the second call of a shape is captured into a graph
            assert np.abs(small - again).max() < 1e-6
            big = emb.embed([list(range(1, 41)), [5] * 17, [9, 8, 7]])   # grows the workspaces
            assert big.shape == (3, 128) and np.allclose(np.linalg.norm(big, axis=1), 1.0, atol=1e-5)
            assert _native.device_bytes() > base
        finally:
            emb.destroy()
        assert _native.device_bytes() == base

        broken = dict(state)
        del broken["encoder.layer.0.attention.self.key.bias"]
        emb = _native.Embedder(c, 1, 128, 2, 512, 100, 64)
        try:
            with pytest.raises(_native.KragError) as e:
                emb.load_state_dict(broken)
            assert e.value.code == _native.KRAG_E_INVALID
        finally:
            emb.destroy()
        assert _native.device_bytes() == base


@pytest.mark.gpu
def test_debug_gemms_free_their_buffers():
    from kaito_b200 import _native
    g = np.random.default_rng(1)
    M, N, K = 16, 128, 64
    A, B = g.standard_normal((M, K)).astype(np.float32), g.standard_normal((N, K)).astype(np.float32)
    bias, R = g.standard_normal(N).astype(np.float32), g.standard_normal((M, N)).astype(np.float32)
    with own_context() as c:
        base = _native.device_bytes()
        got = _native.debug_gemm_tf32(c, A, B, bias, R, gelu=True)
        assert got.shape == (M, N) and np.isfinite(got).all()
        assert _native.device_bytes() == base
        got = _native.debug_linear_ln(c, A, B, bias, R, np.ones(N, np.float32), np.zeros(N, np.float32))
        assert got.shape == (M, N) and np.isfinite(got).all()
        assert _native.device_bytes() == base


@pytest.mark.gpu
def test_p2p_exchange_frees_its_mailbox():
    from kaito_b200 import _native
    with own_context() as c:
        base = _native.device_bytes()
        p = _native.P2PExchange(c, 0, 1, 8, 16)
        p.connect(p.handle.reshape(1, 64))
        assert _native.device_bytes() > base
        p.destroy()
        assert _native.device_bytes() == base


@pytest.mark.gpu
def test_context_close_frees_its_workspaces():
    from kaito_b200 import _native
    before = _native.device_bytes()
    c = _native.Context(device_id=0)
    try:
        ix, vecs, _ = _hybrid_index(c, "mem-context")
        ix.search_dense(vecs[:8], 10)
        ix.drop()
        assert _native.device_bytes() > before     # the search slot's workspaces
    finally:
        c.close()
    assert _native.device_bytes() == before
