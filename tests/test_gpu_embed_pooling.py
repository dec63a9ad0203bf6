"""K5 with mean pooling (krag_embedder_set_pooling(KRAG_POOL_MEAN), mean_normalize_kernel): the sentence-transformers models
users pick instead of bge (all-MiniLM-L6/L12-v2, e5-base/large-v2, gte) pool by the mean over every token of the sequence,
[CLS] and [SEP] included, before the L2 normalisation.  Held to the bounds of tests/test_gpu_embed.py against
transformers.BertModel in fp64 with the mean and the normalisation applied to last_hidden_state in numpy: the L2^2 score
against 64 unit rows moves by less than 1e-4, and the error is at most F = 40 times torch fp32's own.  Also: the device and
host outputs, graph replay and a pooling switch give the same bits; a MiniLM-shaped snapshot goes through
GpuBertEmbedding.from_pretrained and a VectorStore's /retrieve."""
import numpy as np
import pytest

from tests import bert_reference as br
from tests import st_snapshot as sn
from tests.test_gpu_embed import _assert_fp64, _bench_queries, _embedder

MODELS = {   # BertConfig of the sentence-transformers checkpoints (random weights here: no checkpoints offline)
    "all-MiniLM-L6": dict(num_hidden_layers=6, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=30522,
                          max_position_embeddings=512),
    "all-MiniLM-L12": dict(num_hidden_layers=12, hidden_size=384, num_attention_heads=12, intermediate_size=1536,
                           vocab_size=30522, max_position_embeddings=512),
    "e5-base": dict(num_hidden_layers=12, hidden_size=768, num_attention_heads=12, intermediate_size=3072, vocab_size=30522,
                    max_position_embeddings=512),
    "e5-large": dict(num_hidden_layers=24, hidden_size=1024, num_attention_heads=16, intermediate_size=4096, vocab_size=30522,
                     max_position_embeddings=512),
}
REGIMES = ["bench", "stressed"]


class MeanRef:
    """the fp64 BertModel of bert_reference (its Linear range hooks included) and its fp32 twin, mean-pooled"""

    def __init__(self, cfg, state, ref64):
        self.cfg, self.state, self.ref, self._m32 = cfg, state, ref64, None

    def __call__(self, toks):
        """(fp64 embeddings, fp32 embeddings, largest Linear operand of the fp64 forward)"""
        if self._m32 is None:
            self._m32 = br.Fp64Bert(self.cfg, self.state).m64.float()
        self.ref.range_max = 0.0
        return br.mean_pool(self.ref.m64, toks), br.mean_pool(self._m32, toks), self.ref.range_max


def _setup(ctx, model, regime, seed=0):
    import bench
    from kaito_b200 import _native
    cfg = MODELS[model]
    if regime == "stressed":
        state, ref = br.stressed_state(cfg, seed)
    else:
        state = bench.random_bert_state(cfg, seed)
        ref = br.Fp64Bert(cfg, state)
    emb = _embedder(ctx, cfg, state)
    emb.set_pooling(_native.POOL_MEAN)
    return emb, MeanRef(cfg, state, ref)


def _check(label, emb, ref, toks, n_sample, flat=True):
    from kaito_b200 import _native
    got = emb.embed_flat(*_native.Embedder.pack(toks)) if flat else emb.embed(toks)
    idx = br.sample([len(t) for t in toks], n_sample)
    _assert_fp64(f"mean {label} ({len(toks)} seqs, {sum(len(t) for t in toks)} tok, {len(idx)} checked)", got[idx],
                 *ref([toks[i] for i in idx]))
    return got


# ------------------------------------------------------------------------------------------------ against fp64
@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("model", list(MODELS))
def test_query_batch_mean_matches_fp64(ctx, model, regime):
    """256 queries x 32 tokens, the bench's query recipe"""
    emb, ref = _setup(ctx, model, regime)
    try:
        _check(f"{model} {regime} 256x32", emb, ref, _bench_queries(), 32)
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
def test_ragged_mean_matches_fp64(ctx, model):
    """one batch of lengths 1..512 (each side of the 16-row query and 32 / 64-key attention blocks, then random lengths),
    stressed weights"""
    emb, ref = _setup(ctx, model, "stressed", seed=3)
    try:
        g = np.random.default_rng(3)
        lens = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512]
        lens += g.integers(1, 513, 26).tolist()
        toks = [g.integers(1000, 30000, n) for n in lens]
        _check(f"{model} stressed ragged 1-512", emb, ref, toks, 6 if model == "e5-large" else 12)
        edge = [toks[i] for i in (0, 1, 2, 3, 4)]                  # the shortest: every one of them checked, host path
        _assert_fp64(f"mean {model} stressed 1-9 tokens", emb.embed(edge), *ref(edge))
    finally:
        emb.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("model,regime", [("all-MiniLM-L6", "bench"), ("all-MiniLM-L6", "stressed"), ("e5-large", "bench")])
def test_index_batch_mean_matches_fp64(ctx, model, regime):
    """/index: 256 chunks x 256 tokens = 65,536 tokens (all-MiniLM's max_seq_length) through embed_flat, the service's call"""
    emb, ref = _setup(ctx, model, regime, seed=5)
    try:
        g = np.random.default_rng(5)
        toks = [g.integers(1000, 30000, 256) for _ in range(256)]
        _check(f"{model} {regime} 256x256", emb, ref, toks, 8 if model == "e5-large" else 16)
    finally:
        emb.destroy()


# ----------------------------------------------------------------------------------------------- bits and layout
SMALL = dict(num_hidden_layers=2, hidden_size=384, num_attention_heads=12, intermediate_size=1536, vocab_size=1000,
             max_position_embeddings=512)


@pytest.mark.gpu
def test_mean_dev_host_replay_and_write_after_read(ctx):
    """krag_embed and krag_embed_dev (ld_out > hidden) give the same bits, the padding columns keep their sentinel, the final
    writer waits for the consumer stream's earlier work (it sleeps ~50 ms, then copies the buffer), and the third call of a
    shape (a graph replay) gives the bits of the first"""
    import torch
    from kaito_b200 import _native
    emb = _embedder(ctx, SMALL, br.random_state(SMALL, 41))
    emb.set_pooling(_native.POOL_MEAN)
    try:
        d, B = SMALL["hidden_size"], 6
        ld = d + 32
        g = np.random.default_rng(41)
        lens = [3, 9, 1, 20, 7, 130]
        toks1 = [g.integers(0, 1000, n) for n in lens]
        toks2 = [g.integers(0, 1000, n) for n in lens]
        want1 = emb.embed(toks1)
        assert np.array_equal(emb.embed(toks1), want1) and np.array_equal(emb.embed(toks1), want1)   # eager, capture, replay
        want2 = emb.embed(toks2)                                                                       # replay, new tokens
        buf = torch.full((B + 3, ld), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        emb.embed_dev(*_native.Embedder.pack(toks1), buf.data_ptr(), ld, s.cuda_stream)
        with torch.cuda.stream(s):
            snap = buf.clone()
        s.synchronize()
        got = snap.cpu().numpy()
        assert np.array_equal(got[:B, :d], want1)
        assert np.isnan(got[:B, d:]).all() and np.isnan(got[B:]).all()

        with torch.cuda.stream(s):
            torch.cuda._sleep(100_000_000)            # ~50 ms of clock cycles
            old = buf.clone()
        emb.embed_dev(*_native.Embedder.pack(toks2), buf.data_ptr(), ld, s.cuda_stream)
        with torch.cuda.stream(s):
            new = buf.clone()
        s.synchronize()
        assert np.array_equal(old.cpu().numpy()[:B, :d], want1), "the embeddings overwrote rows the consumer was still reading"
        assert np.array_equal(new.cpu().numpy()[:B, :d], want2)
        assert np.isnan(new.cpu().numpy()[:B, d:]).all()
    finally:
        emb.destroy()


@pytest.mark.gpu
def test_pooling_switch_keeps_bits(ctx):
    """mean and back to CLS gives a fresh CLS embedder's bits (captured graphs do not hold the pooling); the mode may be set
    before finalize; an unknown mode is KRAG_E_INVALID and changes nothing"""
    from kaito_b200 import _native
    state = br.random_state(SMALL, 43)
    g = np.random.default_rng(43)
    toks = [g.integers(0, 1000, n) for n in (5, 17, 64, 2)]
    fresh = _embedder(ctx, SMALL, state)
    emb = _embedder(ctx, SMALL, state)
    early = _native.Embedder(ctx, 2, 384, 12, 1536, 1000, 512)
    try:
        cls = fresh.embed(toks)
        assert np.array_equal(emb.embed(toks), cls) and np.array_equal(emb.embed(toks), cls)    # graph captured under CLS
        emb.set_pooling(_native.POOL_MEAN)
        mean = emb.embed(toks)
        assert not np.array_equal(mean, cls)
        assert np.array_equal(emb.embed(toks), mean)
        emb.set_pooling(_native.POOL_CLS)
        assert np.array_equal(emb.embed(toks), cls)
        with pytest.raises(_native.KragError) as e:
            emb.set_pooling(2)
        assert e.value.code == _native.KRAG_E_INVALID
        assert np.array_equal(emb.embed(toks), cls)
        early.set_pooling(_native.POOL_MEAN)
        early.load_state_dict(state)
        assert np.array_equal(early.embed(toks), mean)
    finally:
        fresh.destroy(); emb.destroy(); early.destroy()


# ------------------------------------------------------------------------------------------ snapshot and service
MINI = dict(MODELS["all-MiniLM-L6"], vocab_size=len(sn.VOCAB))
WORDS = [w for w in sn.VOCAB if not w.startswith(("[", "##"))]


def _snapshot(tmp_path):
    import bench
    state = bench.random_bert_state(MINI, 47)
    return sn.write(tmp_path / "minilm", sn.layout("minilm", dict(sn.MINILM_L6, vocab_size=len(sn.VOCAB))), state=state), state


def _texts(g, n, lo=3, hi=40):
    return [" ".join(g.choice(WORDS, int(g.integers(lo, hi)))) for _ in range(n)]


@pytest.mark.gpu
def test_from_pretrained_minilm_snapshot(ctx, tmp_path):
    """the snapshot's spec reaches the forward: mean pooling, 256-token truncation, no query instruction; the embeddings are
    the direct Embedder's with set_pooling(MEAN), bit for bit"""
    from kaito_b200 import _native
    from kaito_b200.embedding import GpuBertEmbedding
    path, state = _snapshot(tmp_path)
    g = np.random.default_rng(47)
    texts = _texts(g, 20) + [" ".join(g.choice(WORDS, 400))]
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    direct = _embedder(ctx, MINI, state)
    direct.set_pooling(_native.POOL_MEAN)
    try:
        assert ge.pooling == "mean" and ge.query_instruction is None and ge.tokenizer.max_length == 256
        toks = ge.tokenizer.encode_batch(texts)
        assert len(toks[-1]) == 256
        got = ge.get_text_embedding_batch(texts)
        assert np.array_equal(got, direct.embed(toks))
        # no instruction before the query (same batch, same bits)
        assert np.array_equal(ge.get_query_embedding_batch(texts[:4]), ge.get_text_embedding_batch(texts[:4]))
        assert np.array_equal(ge.get_query_embedding(texts[0]), ge.get_text_embedding(texts[0]))
    finally:
        ge._emb.destroy(); direct.destroy()


@pytest.mark.gpu
def test_vector_store_retrieve_on_minilm_snapshot(ctx, tmp_path, monkeypatch):
    """/index then /retrieve through VectorStore on the snapshot: every returned dense L2^2 is the fp64 mean-pooled one within
    1e-4, and the dense ranking follows fp64 wherever two fp64 distances differ by more than 1e-4"""
    from kaito_b200.embedding import GpuBertEmbedding
    from kaito_b200.vector_store import VectorStore
    monkeypatch.setenv("KRAG_COMPONENT_SCORES", "1")
    path, state = _snapshot(tmp_path)
    ref = br.Fp64Bert(MINI, state)
    g = np.random.default_rng(53)
    docs = [{"text": t} for t in dict.fromkeys(_texts(g, 60, 5, 60))]
    queries = _texts(g, 6, 2, 8)
    ge = GpuBertEmbedding.from_pretrained(ctx, path)
    try:
        store = VectorStore(ge, ctx)
        store.index_documents("pooling_e2e", docs)
        enc = ge.tokenizer.encode_batch
        for q in queries:
            q64 = br.mean_pool(ref.m64, enc([q]))[0]
            res = store.retrieve("pooling_e2e", q, max_node_count=10)["results"]
            dense = [r for r in res if r["dense_score"] is not None]
            assert dense, q
            d64 = br.mean_pool(ref.m64, enc([r["text"] for r in dense]))
            l2 = ((d64 - q64) ** 2).sum(1)
            assert np.abs(np.array([r["dense_score"] for r in dense]) - l2).max() < 1e-4, q
            ranked = store.dense_candidates("pooling_e2e", q, len(docs))
            assert len(ranked) == len(docs)
            r64 = ((br.mean_pool(ref.m64, enc([n.text for n, _ in ranked])) - q64) ** 2).sum(1)
            assert np.abs(np.array([s for _, s in ranked]) - r64).max() < 1e-4, q
            assert (np.diff(r64) > -1e-4).all(), (q, np.diff(r64).min())
    finally:
        ge._emb.destroy()
