"""ColBERT late interaction (krag_late_rerank, krag_debug_late_vectors) at every shape its readers and the C ABI accept, not
only the two target checkpoints' points.  Three kinds of check, each named in its tests:

1. Exact (test_exact_*): maxsim_kernel states its arithmetic -- one fmaf chain over k = 0 .. dim - 1 in order, an exact max
   over the kept rows, one fp32 += of the row maxima in row order -- so given K5's own token vectors (each sequence's
   krag_debug_late_vectors alone) every pair's score must equal colbert_reference.maxsim_fp32_order bit for bit, and the
   positions and scores krag_late_rerank returns must equal a stable sort of those scores (descending, lower position
   first, -1 / NaN past the pair count).  The matrix, on 2-layer models of hidden 384 (dh 32) and 768 (dh 64), both
   precision modes (MaxSim is fp32 in both):
     dim 16 ... 256 (li_pad 128 and 256: two projection N tiles, zero columns past dim; maxsim_smem past 48 KB from dim
       192 on)                                                              -> test_exact_dims
     q_rows 3, 4, 8, 17, 31, 32 with key counts 3 ... q_rows (threads i >= q_rows idle, shorter row sums)
                                                                            -> test_exact_query_rows
     passage rows 3, 31, 32, 33, 63, 64, 65, 128, 180, 511, 512 (partial last MS_CHUNK = 32 chunks, whose stale rows must
       stay out of the max)                                                 -> every exact test
     keep masks: ColBERT-like random, all kept, exactly one kept row at chunk positions 0 / 7 / 8 / 24 / 31 / 32 / last
                                                                            -> test_exact_keep_masks
     0, 1, 7, 299, 300 pairs per query in one ragged call; top_k 1, 7, 300 -> test_exact_pairs_and_top_k
     n_queries 1, 2, 2 x SMs - 1, 2 x SMs, 2 x SMs + 1 (the slices per query go from 2 x SMs, striding through 300 pairs,
       down to one slice walking all of a query's pairs)                   -> test_exact_query_counts
2. fp64 (test_fp64_*): vectors and scores against colbert_reference.Fp64ColBERT with the bars of tests/test_gpu_colbert.py
   (fp32 mode: F = 40 times torch fp32's own error; fp16 mode: at most torch bf16 autocast's error) across the dim sweep on
   both hidden sizes, query_maxlen 3 / 8 / 32 with attend_to_mask_tokens true and false, passages of 1 ... 512 tokens, a
   2048-position model with passages up to 2048 (the KVL blocking over up to 32 key blocks) and hidden widths 128 ... 1024
   (the projection GEMM's K range).  Sequences checked against fp64 are sampled (bert_reference.sample).
3. The bench's calls (test_bench_call_bits): scripts/colbert_bench.py's 256 queries x 30 distinct 180-token passages (about
   21 forwards of at most RERANK_MAX_TOKENS = 65,536 tokens) at both full-depth shapes: every score has the bits of its
   query's call alone (and, sampled, of its pair alone), a passage's vectors have the same bits first and last in a
   forward, in calls of exactly 65,536 and 65,537 tokens and alone, and 4 queries x 30 pairs match fp64 and the exact
   restatement.
Random weights (no checkpoints offline)."""
import functools

import numpy as np
import pytest

from tests import bert_reference as br
from tests import colbert_reference as cr
from tests.test_gpu_colbert import F, SHAPES
from tests.test_gpu_colbert import _model as _full_model
from tests.test_gpu_colbert import _state as _full_state

EXACT = pytest.mark.skipif(not cr.exact_fmaf_available(), reason="the fmaf restatement needs a 64-bit long double significand")
PRECISIONS = ("fp32", "fp16")


def _cfg(hidden, heads, inter, layers=2, max_pos=512):
    return dict(num_hidden_layers=layers, hidden_size=hidden, num_attention_heads=heads, intermediate_size=inter,
                vocab_size=30522, max_position_embeddings=max_pos)


HIDDEN = {"h384": _cfg(384, 12, 1536), "h768": _cfg(768, 12, 3072)}     # dh 32, dh 64
DIMS = (16, 32, 48, 96, 128, 144, 176, 192, 240, 256)
Q_ROWS = (3, 4, 8, 17, 31, 32)
PASSAGE_ROWS = (3, 31, 32, 33, 63, 64, 65, 128, 180, 511, 512)
ONE_KEPT = (0, 7, 8, 24, 31, 32, -1)             # chunk positions of the only kept row (-1: the last row)
PAIRS = (300, 0, 1, 7, 299)                      # pairs per query, cycled over a call's queries
TOP_K = (1, 7, 300)
N_SAMPLE = 24
RERANK_MAX_TOKENS = 65536                        # engine.h: tokens per forward of a rerank call


@functools.lru_cache(maxsize=None)
def _state(name):
    return br.random_state(HIDDEN[name], 21)


@functools.lru_cache(maxsize=None)
def _weight(hidden, dim):
    return (np.random.default_rng(hidden + dim).standard_normal((dim, hidden)) / np.sqrt(hidden)).astype(np.float32)


_REF = {}


def _ref(cfg, state, w):
    """Fp64ColBERT of one encoder, shared across projections (one fp64 forward per sequence over a dim sweep)"""
    key = tuple(sorted(cfg.items()))
    if key not in _REF:
        _REF[key] = cr.Fp64ColBERT(cfg, state, w)
    return _REF[key].with_weight(w)


def _model(ctx, cfg, state, dim, precision):
    from kaito_b200 import _native
    e = _native.Embedder(ctx, cfg["num_hidden_layers"], cfg["hidden_size"], cfg["num_attention_heads"], cfg["intermediate_size"],
                         cfg["vocab_size"], cfg["max_position_embeddings"])
    e.set_late_interaction(_weight(cfg["hidden_size"], dim))
    e.load_state_dict(state)
    e.set_precision(precision)
    return e


def _query(g, q_rows, keys):
    """[CLS] [unused0] words [SEP] in the first `keys` rows, [MASK] expansion after them"""
    ids = np.full(q_rows, 103, np.int32)
    ids[0], ids[1], ids[keys - 1] = 101, 1, 102
    ids[2:keys - 1] = g.integers(1000, 30000, keys - 3)
    return ids


def _passage(g, rows, keep="random"):
    """(ids, keep) of a passage of `rows` rows; keep: "random" (about 15 % on the skiplist, [CLS] kept), "all", or the one
    kept row's index (-1: the last)"""
    ids = g.integers(1000, 30000, rows).astype(np.int32)
    ids[0] = 101
    ids[-1] = 102 if rows > 1 else 101
    if rows > 2:
        ids[1] = 2
    if keep == "random":
        k = (g.random(rows) > 0.15).astype(np.uint8)
        k[0] = 1
    elif keep == "all":
        k = np.ones(rows, np.uint8)
    else:
        k = np.zeros(rows, np.uint8)
        k[keep] = 1
    return ids, k


def _key_counts(q_rows, n):
    return [int(x) for x in np.linspace(3, q_rows, n).round()]


def _call(e, queries, keys, passages, cands, top_k):
    pp = np.concatenate([np.asarray(c, np.int32) for c in cands] + [np.zeros(0, np.int32)])
    poff = np.concatenate([[0], np.cumsum([len(c) for c in cands])]).astype(np.int32)
    d_off = np.concatenate([[0], np.cumsum([len(p[0]) for p in passages])]).astype(np.int32)
    return e.late_rerank(np.stack(queries), np.asarray(keys), np.concatenate([p[0] for p in passages]), d_off,
                         np.concatenate([p[1] for p in passages]), poff, pp, top_k)


def _alone(e, cache, ids, keys=None):
    """K5's vectors of one sequence in a call of its own (cached per ids and key count)"""
    k = (ids.tobytes(), keys)
    if k not in cache:
        cache[k] = e.debug_late_vectors(ids, np.array([0, len(ids)]), None if keys is None else np.array([keys]))
    return cache[k]


def _same(a, b):
    """equal bits where a number, NaN at the same places (the NaN past a query's pair count has no fixed payload)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


def check_exact(e, queries, keys, passages, cands, top_ks, what):
    """one krag_late_rerank call per top_k (and one at 300, which returns every pair): every pair's score equals
    maxsim_fp32_order on the vectors of its query and passage each encoded alone, and the selection equals the stable sort
    of those scores.  Returns the number of pairs checked."""
    cache, want = {}, {}
    restated = []
    for q, c in enumerate(cands):
        qv = _alone(e, cache, queries[q], keys[q])
        row = []
        for j in c:
            if (q, j) not in want:
                want[(q, j)] = cr.maxsim_fp32_order(qv, _alone(e, cache, passages[j][0]), passages[j][1])
            row.append(want[(q, j)])
        restated.append(np.asarray(row, np.float32))
    for top_k in sorted(set(top_ks) | {300}):
        pos, sc = _call(e, queries, keys, passages, cands, top_k)
        for q, r in enumerate(restated):
            wp, ws = cr.selection(r, top_k)
            if top_k == 300 and not _same(sc[q], ws):   # every pair's score is in the 300 returned: name the first wrong pair
                got = np.full(len(r), np.nan, np.float32)
                got[pos[q, :len(r)][pos[q, :len(r)] >= 0]] = sc[q, :len(r)][pos[q, :len(r)] >= 0]
                bad = [x for x in range(len(r)) if not _same(got[x], r[x])]
                j = int(bad[0]) if len(bad) else 0
                raise AssertionError(f"{what}: query {q} pair {j} (passage {cands[q][j]}, {len(passages[cands[q][j]][0])} rows): "
                                     f"{got[j]!r} != restated {r[j]!r}; {len(bad)} of {len(r)} pairs differ")
            assert np.array_equal(pos[q], wp) and _same(sc[q], ws), (what, q, top_k, pos[q][:8], wp[:8], sc[q][:8], ws[:8])
    return sum(len(c) for c in cands)


# ------------------------------------------------------------------------------------ 1. exact
@EXACT
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("hidden", list(HIDDEN))
def test_exact_dims(ctx, hidden, dim, precision):
    """3 queries of 32 rows (keys 3, 17, 32) against every passage length, each query ragged (all 11 / 11 reversed with
    repeats / 7), top_k cycled over the sweep"""
    e = _model(ctx, HIDDEN[hidden], _state(hidden), dim, precision)
    try:
        g = np.random.default_rng(dim)
        keys = [3, 17, 32]
        queries = [_query(g, 32, k) for k in keys]
        passages = [_passage(g, n) for n in PASSAGE_ROWS]
        cands = [list(range(11)), list(range(10, -1, -1)) + [4, 9, 4], [8, 0, 3, 10, 6, 2, 5]]
        check_exact(e, queries, keys, passages, cands, [TOP_K[DIMS.index(dim) % 3]], f"{hidden} dim {dim} {precision}")
    finally:
        e.destroy()


# q_rows -> (hidden, dim): the row counts spread over the projection widths and both head sizes
Q_ROWS_AT = {3: ("h384", 16), 4: ("h768", 144), 8: ("h384", 96), 17: ("h768", 256), 31: ("h384", 192), 32: ("h768", 128)}


@EXACT
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("q_rows", Q_ROWS)
def test_exact_query_rows(ctx, q_rows, precision):
    """queries of q_rows rows with key counts from 3 to q_rows in one call, against every passage length"""
    hidden, dim = Q_ROWS_AT[q_rows]
    e = _model(ctx, HIDDEN[hidden], _state(hidden), dim, precision)
    try:
        g = np.random.default_rng(100 + q_rows)
        keys = _key_counts(q_rows, 4)
        queries = [_query(g, q_rows, k) for k in keys]
        passages = [_passage(g, n) for n in PASSAGE_ROWS]
        cands = [list(g.permutation(11)) for _ in keys]
        check_exact(e, queries, keys, passages, cands, [7], f"q_rows {q_rows} {hidden} dim {dim} {precision}")
    finally:
        e.destroy()


@EXACT
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dim", [16, 96, 256])
def test_exact_keep_masks(ctx, dim, precision):
    """exactly one kept row at chunk positions 0 / 7 / 8 / 24 / 31 / 32 / last of passages of 33, 65, 180 and 512 rows
    (the row's chunk and its thread's u = 0 ... 3 slot; a partial last chunk), every passage length fully kept, and
    ColBERT-like random masks, in one call"""
    hidden = "h384" if dim <= 96 else "h768"
    e = _model(ctx, HIDDEN[hidden], _state(hidden), dim, precision)
    try:
        g = np.random.default_rng(200 + dim)
        passages = [_passage(g, n, p) for n in (33, 65, 180, 512) for p in ONE_KEPT]
        passages += [_passage(g, n, "all") for n in PASSAGE_ROWS] + [_passage(g, n) for n in PASSAGE_ROWS]
        keys = [10, 32]
        queries = [_query(g, 32, k) for k in keys]
        cands = [list(range(len(passages))), list(g.permutation(len(passages)))]
        check_exact(e, queries, keys, passages, cands, [300], f"keep masks {hidden} dim {dim} {precision}")
    finally:
        e.destroy()


@EXACT
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("top_k", TOP_K)
def test_exact_pairs_and_top_k(ctx, top_k, precision):
    """5 queries with 300, 0, 1, 7 and 299 pairs in one call, drawn with repeats from 12 passages of the listed lengths:
    about 53 slices per query, each striding through up to 300 pairs; equal scores (a passage twice) keep position order"""
    e = _model(ctx, HIDDEN["h384"], _state("h384"), 96, precision)
    try:
        g = np.random.default_rng(300 + top_k)
        passages = [_passage(g, n) for n in PASSAGE_ROWS + (1,)]
        keys = _key_counts(32, len(PAIRS))
        queries = [_query(g, 32, k) for k in keys]
        cands = [list(g.integers(0, len(passages), n)) for n in PAIRS]
        check_exact(e, queries, keys, passages, cands, [top_k], f"pairs top_k {top_k} {precision}")
    finally:
        e.destroy()


@functools.lru_cache(maxsize=None)
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


QUERY_COUNTS = {"1": lambda s: 1, "2": lambda s: 2, "2sm-1": lambda s: 2 * s - 1, "2sm": lambda s: 2 * s, "2sm+1": lambda s: 2 * s + 1}


@EXACT
@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n_queries", list(QUERY_COUNTS))
def test_exact_query_counts(ctx, n_queries, precision):
    """n_queries queries of 8 rows (keys 3 ... 8) with 300, 0, 1, 7, 299, ... pairs over 5 short passages: slices per
    query from 2 x SMs (one query, 300 pairs) down to one (more than 2 x SMs queries: one CTA walks all of a query's
    pairs).  The SM count is the device's."""
    n = QUERY_COUNTS[n_queries](_sm_count())
    e = _model(ctx, HIDDEN["h384"], _state("h384"), 32, precision)
    try:
        g = np.random.default_rng(400 + n)
        passages = [_passage(g, r) for r in (3, 32, 33, 65, 180)]
        keys = [3 + q % 6 for q in range(n)]
        queries = [_query(g, 8, k) for k in keys]
        cands = [list(g.integers(0, len(passages), PAIRS[q % len(PAIRS)])) for q in range(n)]
        check_exact(e, queries, keys, passages, cands, [TOP_K[n % 3]], f"{n} queries ({_sm_count()} SMs) {precision}")
    finally:
        e.destroy()


# ------------------------------------------------------------------------------------ 2. fp64
def check_fp64(e, ref, precision, queries, keys, passages, cands, what, sample=None):
    """vectors (one call of every query, one of every passage) and every pair's score against fp64: fp32 mode within F
    times torch fp32's error, fp16 mode within torch bf16 autocast's.  sample: the passages checked (default: all); the
    pairs of other passages are not scored against fp64"""
    fp16 = precision == "fp16"
    q_rows = len(queries[0])
    gq = e.debug_late_vectors(np.concatenate(queries), np.arange(0, q_rows * len(queries) + 1, q_rows), np.asarray(keys))
    gq = gq.reshape(len(queries), q_rows, -1)
    d_off = np.concatenate([[0], np.cumsum([len(p[0]) for p in passages])])
    gd = e.debug_late_vectors(np.concatenate([p[0] for p in passages]), d_off)
    pos, sc = _call(e, queries, keys, passages, cands, 300)
    sample = range(len(passages)) if sample is None else sample
    bar = (lambda i, k=None: ref.vectors_bf16(i, k)) if fp16 else (lambda i, k=None: ref.vectors(i, k)[1])
    q64 = [ref.vectors(q, k)[0] for q, k in zip(queries, keys)]
    qb = [bar(q, k) for q, k in zip(queries, keys)]
    d64 = {j: ref.vectors(passages[j][0])[0] for j in sample}
    db = {j: bar(passages[j][0]) for j in sample}
    v_k5 = max(max(float(np.abs(gq[i] - q64[i]).max()) for i in range(len(queries))),
               max(float(np.abs(gd[d_off[j]:d_off[j + 1]] - d64[j]).max()) for j in sample))
    v_t = max(max(float(np.abs(qb[i] - q64[i]).max()) for i in range(len(queries))),
              max(float(np.abs(db[j] - d64[j]).max()) for j in sample))
    s_k5 = s_t = 0.0
    for q, c in enumerate(cands):
        got = np.full(len(c), np.nan, np.float32)
        got[pos[q, :len(c)]] = sc[q, :len(c)]
        for p, j in enumerate(c):
            if j in d64:
                s64 = cr.maxsim(q64[q], d64[j], passages[j][1])
                s_k5 = max(s_k5, abs(float(got[p]) - s64))
                s_t = max(s_t, abs(cr.maxsim(qb[q], db[j], passages[j][1]) - s64))
    if fp16:
        print(f"colbert fp16 vs fp64 | {what} | vector err {v_k5:.2e} (bf16 autocast {v_t:.2e}) | score err {s_k5:.2e} "
              f"(bf16 autocast {s_t:.2e})")
        assert v_k5 <= v_t and s_k5 <= s_t, (what, v_k5, v_t, s_k5, s_t)
    else:
        vr, sr = v_k5 / max(v_t, 2.0 ** -23), s_k5 / max(s_t, 2.0 ** -23)
        print(f"colbert vs fp64 | {what} | vector err {v_k5:.2e} (torch fp32 {v_t:.2e}, ratio {vr:.2f}) | score err {s_k5:.2e} "
              f"(torch fp32 {s_t:.2e}, ratio {sr:.2f})")
        assert vr <= F and sr <= F, (what, vr, sr)


def _both_precisions(ctx, cfg, state, dim, body):
    ref = _ref(cfg, state, _weight(cfg["hidden_size"], dim))
    for precision in PRECISIONS:
        e = _model(ctx, cfg, state, dim, precision)
        try:
            body(e, ref, precision)
        finally:
            e.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", DIMS)
@pytest.mark.parametrize("hidden", list(HIDDEN))
def test_fp64_dims(ctx, hidden, dim):
    g = np.random.default_rng(500)                     # the same sequences at every dim: one fp64 forward each
    keys = [3, 12, 32]
    queries = [_query(g, 32, k) for k in keys]
    passages = [_passage(g, n) for n in (1, 3, 33, 65, 180, 512)]
    cands = [list(range(6))] * 3
    _both_precisions(ctx, HIDDEN[hidden], _state(hidden), dim,
                     lambda e, ref, p: check_fp64(e, ref, p, queries, keys, passages, cands, f"{hidden} dim {dim} {p}"))


@pytest.mark.gpu
@pytest.mark.parametrize("attend", [False, True], ids=["mask-not-keys", "attend-to-mask"])
@pytest.mark.parametrize("query_maxlen", [3, 8, 32])
def test_fp64_query_maxlen(ctx, query_maxlen, attend):
    """queries of query_maxlen rows with 0 ... query_maxlen - 3 words; attend_to_mask_tokens false: the [MASK] rows are no
    keys (the rerank path's key counts), true: every row is a key"""
    g = np.random.default_rng(600 + query_maxlen)
    real = _key_counts(query_maxlen, 4)
    queries = [_query(g, query_maxlen, k) for k in real]
    keys = [query_maxlen] * len(real) if attend else real
    passages = [_passage(g, n) for n in (20, 64, 180)]
    cands = [[0, 1, 2], [2, 1], [1], [0, 2]]
    _both_precisions(ctx, HIDDEN["h384"], _state("h384"), 96,
                     lambda e, ref, p: check_fp64(e, ref, p, queries, keys, passages, cands,
                                                  f"query_maxlen {query_maxlen} attend {attend} {p}"))


EDGE_LENS = [1, 2, 3, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 180, 255, 256, 257, 300, 511, 512]


@pytest.mark.gpu
@pytest.mark.parametrize("hidden", list(HIDDEN))
def test_fp64_passage_lengths(ctx, hidden):
    """passages of 1 ... 512 tokens (each side of the 16-row, 32-row chunk and 64-key block edges) in one call on a
    512-position model, sampled"""
    g = np.random.default_rng(700)
    passages = [_passage(g, n) for n in EDGE_LENS]
    keys = [5, 32]
    queries = [_query(g, 32, k) for k in keys]
    cands = [list(range(len(passages))), list(range(len(passages) - 1, -1, -1))]
    sample = br.sample(EDGE_LENS, N_SAMPLE // 2).tolist()
    dim = 96 if hidden == "h384" else 128
    _both_precisions(ctx, HIDDEN[hidden], _state(hidden), dim,
                     lambda e, ref, p: check_fp64(e, ref, p, queries, keys, passages, cands, f"passages 1..512 {hidden} {p}", sample))


LONG = _cfg(384, 12, 1536, max_pos=2048)          # test_gpu_embed_shapes.py's long-384: dh 32 over up to 32 key blocks


@pytest.mark.gpu
def test_fp64_long_model(ctx):
    """a 2048-position model, passages past 512 up to 2048 tokens among short ones: doc_maxlen up to
    max_position_embeddings"""
    g = np.random.default_rng(800)
    lens = [511, 1, 512, 5, 513, 575, 33, 576, 577, 1000, 64, 2047, 2, 2048]
    passages = [_passage(g, n) for n in lens]
    keys = [9, 32]
    queries = [_query(g, 32, k) for k in keys]
    cands = [list(range(len(lens))), [13, 11, 9, 4]]
    sample = sorted(set(br.sample(lens, 8).tolist()) | {11, 13})
    _both_precisions(ctx, LONG, br.random_state(LONG, 21), 128,
                     lambda e, ref, p: check_fp64(e, ref, p, queries, keys, passages, cands, f"long-384 {p}", sample))


WIDTHS = {  # hidden width: (config, dim) -- the projection GEMM's K = hidden; test_gpu_embed_shapes.py's tiny, mini, w640, large-dh32
    128: (_cfg(128, 2, 512), 32),
    256: (_cfg(256, 4, 1024), 144),
    640: (_cfg(640, 10, 2560), 192),
    1024: (_cfg(1024, 32, 4096, layers=1), 256),
}


@pytest.mark.gpu
@pytest.mark.parametrize("width", list(WIDTHS))
def test_fp64_hidden_widths(ctx, width):
    cfg, dim = WIDTHS[width]
    g = np.random.default_rng(900 + width)
    keys = [4, 32]
    queries = [_query(g, 32, k) for k in keys]
    passages = [_passage(g, n) for n in (2, 65, 180, 300)]
    cands = [[0, 1, 2, 3], [3, 1]]
    _both_precisions(ctx, cfg, br.random_state(cfg, 21), dim,
                     lambda e, ref, p: check_fp64(e, ref, p, queries, keys, passages, cands, f"hidden {width} dim {dim} {p}"))


# ------------------------------------------------------------------------------------ 3. the bench's calls
_BENCH_REF = {}


@pytest.mark.gpu
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_bench_call_bits(ctx, shape, precision):
    from scripts.colbert_bench import inputs
    cfg, st, w = _full_state(*SHAPES[shape], "bench")
    e = _full_model(ctx, cfg, st, w, precision)
    try:
        g = np.random.default_rng(30 + 180)
        q, keys, p_ids, d_off, keep, poff, pp = inputs(g, 256, 30, 180)
        plen, n_pass = 180, len(d_off) - 1
        assert d_off[-1] > 20 * RERANK_MAX_TOKENS
        pos, sc = e.late_rerank(q, keys, p_ids, d_off, keep, poff, pp, 30)
        full = np.full((256, 30), np.nan, np.float32)
        for i in range(256):
            full[i, pos[i]] = sc[i]
        assert not np.isnan(full).any()
        # every pair: the bits of its query's call alone; a sample: the bits of the pair alone
        psg = lambda j: (p_ids[d_off[j]:d_off[j + 1]], keep[d_off[j]:d_off[j + 1]])          # noqa: E731
        for i in range(256):
            ps = [psg(j) for j in range(30 * i, 30 * i + 30)]
            a_pos, a_sc = _call(e, [q[i]], [keys[i]], ps, [list(range(30))], 30)
            alone = np.full(30, np.nan, np.float32)
            alone[a_pos[0]] = a_sc[0]
            assert _same(alone, full[i]), (shape, precision, i)
        for i, j in zip(g.integers(0, 256, 12), g.integers(0, 30, 12)):
            _, one = _call(e, [q[i]], [keys[i]], [psg(30 * i + j)], [[0]], 1)
            assert _same(one[0, 0], full[i, j]), (shape, precision, i, j)
        # a passage's vectors: first / last in a forward (364 passages of 180 rows fit in 65,536 tokens), in calls of exactly
        # 65,536 and 65,537 tokens (a 16- / 17-row passage after the 364), and alone
        per = RERANK_MAX_TOKENS // plen
        cache = {}
        ids = lambda j: psg(j)[0]                                                           # noqa: E731
        many = e.debug_late_vectors(p_ids[:d_off[2 * per + 1]], d_off[:2 * per + 2])
        for j in (0, per - 1, per, 2 * per - 1, 2 * per):
            assert _same(many[d_off[j]:d_off[j + 1]], _alone(e, cache, ids(j))), (shape, precision, j)
        for tail in (16, 17):
            extra = _passage(g, tail)[0]
            toks = np.concatenate([p_ids[:d_off[per]], extra])
            assert len(toks) == RERANK_MAX_TOKENS + tail - 16
            v = e.debug_late_vectors(toks, np.append(d_off[:per + 1], len(toks)))
            for j in (0, per - 1):
                assert _same(v[d_off[j]:d_off[j + 1]], _alone(e, cache, ids(j))), (shape, precision, tail, j)
            assert _same(v[d_off[per]:], _alone(e, cache, extra)), (shape, precision, tail)
        # 4 queries x 30 pairs: MaxSim of the fetched vectors restated exactly, and fp64
        key = (shape,)
        if key not in _BENCH_REF:
            _BENCH_REF.clear()
            _BENCH_REF[key] = cr.Fp64ColBERT(cfg, st, w)
        ref = _BENCH_REF[key]
        qs = (0, 85, 170, 255)
        exact = cr.exact_fmaf_available()
        s_k5 = s_t = 0.0
        for i in qs:
            qv = _alone(e, cache, q[i], int(keys[i]))
            q64 = ref.vectors(q[i], keys[i])[0]
            qb = ref.vectors_bf16(q[i], keys[i]) if precision == "fp16" else ref.vectors(q[i], keys[i])[1]
            for j in range(30):
                pid, pk = psg(30 * i + j)
                if exact:
                    assert cr.maxsim_fp32_order(qv, _alone(e, cache, pid), pk) == full[i, j], (shape, precision, i, j)
                d64 = ref.vectors(pid)[0]
                db = ref.vectors_bf16(pid) if precision == "fp16" else ref.vectors(pid)[1]
                s64 = cr.maxsim(q64, d64, pk)
                s_k5 = max(s_k5, abs(float(full[i, j]) - s64))
                s_t = max(s_t, abs(cr.maxsim(qb, db, pk) - s64))
        print(f"colbert bench call | {shape} {precision} | {d_off[-1]} passage tokens | score err {s_k5:.2e} | "
              f"{'bf16 autocast' if precision == 'fp16' else 'torch fp32'} {s_t:.2e}")
        if precision == "fp16":
            assert s_k5 <= s_t, (s_k5, s_t)
        else:
            assert s_k5 <= F * max(s_t, 2.0 ** -23), (s_k5, s_t)
    finally:
        e.destroy()
