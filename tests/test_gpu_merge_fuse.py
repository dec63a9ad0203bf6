"""K4 (merge_fuse.cu) against exact references, through the device-pointer stage API.

merge: G sorted-key lists -> the P smallest keys (krag_dev_merge); the reference is numpy's sort of the non-pad keys.
fuse : the reference's weighted fusion (krag_dev_fuse); the references are oracle.fuse (the C restatement in IEEE fp64)
       and, for mode 0, oracle.py_fuse (the line-by-line Python _fuse).  Every output array must match bit for bit."""
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PAD = np.uint64(0xFFFFFFFFFFFFFFFF)
M32 = np.uint64(0xFFFFFFFF)


def obits(v):
    """order-preserving bits of fp32 values (common.cuh f32_ordered_bits)"""
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & np.uint64(0x80000000), ~u & M32, u | np.uint64(0x80000000))


def key_asc(v, ordn):
    return (obits(v) << np.uint64(32)) | np.asarray(ordn, np.uint64)


def key_desc(v, ordn):
    return ((~obits(v) & M32) << np.uint64(32)) | np.asarray(ordn, np.uint64)


def val_asc(keys):
    o = (np.asarray(keys, np.uint64) >> np.uint64(32)).astype(np.uint64)
    u = np.where(o & np.uint64(0x80000000), o & np.uint64(0x7FFFFFFF), ~o & M32).astype(np.uint32)
    return u.view(np.float32)


def val_desc(keys):
    return val_asc(((~(np.asarray(keys, np.uint64) >> np.uint64(32))) & M32) << np.uint64(32))


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64 if a.dtype == np.uint64 else np.int32)).cuda()


# --------------------------------------------------------------------------------------------------------- merge
def _merge_keys(order, n_lists, batch, P, rng):
    """[n_lists, batch, P] keys in the order the kernel reads them (list by list).  Ordinals are unique per batch entry:
    an odd multiplier is a bijection mod 2^32."""
    idx = np.arange(n_lists * P, dtype=np.uint64).reshape(n_lists, 1, P)
    b = np.arange(batch, dtype=np.uint64).reshape(1, batch, 1)
    ordn = ((idx * np.uint64(2654435761) + b * np.uint64(7919)) & M32)
    ordn = np.broadcast_to(ordn, (n_lists, batch, P))
    if order == "asc":            # ascending across lists: every key passes until the first prune
        v = (idx.astype(np.float32) * np.float32(0.25) - np.float32(3.0)) + np.zeros((1, batch, 1), np.float32)
    elif order == "desc":         # descending: every key beats the threshold, the buffer churns at every epoch
        v = (-idx.astype(np.float32) * np.float32(0.25) + np.float32(3.0)) + np.zeros((1, batch, 1), np.float32)
    elif order == "same":         # identical value bits: the ordinal alone decides
        v = np.full((n_lists, batch, P), 0.625, np.float32)
    else:                         # random, with repeats of values
        v = rng.choice(np.float32([-1.5, 0.0, 0.3, 2.0, 7.0]), size=(n_lists, batch, P)) if order == "dup" else \
            rng.standard_normal((n_lists, batch, P)).astype(np.float32)
    keys = key_asc(np.broadcast_to(v, (n_lists, batch, P)), ordn)
    if order in ("random", "dup"):
        # sorted lists of mixed lengths padded with KEY_PAD, as the shards return them; some lists and the last
        # batch entry are all padding
        keys = np.sort(keys, axis=-1)
        lens = rng.integers(0, P + 1, size=(n_lists, batch))
        lens[rng.random((n_lists, batch)) < 0.3] = P
        if n_lists > 1:
            lens[n_lists // 2, :] = 0
        lens[:, -1] = 0
        keys = np.where(np.arange(P).reshape(1, 1, P) < lens[..., None], keys, PAD)
    return np.ascontiguousarray(keys, np.uint64)


def _merge_ref(keys, P):
    n_lists, batch, _ = keys.shape
    flat = keys.transpose(1, 0, 2).reshape(batch, -1)
    out = np.full((batch, P), PAD, np.uint64)
    for b in range(batch):
        s = np.sort(flat[b][flat[b] != PAD])[:P]
        out[b, : len(s)] = s
    return out


def _run_merge(ctx, keys, P):
    import torch
    n_lists, batch, _ = keys.shape
    d_in = _dev(keys)
    d_out = torch.full((batch, P), 7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    ctx.dev_merge(n_lists, batch, P, d_in.data_ptr(), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("P", [1, 30, 512, 513, 900, 1024])
@pytest.mark.parametrize("order", ["asc", "desc", "random", "same", "dup"])
def test_merge_equals_sorted_union(ctx, P, order):
    """The epoch (pushes between prunes) is 3 up to P = 512 and 2 above; at P = 1024 it exactly fills the 2048-key
    buffer.  A key dropped past the buffer's end would leave a plausible but wrong top-P, so every order that pushes
    many keys per epoch (desc above all) is checked at every list count: 2-8 shards, the 77 groups of the legacy BM25
    path at 10M rows and K1's 264 partial lists."""
    rng = np.random.default_rng(P * 31 + len(order))
    for n_lists in (1, 2, 3, 8, 77, 264):
        batch = 256 if n_lists <= 8 else 1
        keys = _merge_keys(order, n_lists, batch, P, rng)
        got = _run_merge(ctx, keys, P)
        ref = _merge_ref(keys, P)
        bad = np.nonzero((got != ref).any(axis=1))[0]
        assert bad.size == 0, (n_lists, batch, bad[:5].tolist())


def test_merge_widest_grid(ctx):
    """K1's 264 lists for a 256-query batch at P = 1024, keys descending: 528 pushes per thread, a prune every epoch"""
    rng = np.random.default_rng(3)
    keys = _merge_keys("desc", 264, 256, 1024, rng)
    assert np.array_equal(_run_merge(ctx, keys, 1024), _merge_ref(keys, 1024))


# ---------------------------------------------------------------------------------------------------------- fuse
def _bitmap(allowed, n_ords):
    bm = np.zeros((n_ords + 31) // 32 + 1, np.uint32)
    idx = np.asarray(allowed, np.int64)
    np.bitwise_or.at(bm, idx >> 5, np.uint32(1) << (idx & 31).astype(np.uint32))
    return bm


def _allowed(bm, ordn):
    ordn = np.asarray(ordn, np.int64)
    return ((bm[ordn >> 5] >> (ordn & 31).astype(np.uint32)) & 1).astype(bool)


def _fuse_lists(P, overlap, mode, rng, with_inf):
    """one query's dense list (L2^2 ascending) and BM25 list (score descending), both as keys padded to P, plus the
    ordinal range they use.  The query's shape is drawn: full lists, short lists, or an empty BM25 list."""
    n_ords = 4 * P + 64
    shape = rng.integers(0, 4)
    nd = P if shape in (0, 2) else int(rng.integers(1, P + 1))
    nb = 0 if shape == 2 else (P if shape == 0 else int(rng.integers(1, P + 1)))
    pool = rng.permutation(n_ords)
    d_ord = pool[:nd]
    n_shared = min(int(round(overlap * nb)), nd)
    b_ord = np.concatenate([rng.permutation(d_ord)[:n_shared], pool[nd: nd + nb - n_shared]])
    rng.shuffle(b_ord)
    dist = (rng.random(nd) * 4.0).astype(np.float32)              # L2^2 of unit vectors spans [0, 4]
    specials = [2.0, np.finfo(np.float32).max] + ([np.inf] if with_inf else [])
    for s in specials:
        if nd > 4 and rng.random() < 0.5:
            dist[rng.integers(0, nd)] = s
    score = (rng.random(nb) * 20.0).astype(np.float32)
    score[rng.random(nb) < 0.2] = 0.0                              # zero-fill entries at the end of a short match
    dk = np.full(P, PAD, np.uint64)
    bk = np.full(P, PAD, np.uint64)
    dk[:nd] = np.sort(key_asc(dist, d_ord))
    bk[:nb] = np.sort(key_desc(score, b_ord))
    return dk, bk, n_ords


def _run_fuse(ctx, dk, bk, P, k, vw, tw, mode, allow):
    import torch
    B = dk.shape[0]
    d_dk = _dev(dk)
    d_bk = None if bk is None else _dev(bk)
    d_al = None if allow is None else _dev(allow)
    out = {"final": torch.full((B, k), 5.0, dtype=torch.float64, device="cuda"),
           "dense": torch.full((B, k), 5.0, dtype=torch.float32, device="cuda"),
           "sparse": torch.full((B, k), 5.0, dtype=torch.float32, device="cuda"),
           "rank": torch.full((B, k), 5, dtype=torch.int32, device="cuda"),
           "ordinal": torch.full((B, k), 5, dtype=torch.int64, device="cuda"),
           "count": torch.full((B,), 5, dtype=torch.int32, device="cuda")}
    torch.cuda.synchronize()
    ctx.dev_fuse(B, P, k, d_dk.data_ptr(), None if d_bk is None else d_bk.data_ptr(), vw, tw, mode,
                 None if d_al is None else d_al.data_ptr(), out["final"].data_ptr(), out["dense"].data_ptr(),
                 out["sparse"].data_ptr(), out["rank"].data_ptr(), out["ordinal"].data_ptr(), out["count"].data_ptr(),
                 torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return {n: t.cpu().numpy() for n, t in out.items()}


def _check_row(got, b, k, ref, what):
    fin, de, sp, rk, od = ref
    c = len(od)
    assert int(got["count"][b]) == c, what
    assert np.array_equal(got["ordinal"][b, :c], od), what
    assert np.array_equal(got["final"][b, :c].view(np.uint64), fin.view(np.uint64)), what
    assert np.array_equal(got["dense"][b, :c], de, equal_nan=True), what
    assert np.array_equal(got["sparse"][b, :c], sp, equal_nan=True), what
    assert np.array_equal(got["rank"][b, :c], rk), what
    # the padded tail: final 0.0, NaN dense and sparse, rank -1, ordinal -1
    assert np.array_equal(got["final"][b, c:].view(np.uint64), np.zeros(k - c, np.uint64)), what
    assert np.isnan(got["dense"][b, c:]).all() and np.isnan(got["sparse"][b, c:]).all(), what
    assert (got["rank"][b, c:] == -1).all() and (got["ordinal"][b, c:] == -1).all(), what


def _fuse_refs(oracle, dk_row, bk_row, k, vw, tw, mode, allow):
    dv = dk_row != PAD
    dd, do = val_asc(dk_row[dv]), (dk_row[dv] & M32).astype(np.int64)
    bv = bk_row != PAD
    bs, bo = val_desc(bk_row[bv]), (bk_row[bv] & M32).astype(np.int64)
    if allow is not None:                         # the keyword-side post-filter drops entries before ranking
        keep = _allowed(allow, bo)
        bs, bo = bs[keep], bo[keep]
    ref = oracle.fuse(dd, do, bs, bo, k, vw, tw, mode)
    if mode == 0:
        py = oracle.py_fuse(list(zip(do.tolist(), dd.astype(np.float64).tolist())), list(zip(bo.tolist(), bs.tolist())),
                            k, vw, tw)
        assert [i for i, _ in py] == ref[4].tolist()
        assert [f for _, f in py] == ref[0].tolist()
    return ref


WEIGHTS = [(0.7, 0.3), (1.0, 0.0), (0.0, 1.0), (2.0, 5.0)]
ALLOWS = ["none", "3%", "60%", "zero", "outside"]


@pytest.mark.parametrize("P", [1, 3, 30, 900, 1024])
@pytest.mark.parametrize("overlap", [0.0, 0.5, 1.0])
def test_fuse_against_oracle(ctx, oracle, P, overlap):
    """every k (including k above the union: the padded tail), both fusion modes (mode 1 with L2^2 above 2 gives negative
    finals), normalised and unnormalised weights, and the keyword allow bitmap at several selectivities: none, 3 %, 60 %,
    nothing allowed, and only ordinals outside both lists (every BM25 entry dropped, dense entries keep rank -1).
    At P = 1024 with overlap 0 the union fills the kernel's 2048 entries."""
    rng = np.random.default_rng(int(P * 10 + overlap * 4))
    B = 6
    for i, (k, mode, (vw, tw)) in enumerate(itertools.product([1, 10, 300, 1024], [0, 1], WEIGHTS)):
        allow_kind = ALLOWS[i % len(ALLOWS)]
        # 0 * inf is NaN: +inf distances only where the vector weight is not zero
        lists = [_fuse_lists(P, overlap, mode, rng, with_inf=vw > 0) for _ in range(B)]
        dk = np.stack([l[0] for l in lists])
        bk = np.stack([l[1] for l in lists])
        if P == 1024 and overlap == 0.0:
            # union of two disjoint full lists: 2048 entries
            dk[0] = np.sort(key_asc((rng.random(P) * 4).astype(np.float32), np.arange(P)))
            bk[0] = np.sort(key_desc((rng.random(P) * 9).astype(np.float32), np.arange(P, 2 * P)))
        n_ords = max(l[2] for l in lists)
        allow = None
        if allow_kind in ("3%", "60%"):
            frac = 0.03 if allow_kind == "3%" else 0.6
            allow = _bitmap(np.nonzero(rng.random(n_ords) < frac)[0], n_ords)
        elif allow_kind == "zero":
            allow = np.zeros((n_ords + 31) // 32 + 1, np.uint32)
        elif allow_kind == "outside":
            used = np.unique(np.concatenate([dk[dk != PAD], bk[bk != PAD]]) & M32).astype(np.int64)
            allow = _bitmap(np.setdiff1d(np.arange(n_ords), used), n_ords)
        got = _run_fuse(ctx, dk, bk, P, k, vw, tw, mode, allow)
        for b in range(B):
            ref = _fuse_refs(oracle, dk[b], bk[b], k, vw, tw, mode, allow)
            _check_row(got, b, k, ref, (k, mode, vw, tw, allow_kind, b))
            if allow_kind == "outside":
                assert (got["rank"][b] == -1).all() and np.isnan(got["sparse"][b]).all()


@pytest.mark.parametrize("mode", [0, 1])
def test_fuse_exact_ties_break_by_ascending_ordinal(ctx, oracle, mode):
    """constructed exact ties on the fp64 final: with w_v = w_t, a dense-only entry whose vector score equals 1/(1 + r)
    ties with the BM25-only entry at rank r.  The tie breaks by ascending ordinal, whichever list the lower one is in."""
    P, k = 16, 32
    B = 2
    dk = np.full((B, P), PAD, np.uint64)
    bk = np.full((B, P), PAD, np.uint64)
    ranks = np.array([0, 1, 3, 7])
    txt = 1.0 / (1.0 + ranks)                                # exact in fp32: powers of two
    vec = txt if mode == 0 else 2.0 - 2.0 * txt              # mode 1: 1 - L2^2 / 2 == txt exactly
    for b in range(B):
        b_ord = np.arange(100, 100 + P)                       # BM25-only ordinals 100..115
        # batch entry 0: the dense twins have LOWER ordinals than their BM25 partners; entry 1: HIGHER
        d_twin = (ranks + 10) if b == 0 else (ranks + 200)
        d_other = np.arange(300, 300 + P - len(ranks))
        d_val = np.concatenate([vec, np.full(len(d_other), 3.5 if mode == 0 else 3.9)]).astype(np.float32)
        dk[b] = np.sort(key_asc(d_val, np.concatenate([d_twin, d_other])))
        bk[b] = np.sort(key_desc(np.linspace(9.0, 1.0, P).astype(np.float32), b_ord))
    got = _run_fuse(ctx, dk, bk, P, k, 1.0, 1.0, mode, None)
    for b in range(B):
        ref = _fuse_refs(oracle, dk[b], bk[b], k, 1.0, 1.0, mode, None)
        _check_row(got, b, k, ref, b)
        fin, od = got["final"][b], got["ordinal"][b]
        for r in ranks:
            i = int(np.nonzero(od == 100 + r)[0][0])
            twin = (r + 10) if b == 0 else (r + 200)
            j = int(np.nonzero(od == twin)[0][0])
            assert fin[i] == fin[j] and (j < i) == (twin < 100 + r), (b, r)
    # weights (1, 0): every BM25-only entry ties at 0.0, ascending ordinal
    got = _run_fuse(ctx, dk, bk, P, 2 * P, 1.0, 0.0, mode, None)
    for b in range(B):
        _check_row(got, b, 2 * P, _fuse_refs(oracle, dk[b], bk[b], 2 * P, 1.0, 0.0, mode, None), b)


@pytest.mark.parametrize("P,k", [(1, 1), (1, 1024), (30, 300), (900, 1024), (1024, 1024)])
def test_dense_only_fuse(ctx, P, k):
    """vector-only fallback (null BM25 list): the first k dense entries, final = the fp32 distance widened; with k > P
    or a short list the tail is padded"""
    rng = np.random.default_rng(P + k)
    B = 4
    dk = np.full((B, P), PAD, np.uint64)
    lens = [P, max(P // 2, 1), 0, P]
    for b in range(B):
        n = lens[b]
        dk[b, :n] = np.sort(key_asc((rng.random(n) * 4).astype(np.float32), rng.permutation(10 * P)[:n]))
    got = _run_fuse(ctx, dk, None, P, k, 0.7, 0.3, 0, None)
    for b in range(B):
        c = min(lens[b], k)
        v = val_asc(dk[b, :c])
        ref = (v.astype(np.float64), v, np.full(c, np.nan, np.float32), np.full(c, -1, np.int32),
               (dk[b, :c] & M32).astype(np.int64))
        _check_row(got, b, k, ref, b)
