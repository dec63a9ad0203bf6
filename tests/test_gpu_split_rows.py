"""Device rows stored as split rows (bf16 high halves beside their low halves, kaito_b200/csrc/split_rows.cuh) on the H100:
crafted bit patterns round-trip through add -> read_rows and persist -> load; the default K2 prune pass streams the high
halves (kernel id 5, 2 bytes per element) and returns the oracle's results, as do the bf16-shadow and TF32 passes, K1,
compaction and a two-shard redeal; indexes with dpad % 64 == 32 keep plain rows and the TF32 pass."""
import numpy as np
import pytest

from tests.test_gpu_sharded_compact import RR, LoopbackA2A, check_layout
from tests.test_split_rows_cpu import encode_rows

pytestmark = pytest.mark.gpu


@pytest.fixture
def loopback(monkeypatch):
    from kaito_b200 import sharded
    monkeypatch.setattr(sharded, "dist", LoopbackA2A)
    monkeypatch.setenv("KRAG_P2P", "0")
    return sharded


def _crafted(n, d, seed):
    """rows of edge patterns: +-0, subnormals, lo = 0x7FFF / 0x8000 / 0x8001 / 0xFFFF, rounding that carries into the
    exponent, values whose high half is bf16 infinity; then random finite bits"""
    highs = np.array([0x0000, 0x0001, 0x007F, 0x0080, 0x3F7F, 0x3F80, 0x7F7E, 0x7F7F], np.uint32)
    lows = np.array([0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF], np.uint32)
    pat = ((highs[:, None] << 16) | lows[None, :]).ravel()
    pat = np.concatenate([pat, pat | 0x80000000])
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 1 << 32, size=n * d, dtype=np.uint64).astype(np.uint32)
    bits[(bits >> 23 & 0xFF) == 0xFF] &= 0xBFFFFFFF
    bits[:len(pat) * 3] = np.tile(pat, 3)
    bits[len(pat) * 3:len(pat) * 6] = np.roll(np.tile(pat, 3), 17)
    return bits.reshape(n, d).view(np.float32)


@pytest.mark.parametrize("d", [64, 128, 200, 768])
def test_crafted_rows_round_trip_bitwise(tmp_path, d):
    from kaito_b200 import _native
    n = 3000
    x = _crafted(n, d, d)
    c = _native.Context(device_id=0)
    try:
        ix = c.create_index(f"rt_{d}", d)
        ix.add(np.arange(1000, dtype=np.uint64), x[:1000])
        ix.add(np.arange(1000, n, dtype=np.uint64), x[1000:])
        assert np.array_equal(ix.read_rows(0, n).view(np.uint32), x.view(np.uint32))
        assert np.array_equal(ix.read_rows(1234, 77).view(np.uint32), x[1234:1311].view(np.uint32))
        dpad = ix.stats().dim_padded
        xp = np.pad(x, ((0, 0), (0, dpad - d)))
        stored = ix.debug_stored_rows(0, n)                                     # the bytes on the device
        assert np.array_equal(stored, encode_rows(xp) if dpad % 64 == 0 else xp.view(np.uint32))
        ix.persist(str(tmp_path))
        ix.drop()
        ix = c.load_index(f"rt_{d}_loaded", str(tmp_path))
        assert np.array_equal(ix.read_rows(0, n).view(np.uint32), x.view(np.uint32))
        ix.drop()
    finally:
        c.close()


@pytest.fixture(scope="module")
def wide(oracle):
    n, d = 270_000, 768
    x = oracle.synth_dense(n, d, seed=41)
    q = oracle.synth_queries(x, 256, seed=42)
    return x, q, oracle.dense_topk(x, q, 30)


def test_default_pass_reads_high_halves(wide):
    """AUTO at d = 768, batch 256: kernel id 5 over n * dpad * 2 bytes, the oracle's results; the bf16 shadow (id 4) and
    the TF32 pass on split rows (id 3) give the same; K1 at batch 1 too"""
    from kaito_b200 import _native
    x, q, (rd, ro) = wide
    n, d = x.shape
    c = _native.Context(device_id=0)
    try:
        ix = c.create_index("wide", d)
        ix.add(np.arange(n, dtype=np.uint64), x)
        rows_bytes = ix.stats().device_bytes
        assert rows_bytes >= n * d * 4
        fb0 = _native.load().krag_tc_fallback_queries()
        dist, ordn = ix.search_dense(q, 30)
        _, kid, by, _ = _native.last_dense_kernel()
        assert (kid, by) == (5, n * d * 2)
        # the pass pruned on the right bytes: every query certified, none re-run on K1
        assert _native.load().krag_tc_fallback_queries() == fb0
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        d1, o1 = ix.search_dense(q[:1], 30)
        assert _native.last_dense_kernel()[1] == 1 and np.array_equal(o1, ro[:1]) and np.array_equal(d1, rd[:1])
        ix.set_dense_mode(_native.DENSE_TC_TF32)
        d3, o3 = ix.search_dense(q, 30)
        assert _native.last_dense_kernel()[1] == 3 and np.array_equal(o3, ro) and np.array_equal(d3, rd)
        assert _native.load().krag_tc_fallback_queries() == fb0
        ix.set_dense_mode(_native.DENSE_TC_BF16)
        assert ix.stats().device_bytes > rows_bytes                            # the shadow is extra memory
        d4, o4 = ix.search_dense(q, 30)
        assert _native.last_dense_kernel()[1] == 4 and np.array_equal(o4, ro) and np.array_equal(d4, rd)
        assert _native.load().krag_tc_fallback_queries() == fb0
        assert np.array_equal(ix.debug_stored_rows(0, 1000), encode_rows(x[:1000]))   # the shadow build left the rows intact
        ix.set_dense_mode(_native.DENSE_AUTO, release_shadow=True)
        d5, o5 = ix.search_dense(q, 30)
        assert _native.last_dense_kernel()[1] == 5 and np.array_equal(o5, ro) and np.array_equal(d5, rd)
        assert _native.load().krag_tc_fallback_queries() == fb0
        ix.drop()
    finally:
        c.close()


def test_tf32_dump_on_split_rows_equals_plain_rows(oracle):
    """the TF32 tensor-core values of split rows (high and low halves rebuilt in the A registers) equal those of the same
    rows stored plain: d = 64 is split, d = 64 zero-padded to 96 is not, and the padding adds exact zeros"""
    from kaito_b200 import _native
    n = 5000
    x = oracle.synth_dense(n, 64, seed=5)
    q = oracle.synth_queries(x, 100, seed=6)
    c = _native.Context(device_id=0, dense_mode=_native.DENSE_TC_TF32)
    try:
        a = c.create_index("split64", 64)
        b = c.create_index("plain96", 96)
        a.add(np.arange(n, dtype=np.uint64), x)
        b.add(np.arange(n, dtype=np.uint64), np.pad(x, ((0, 0), (0, 32))))
        da = a.debug_tc_dump(q)
        db = b.debug_tc_dump(np.pad(q, ((0, 0), (0, 32))))
        assert np.array_equal(da.view(np.uint32), db.view(np.uint32))
        a.drop(); b.drop()
    finally:
        c.close()


def test_compaction_keeps_results(oracle):
    from kaito_b200 import _native
    n, d = 400_000, 128                                                      # 320k live rows: K2 still serves batch 64
    x = oracle.synth_dense(n, d, seed=11)
    q = oracle.synth_queries(x, 64, seed=12)
    live = np.random.default_rng(13).random(n) >= 0.2
    c = _native.Context(device_id=0)
    try:
        ix = c.create_index("cmp", d)
        ix.add(np.arange(n, dtype=np.uint64), x)
        ix.remove(np.flatnonzero(~live).astype(np.uint64))
        assert ix.compact() == int((~live).sum())
        xl = x[live]
        assert np.array_equal(ix.read_rows(0, len(xl)), xl)
        rd, ro = oracle.dense_topk(xl, q, 30)
        dist, ordn = ix.search_dense(q, 30)
        assert _native.last_dense_kernel()[1] == 5 and np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        d1, o1 = ix.search_dense(q[:3], 30)
        assert np.array_equal(o1, ro[:3]) and np.array_equal(d1, rd[:3])
        ix.drop()
    finally:
        c.close()


def test_two_shard_redeal_moves_split_rows(oracle, loopback):
    from kaito_b200 import _native
    n, d, vocab = 20_000, 128, 3000
    x = oracle.synth_dense(n, d, seed=21)
    csr = oracle.synth_sparse(n, vocab, 22, mean_len=24.0)
    dead = np.random.default_rng(23).random(n) < 0.3
    c = _native.Context(device_id=0)
    try:
        sh = RR(loopback, c, "rd", x, csr, vocab, 2)
        sh.commit()
        sh.remove(np.flatnonzero(dead))
        sh.commit()
        sh.compact()
        live_ords = np.flatnonzero(~dead)
        check_layout(sh, x, live_ords)
        q = oracle.synth_queries(x, 8, seed=24)
        for s, ix in enumerate(sh.ix):
            mine = live_ords[s::2]
            dist, ordn = ix.search_dense(q, 10)
            rd, ro = oracle.dense_topk(x[mine], q, 10)
            assert np.array_equal(dist, rd) and np.array_equal((ordn - s) // 2, ro), s
        sh.drop()
    finally:
        c.close()


def test_dpad_32_mod_64_keeps_plain_rows(oracle):
    from kaito_b200 import _native
    n, d = 270_000, 96
    x = oracle.synth_dense(n, d, seed=31)
    q = oracle.synth_queries(x, 64, seed=32)
    c = _native.Context(device_id=0)
    try:
        ix = c.create_index("d96", d)
        ix.add(np.arange(n, dtype=np.uint64), x)
        dist, ordn = ix.search_dense(q, 30)
        _, kid, by, _ = _native.last_dense_kernel()
        assert (kid, by) == (3, n * d * 4)
        rd, ro = oracle.dense_topk(x, q, 30)
        assert np.array_equal(ordn, ro) and np.array_equal(dist, rd)
        ix.drop()
    finally:
        c.close()
