"""The split-row encoding of device-resident fp32 rows (kaito_b200/csrc/split_rows.cuh), restated in numpy: a value's bits x
become hi = bf16 of x rounded to nearest with ties toward zero and lo = the low 16 bits, and x is rebuilt from them bit for
bit.  Checked exhaustively over all 65,536 low halves for a spread of high halves, and the row layout of 256-byte blocks
whose halves hold their elements in K1's lane order."""
import numpy as np

SPLIT_BLOCK = 64
# element held at each position of a half-block: position 8 l + 4 h + c holds element 32 h + 4 l + c
SPLIT_ELEM = np.array([32 * ((p >> 2) & 1) + 4 * (p >> 3) + (p & 3) for p in range(SPLIT_BLOCK)])


def split_hi(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.uint32)
    return (((x >> 16) + ((x & 0xFFFF) > 0x8000)) & 0xFFFF).astype(np.uint32)


def split_join(hi: np.ndarray, lo: np.ndarray) -> np.ndarray:
    hi, lo = hi.astype(np.uint32), lo.astype(np.uint32)
    return (((hi - (lo > 0x8000).astype(np.uint32)) << 16) | lo).astype(np.uint32)


def bf16_rne(x: np.ndarray) -> np.ndarray:
    """bf16 bits of finite fp32 bits x, round to nearest even (what __float2bfloat16_rn gives)"""
    x = x.astype(np.uint64)
    return (((x + 0x7FFF + ((x >> 16) & 1)) >> 16) & 0xFFFF).astype(np.uint32)


def encode_rows(x: np.ndarray) -> np.ndarray:
    """[n, dpad] fp32 -> [n, dpad] u32 words of the split layout: per 64-element block, 64 high halves then 64 low halves,
    each in lane order"""
    b = np.ascontiguousarray(x).view(np.uint32).reshape(x.shape[0], -1, SPLIT_BLOCK)[:, :, SPLIT_ELEM]
    halves = np.concatenate([split_hi(b), b & 0xFFFF], axis=2).astype(np.uint16)
    return np.ascontiguousarray(halves.reshape(x.shape[0], -1)).view(np.uint32)


def decode_rows(w: np.ndarray) -> np.ndarray:
    h = w.view(np.uint16).reshape(w.shape[0], -1, 2 * SPLIT_BLOCK)
    b = np.empty(h.shape[:2] + (SPLIT_BLOCK,), np.uint32)
    b[:, :, SPLIT_ELEM] = split_join(h[:, :, :SPLIT_BLOCK], h[:, :, SPLIT_BLOCK:])
    return np.ascontiguousarray(b.reshape(w.shape[0], -1)).view(np.float32)


HIGHS = [0x0000, 0x0001, 0x007F, 0x0080, 0x0081, 0x3F7F, 0x3F80, 0x3F81, 0x4049, 0x7F7E, 0x7F7F,
         0x8000, 0x8001, 0x807F, 0x8080, 0xBF7F, 0xBF80, 0xC2F7, 0xFF7E, 0xFF7F]


def _all_lows(high: int) -> np.ndarray:
    return (np.uint32(high) << np.uint32(16)) | np.arange(1 << 16, dtype=np.uint32)


def test_round_trip_is_exact_for_every_low_half():
    for high in HIGHS + [0x7F80, 0x7FC0, 0xFF80, 0xFFFF]:     # the last four: infinities and NaN patterns also round-trip
        x = _all_lows(high)
        assert np.array_equal(split_join(split_hi(x), x & 0xFFFF), x), hex(high)


def test_high_half_is_bf16_rounded_to_nearest_ties_toward_zero():
    for high in HIGHS:
        x = _all_lows(high)
        hi, rne = split_hi(x), bf16_rne(x)
        tie = (x & 0xFFFF) == 0x8000
        assert np.array_equal(hi[~tie], rne[~tie]), hex(high)
        assert np.array_equal(hi[tie], x[tie] >> 16), hex(high)                      # ties keep the smaller magnitude
        # at most half a bf16 ulp from x: the K2 certificate's bf16 operand bound holds unchanged
        xf = x.view(np.float32).astype(np.float64)
        hf = (hi << 16).astype(np.uint32).view(np.float32).astype(np.float64)
        ulp = np.abs((((x >> 16) + 1) << 16).astype(np.uint32).view(np.float32).astype(np.float64) -
                     ((x >> 16) << 16).astype(np.uint32).view(np.float32).astype(np.float64))
        finite = np.isfinite(hf)
        assert (np.abs(hf - xf)[finite] <= 0.5 * ulp[finite]).all(), hex(high)


def test_rounding_carries_into_the_exponent():
    x = np.array([0x3F7F8001, 0x007F8001, 0xBF7FFFFF, 0x7F7F8001, 0x7F7F8000], np.uint32)
    assert split_hi(x).tolist() == [0x3F80, 0x0080, 0xBF80, 0x7F80, 0x7F7F]        # 0x7F80: bf16 infinity
    assert np.array_equal(split_join(split_hi(x), x & 0xFFFF), x)


def test_row_layout_round_trips_and_streams_the_high_halves():
    rng = np.random.default_rng(7)
    bits = rng.integers(0, 1 << 32, size=(5, 192), dtype=np.uint64).astype(np.uint32)
    bits[(bits >> 23 & 0xFF) == 0xFF] &= 0xBFFFFFFF                                  # finite values only
    x = bits.view(np.float32)
    w = encode_rows(x)
    assert w.shape == x.shape and w.dtype == np.uint32                                # same bytes per row
    assert np.array_equal(decode_rows(w).view(np.uint32), bits)
    h = w.view(np.uint16).reshape(5, 3, 2 * SPLIT_BLOCK)
    blk = bits.reshape(5, 3, SPLIT_BLOCK)
    assert np.array_equal(h[:, :, :SPLIT_BLOCK], split_hi(blk)[:, :, SPLIT_ELEM])    # block b: 128 B of high halves first
    assert np.array_equal(h[:, :, SPLIT_BLOCK:], (blk & 0xFFFF)[:, :, SPLIT_ELEM])
    # K1's lane l reads 16 bytes at 16 l of each half: the elements it sums at steps 2 b and 2 b + 1
    for lane in range(8):
        assert SPLIT_ELEM[8 * lane:8 * lane + 8].tolist() == [4 * lane + c for c in range(4)] + [32 + 4 * lane + c for c in range(4)]
    assert sorted(SPLIT_ELEM.tolist()) == list(range(SPLIT_BLOCK))
