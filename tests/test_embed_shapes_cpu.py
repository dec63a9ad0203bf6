"""The case table of tests/test_gpu_embed_shapes.py stays inside the shapes K5 accepts and keeps covering them: every mean
pooling width G = 1 ... 8, both head dims at several widths, position tables past 512 and each attention variant."""
from kaito_b200.embedding import check_bert_config
from tests.test_gpu_embed_shapes import CASES, STRESSED, batch_lengths


def test_every_case_is_accepted():
    for name, cfg in CASES.items():
        assert check_bert_config(f"{name}/config.json", dict(cfg, model_type="bert")) == cfg["hidden_size"]
    assert set(STRESSED) <= set(CASES)


def test_every_mean_pool_width():
    assert sorted({c["hidden_size"] // 128 for c in CASES.values()}) == list(range(1, 9))


def test_both_head_dims_at_four_widths():
    for dh in (32, 64):
        widths = {c["hidden_size"] for c in CASES.values() if c["hidden_size"] // c["num_attention_heads"] == dh}
        assert len(widths) >= 4, (dh, widths)


def test_positions_past_512():
    longest = {name: max(max(lens) for lens in batch_lengths(c).values()) for name, c in CASES.items()}
    assert max(longest.values()) > 512
    for name, c in CASES.items():
        assert longest[name] == c["max_position_embeddings"], name      # each case runs up to its position table's end


def test_every_attention_variant():
    """each case runs a batch of max_len <= 32 (one 32-key block), one in (32, 64] (one 64-key block) and one above 64
    (double-buffered 64-key blocks)"""
    for name, c in CASES.items():
        max_lens = [max(lens) for lens in batch_lengths(c).values()]
        assert any(m <= 32 for m in max_lens) and any(32 < m <= 64 for m in max_lens) and any(m > 64 for m in max_lens), name
