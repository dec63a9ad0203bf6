"""CPU tests of the reranker's precision switch: KRAG_RERANK_PRECISION parsing and the start-up refusal, the `precision`
argument of GpuCrossEncoder reaching krag_embedder_set_precision (a recording stand-in for the native embedder), and the
header's declarations agreeing with the ctypes signatures."""
import os
import re

import numpy as np
import pytest

from kaito_b200 import _native, rerank
from tests import st_snapshot as sts
from tests.test_rerank_cpu import MINILM_CE, TOKENIZER_CONFIG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("value,want", [(None, "fp32"), ("", "fp32"), ("fp32", "fp32"), ("fp16", "fp16")])
def test_precision_from_env(monkeypatch, value, want):
    if value is None:
        monkeypatch.delenv("KRAG_RERANK_PRECISION", raising=False)
    else:
        monkeypatch.setenv("KRAG_RERANK_PRECISION", value)
    assert rerank.precision_from_env() == want


@pytest.mark.parametrize("value", ["bf16", "FP16", "half", "1"])
def test_unknown_precision_is_refused(monkeypatch, value):
    monkeypatch.setenv("KRAG_RERANK_PRECISION", value)
    with pytest.raises(ValueError, match="KRAG_RERANK_PRECISION"):
        rerank.precision_from_env()


def test_service_exits_on_an_unknown_precision_before_any_gpu_work(tmp_path, monkeypatch):
    import sys
    from kaito_b200 import service
    monkeypatch.setattr(sys, "setswitchinterval", lambda s: None)

    def no_gpu(*a, **k):
        raise AssertionError("the service reached the GPU")
    monkeypatch.setattr(_native, "Context", no_gpu)
    monkeypatch.delenv("KRAG_MODEL_DIR", raising=False)
    monkeypatch.setenv("EMBEDDING_SOURCE_TYPE", "local")
    monkeypatch.setenv("VECTOR_DB_TYPE", "faiss")
    monkeypatch.setenv("KRAG_RERANK_MODEL_DIR", sts.write(tmp_path, {"config.json": MINILM_CE, "tokenizer_config.json": TOKENIZER_CONFIG}))
    monkeypatch.setenv("KRAG_RERANK_PRECISION", "bf16")
    with pytest.raises(SystemExit, match=r"reranker '.*' is not supported by this image: KRAG_RERANK_PRECISION 'bf16'"):
        service.main()


class RecordingEmbedder:
    """the calls GpuCrossEncoder makes on _native.Embedder"""
    made = []

    def __init__(self, *a):
        self.calls = []
        RecordingEmbedder.made.append(self)

    def load_state_dict(self, state, head=False):
        self.calls.append(("load", head))

    def set_precision(self, precision):
        self.calls.append(("precision", precision))


@pytest.mark.parametrize("kw,want", [({}, "fp32"), ({"precision": "fp32"}, "fp32"), ({"precision": "fp16"}, "fp16")])
def test_precision_reaches_the_embedder(tmp_path, monkeypatch, kw, want):
    monkeypatch.setattr(_native, "Embedder", RecordingEmbedder)
    d = 384
    state = {"bert.pooler.dense.weight": np.zeros((d, d), np.float32), "bert.pooler.dense.bias": np.zeros(d, np.float32),
             "classifier.weight": np.zeros((1, d), np.float32), "classifier.bias": np.zeros(1, np.float32)}
    snap = sts.write(tmp_path, {"config.json": MINILM_CE, "tokenizer_config.json": TOKENIZER_CONFIG}, state=state)
    ce = rerank.GpuCrossEncoder.from_pretrained(None, snap, **kw)
    assert ce.precision == want
    assert RecordingEmbedder.made[-1].calls == [("load", True), ("precision", want)]
    with pytest.raises(ValueError, match="precision 'bf16'"):
        rerank.GpuCrossEncoder.from_pretrained(None, snap, precision="bf16")


def test_embedder_set_precision_refuses_unknown_names_before_the_library():
    e = _native.Embedder.__new__(_native.Embedder)       # no handle: the name is checked first
    with pytest.raises(ValueError, match="'fp32' or 'fp16'"):
        e.set_precision("bf16")


def test_header_declares_what_ctypes_binds():
    header = open(os.path.join(ROOT, "include", "kaito_rag.h")).read()
    flat = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", " ", header, flags=re.S))
    assert re.search(r"#define KRAG_PRECISION_FP32 0\b", header) and re.search(r"#define KRAG_PRECISION_FP16 1\b", header)
    assert _native.PRECISIONS == {"fp32": 0, "fp16": 1}
    assert "int32_t krag_embedder_set_precision(krag_embedder* e, int32_t mode);" in flat
    args = lambda name: re.search(name + r"\((.*?)\);", flat).group(1)
    strip = lambda s: re.sub(r"\s+", " ", s).strip()
    assert strip(args("krag_debug_gemm_f16")) == strip(args("krag_debug_gemm_tf32"))        # "same argument list"
    assert {"krag_embedder_set_precision", "krag_debug_gemm_f16"} <= set(_native.SYMBOLS)
    lib = os.path.join(ROOT, "kaito_b200", "libkaito_rag.so")
    if os.path.exists(lib):
        L = _native.load()
        assert L.krag_debug_gemm_f16.argtypes == L.krag_debug_gemm_tf32.argtypes
        assert len(L.krag_embedder_set_precision.argtypes) == 2
