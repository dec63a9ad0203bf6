"""CPU checks of host-resident rows (KRAG_ROWS_HOST): HostArray (kaito_b200/csrc/engine.h) is the only owner of pinned host
memory, and KRAG_ROW_STORAGE, which the service and its shard workers read, accepts `device` and `host` only."""
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kaito_b200", "csrc")


def test_only_hostarray_allocates_and_frees_pinned_memory():
    """a cudaHostAlloc / cudaMallocHost / cudaHostRegister / cudaFreeHost anywhere else is pinned memory without an owner
    (and without a place in krag_host_pinned_bytes)"""
    pinned = re.compile(r"\bcuda(HostAlloc|MallocHost|HostRegister|HostUnregister|FreeHost)\b")
    engine = open(os.path.join(CSRC, "engine.h")).read()
    start = engine.index("struct HostArray {")
    depth, end = 0, start
    for end in range(start, len(engine)):
        depth += {"{": 1, "}": -1}.get(engine[end], 0)
        if depth == 0 and engine[end] == "}":
            break
    body = engine[start:end]
    assert re.search(r"\bcudaHostAlloc\b", body) and re.search(r"\bcudaFreeHost\b", body), "HostArray no longer allocates"
    assert "cudaHostGetDevicePointer" in body, "the mapped address must come from cudaHostGetDevicePointer"
    found = []
    for path in sorted(glob.glob(os.path.join(CSRC, "*"))):
        if not path.endswith((".cu", ".cuh", ".h", ".cpp")):
            continue
        txt = open(path).read()
        for m in pinned.finditer(txt):
            if not (path.endswith("engine.h") and start < m.start() < end):
                found.append(f"{os.path.basename(path)}:{txt.count(chr(10), 0, m.start()) + 1}")
    assert not found, found


def test_row_storage_from_env():
    from kaito_b200 import _native
    assert _native.row_storage_from_env({}) == _native.ROWS_DEVICE
    assert _native.row_storage_from_env({"KRAG_ROW_STORAGE": "device"}) == _native.ROWS_DEVICE
    assert _native.row_storage_from_env({"KRAG_ROW_STORAGE": "host"}) == _native.ROWS_HOST
    assert _native.row_storage_from_env({"KRAG_ROW_STORAGE": " Host "}) == _native.ROWS_HOST
    for junk in ("", "1", "hbm", "pinned", "host,device"):
        with pytest.raises(ValueError):
            _native.row_storage_from_env({"KRAG_ROW_STORAGE": junk})


def test_config_layout_is_unchanged():
    """row_storage takes the first reserved word: the struct keeps its size and the fields before it their offsets"""
    import ctypes as C
    from kaito_b200 import _native
    assert C.sizeof(_native.Config) == 32
    assert _native.Config.row_storage.offset == 20 and _native.Config.reserved.offset == 24
