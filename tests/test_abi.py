"""CPU tests of the drop-in boundary: libkaito_rag.so loads here (no GPU) and exports every
symbol include/kaito_rag.h declares; without a device krag_init fails loudly (no fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "kaito_rag.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(krag_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    from kaito_b200 import _native
    assert sorted(_native.SYMBOLS) == _declared_symbols()


def test_library_exports_every_declared_symbol():
    from kaito_b200 import _native
    L = _native.load()
    for name in _declared_symbols():
        assert getattr(L, name) is not None, name
    assert L.krag_version() >= 100


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: the no-device error path cannot be exercised")
    from kaito_b200 import _native
    with pytest.raises(_native.KragError) as e:
        _native.Context(device_id=0)
    assert e.value.code == _native.KRAG_E_NO_DEVICE


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "kaito_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
                assert "libkrag_oracle" not in txt and not re.search(r'#include\s*"[^"]*oracle', txt), f


def test_every_env_variable_the_library_reads_is_documented():
    """each KRAG_* variable the native library reads is a supported setting, listed in INTEGRATION.md's variable table"""
    read = set()
    csrc = os.path.join(ROOT, "kaito_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        if not f.endswith((".cu", ".cuh", ".h", ".cpp")):
            continue
        txt = open(os.path.join(csrc, f)).read()
        read |= set(re.findall(r'\b(?:getenv|env_int)\(\s*"(KRAG_[A-Z0-9_]+)"', txt))
    assert read, "no getenv(\"KRAG_...\") found: the pattern no longer matches the sources"
    lines = open(os.path.join(ROOT, "INTEGRATION.md")).read().splitlines()
    start = lines.index("| variable | default | effect |")
    table = []
    for line in lines[start + 2:]:
        if not line.startswith("|"):
            break
        table.append(line.split("|")[1])
    documented = set(re.findall(r"`(KRAG_[A-Z0-9_]+)`", "\n".join(table)))
    assert sorted(read - documented) == []


def test_header_is_plain_c99_and_links(tmp_path):
    """include/kaito_rag.h is consumed by cgo: it must compile as C99 (no C++-isms, no torch/CUDA types) and a C program
    calling an entry point must link against libkaito_rag.so (no compute call: there is no GPU here)."""
    import shutil
    import subprocess
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "abi.c"
    src.write_text('#include "kaito_rag.h"\n#include <stdio.h>\n'
                   'int main(void) { krag_config c; krag_stats_t s; (void)c; (void)s;\n'
                   '  printf("%lld %s\\n", (long long)krag_tc_fallback_queries(), KRAG_KEY_PAD == 0xFFFFFFFFFFFFFFFFull ? "pad" : "?");\n'
                   '  return 0; }\n')
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"), "-fsyntax-only", str(src)],
                   check=True)
    exe = tmp_path / "abi"
    lib_dir = os.path.join(root, "kaito_b200")
    subprocess.run([gcc, "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe), "-L", lib_dir, "-lkaito_rag",
                    "-Wl,-rpath," + lib_dir], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert out.strip() == "0 pad"


def test_c_example_builds_and_fails_loudly_without_a_gpu(tmp_path):
    """examples/krag_demo.c (the cgo-equivalent call sequence in plain C) compiles as pedantic C99 and links; on a machine
    without an sm_90 GPU it stops at krag_init with KRAG_E_NO_DEVICE -- there is no CPU path to fall back to."""
    import shutil
    import subprocess
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    lib_dir = os.path.join(ROOT, "kaito_b200")
    exe = tmp_path / "krag_demo"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "krag_demo.c"), "-o", str(exe), "-L", lib_dir, "-lkaito_rag", "-Wl,-rpath," + lib_dir, "-lm"],
                   check=True)
    import torch
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 0 and r.stdout.count("\n") == 3 and r.stdout.startswith("#0 node ")
    else:
        assert r.returncode == 1 and "-> -2" in r.stderr and "no CPU fallback" in r.stderr
