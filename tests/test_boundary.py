"""The drop-in boundary: the C-ABI library loads (no GPU needed), exports every symbol that
include/torchrl_b200.h declares, the binding takes its types from that header and checks operands against it, and
the product package never imports the oracle."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "torchrl_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(trl_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(native_lib):
    from torchrl_b200 import _lib
    declared = _declared_symbols()
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(native_lib, name), "header declares %s but the library does not export it" % name
    # and the python binding types exactly the declared set
    assert sorted(_lib.SIGNATURES) == declared


def test_definitions_match_declarations():
    """Every TRL_API definition in csrc/ is declared in the header and the other way round (the compiler checks
    their types: every kernel source includes the header)."""
    csrc = os.path.join(ROOT, "torchrl_b200", "csrc")
    defined = set()
    for fn in os.listdir(csrc):
        if fn.endswith((".cu", ".cuh")):
            src = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(os.path.join(csrc, fn)).read(), flags=re.S)
            defined |= set(re.findall(r"\bTRL_API\s[\w\s*]*?\b(trl_[a-z0-9_]+)\s*\(", src))
    assert sorted(defined) == _declared_symbols()


def test_header_parse_errors(tmp_path):
    """A missing header or a type the binding does not map fails loudly, naming the declaration."""
    from torchrl_b200 import _lib
    with pytest.raises(_lib.NativeLibraryError):
        _lib.parse_header(str(tmp_path / "missing.h"))
    h = tmp_path / "bad.h"
    h.write_text("int trl_ok(const float* x, int64_t n, void* stream);\nint trl_bad(const short* x, int n);\n")
    with pytest.raises(_lib.NativeLibraryError, match="trl_bad"):
        _lib.parse_header(str(h))


def test_call_checks_argument_count(native_lib):
    """Too many or too few arguments raise before the library is called (ctypes alone passes extra ones through)."""
    from torchrl_b200 import _lib
    args = [None] * 7 + [4, 4, 0.99, 0.95, 1, 1, None]
    before = _lib.launch_count()
    with pytest.raises(TypeError, match="takes 14 arguments, got 15"):
        _lib.call("trl_gae_scan", *args, 7)
    with pytest.raises(TypeError, match="takes 14 arguments, got 13"):
        _lib.call("trl_gae_scan", *args[:-1])
    assert _lib.launch_count() == before


def test_call_rejects_cpu_tensors(native_lib):
    """A CPU tensor for a typed pointer parameter raises ValueError naming the header's parameter; nothing reaches
    the library (which would reject the NULL operands with RuntimeError)."""
    import torch

    from torchrl_b200 import _lib
    x = torch.zeros(16)
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="trl_gae_scan: values must be a CUDA tensor"):
        _lib.call("trl_gae_scan", None, x, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, 1, None)
    with pytest.raises(ValueError, match="trl_skinny_reduce_jobs: scratch must be a CUDA tensor"):
        _lib.call("trl_skinny_reduce_jobs", 1, None, [x], [None], [None], None, None, None, None, None)
    with pytest.raises(RuntimeError, match="trl_gae_scan failed"):
        _lib.call("trl_gae_scan", None, None, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, 1, None)
    assert _lib.launch_count() == before


def test_abi_version_and_error_string(native_lib):
    assert native_lib.trl_abi_version() == 3
    assert native_lib.trl_last_error() is not None


def test_argument_errors_without_gpu(native_lib):
    """Argument validation happens before any CUDA call, so it is testable on CPU."""
    rc = native_lib.trl_gae_scan(None, None, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, 1, None)
    assert rc == -1
    assert b"null" in native_lib.trl_last_error()
    rc = native_lib.trl_gae_scan(None, None, None, None, None, None, None, -1, 4, 0.99, 0.95, 1, 1, None)
    assert rc == -1
    rc = native_lib.trl_gae_scan(None, None, None, None, None, None, None, 0, 4, 0.99, 0.95, 1, 1, None)
    assert rc == 0  # empty rollout is a no-op


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "torchrl_b200")
    pat = re.compile(r"^\s*(from|import)\s+oracle\b", re.M)
    for dp, _, fns in os.walk(pkg):
        for fn in fns:
            if fn.endswith(".py"):
                txt = open(os.path.join(dp, fn)).read()
                assert not pat.search(txt), "%s imports the oracle" % os.path.join(dp, fn)
                assert "/root/reference" not in txt.replace("/root/reference/torchrl", "REFDOC"), fn


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from torchrl_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    monkeypatch.setenv("TORCHRL_B200_NO_AUTOBUILD", "1")
    import pytest
    with pytest.raises(_lib.NativeLibraryError):
        _lib.load()


def test_deferred_reduce_scope_is_strict():
    """networks.fused.deferred_reduces(): pending slab-sum jobs must be flushed inside the scope (a silent drop would
    lose gradients); an empty flush is a no-op and the scope restores the previous state.  Host logic only."""
    from torchrl_b200.networks import fused
    assert fused._DEFER is None
    with fused.deferred_reduces():
        assert fused._DEFER == []
        fused.flush_reduces()                      # nothing recorded: no library call
        with fused.deferred_reduces():             # nested scopes keep their own job lists
            assert fused._DEFER == []
        assert fused._DEFER == []
    assert fused._DEFER is None
    with pytest.raises(RuntimeError):
        with fused.deferred_reduces():
            fused._DEFER.append((0, None, None, None, 1, 32, 1, 0))
    assert fused._DEFER is None
    assert not fused._can_defer(object())          # outside a scope nothing is deferred
