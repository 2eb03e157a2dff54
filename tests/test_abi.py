"""CPU-side checks of the C ABI: the in-tree library loads, exports every symbol include/b200asr.h declares, the ctypes
prototypes agree with the header's parameter counts, and entry points fail with an error code (never crash, never
compute on the CPU) when no H100 is present."""
import ctypes
import re

import pytest
import torch

import b200asr

L = b200asr._lib


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    import os
    if not os.path.exists(L.LIB_PATH):
        __graft_entry__.build()
    return L.load()


def test_every_header_symbol_is_exported_and_bound(lib):
    names = L.header_symbols()
    assert len(names) >= 38
    for n in names:
        assert hasattr(lib, n), n
    assert set(names) == set(L.SIGNATURES)


def test_prototypes_match_header_parameter_counts(lib):
    text = open(L.HEADER_PATH).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    for name, (_, argtypes) in L.SIGNATURES.items():
        m = re.search(r"\b%s\s*\(([^;]*?)\)\s*;" % name, text, flags=re.S)
        assert m, name
        params = m.group(1).strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(argtypes), (name, n, len(argtypes))


def test_version_and_error_string(lib):
    assert lib.b200asr_version() >= 100
    assert isinstance(L.last_error(), str)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_gpu_means_error_not_fallback(lib):
    assert lib.b200asr_device_check() == -3                      # B200ASR_UNSUPPORTED_ARCH
    assert "CUDA" in L.last_error() or "device" in L.last_error()
    with pytest.raises(RuntimeError):
        L.load(check_device=True)
    # argument validation happens before any launch: bad shapes are rejected with a message
    assert lib.b200asr_add_ln_fwd(None, None, None, None, None, 0, None, None, None, None, None, 4, 6, 1e-5, 0.0, 0, 0, None) == -5
    assert lib.b200asr_ce_fwd(None, None, None, None, 1, 8, 0.0, None) == -5


def test_missing_library_is_a_loud_error(monkeypatch):
    monkeypatch.setattr(L, "_lib", None)
    monkeypatch.setattr(L, "LIB_PATH", "/nonexistent/libb200asr.so")
    with pytest.raises(RuntimeError, match="no CPU or PyTorch fallback"):
        L.load()
