"""CPU: the C-ABI library loads and exports every symbol include/masr_b200.h declares (no compute
calls — there is no GPU here), and the ctypes table agrees with the header."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "masr_b200.h")


def declared_functions():
    src = open(HEADER, encoding="utf-8").read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.findall(r"\b(?:int|const char\*)\s+(masr_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", src, flags=re.S)


@pytest.fixture(scope="module")
def lib():
    from masr_b200 import build, _lib
    build.build()                      # nvcc cross-compiles sm_90a without a GPU
    return _lib.load()


def test_every_declared_symbol_is_exported(lib):
    decl = declared_functions()
    assert len(decl) >= 13
    for name, _ in decl:
        assert hasattr(lib, name), name


def test_ctypes_table_matches_header(lib):
    from masr_b200 import _lib
    decl = dict(declared_functions())
    for name, argtypes in _lib.SIGNATURES.items():
        assert name in decl, name
        params = [p for p in decl[name].split(",") if p.strip() and p.strip() != "void"]
        assert len(params) == len(argtypes), (name, len(params), len(argtypes))
        for p, t in zip(params, argtypes):
            is_ptr = "*" in p
            if is_ptr:
                assert t in (ctypes.c_void_p,) or hasattr(t, "_type_") and not isinstance(t._type_, str) or t is ctypes.c_void_p, (name, p)
            elif "int64_t" in p:
                assert t is ctypes.c_int64, (name, p)
            elif "float" in p:
                assert t is ctypes.c_float, (name, p)
            else:
                assert t is ctypes.c_int, (name, p)
    missing = set(decl) - set(_lib.SIGNATURES) - {"masr_last_error"}
    assert not missing, missing


def test_abi_version_and_error_string(lib):
    assert lib.masr_abi_version() == 1
    assert isinstance(lib.masr_last_error(), bytes)


def test_library_has_sm90a_sass_only():
    import shutil
    import subprocess
    from masr_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "masr_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), encoding="utf-8").read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_max_len_guard_matches_the_reference_assert():
    """ADVICE r1: utterances whose subsampled length reaches the position table (embedding.py:95-97) fail on the host."""
    import pytest
    from masr_b200.engine import check_max_len, num_frames, subsampled_len
    check_max_len([], 5000)
    check_max_len([0, 4999], 5000)
    check_max_len([123456], 0)                       # DeepSpeech2: no position table
    n = 16000 * 201
    assert subsampled_len(num_frames(n)) >= 5000
    with pytest.raises(AssertionError, match="larger than the max_len: 5000"):
        check_max_len([10, subsampled_len(num_frames(n))], 5000)


def test_unsupported_reference_variants_are_rejected_not_mispacked():
    """ADVICE r1: batch_norm conv modules, conv2d6/8 front-ends, GRU DeepSpeech2 and odd head widths raise a clear error."""
    import numpy as np
    import pytest
    import torch
    from masr_b200.weights import UnsupportedConfig, check_supported
    base = {"encoder.after_norm.weight": torch.zeros(256), "encoder.encoders.0.self_attn.pos_bias_u": torch.zeros(4, 64)}
    check_supported(base)
    with pytest.raises(UnsupportedConfig, match="batch_norm"):
        check_supported({**base, "encoder.encoders.0.conv_module.norm.running_mean": torch.zeros(256)})
    with pytest.raises(UnsupportedConfig, match="conv2d6"):
        check_supported({**base, "encoder.embed.conv.4.weight": torch.zeros(1)})
    with pytest.raises(UnsupportedConfig, match="heads"):
        check_supported({**base, "encoder.encoders.0.self_attn.pos_bias_u": torch.zeros(8, 32)})
    with pytest.raises(UnsupportedConfig, match="use_gru"):
        check_supported({"encoder.rnns.0.rnn.weight_hh_l0": torch.zeros(3 * 16, 16)}, "deepspeech2")
    check_supported({"encoder.rnns.0.rnn.weight_hh_l0": torch.zeros(4 * 16, 16)}, "deepspeech2")


def test_engine_without_cuda_raises_the_library_error(monkeypatch):
    """No CUDA device: the engine refuses with the package's own error type (there is no CPU fallback)."""
    import torch
    from masr_b200 import _lib
    from masr_b200.engine import ConformerEngine
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(_lib.MasrB200Error, match="needs a CUDA device"):
        ConformerEngine({})
