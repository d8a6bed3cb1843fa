"""CPU test: the C-ABI library loads and exports every entry point include/*.h declares."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        text = open(h).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        names.update(re.findall(r"\b(shb_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_library_exports_every_declared_symbol():
    from shasta_b200 import capi
    assert os.path.exists(capi.LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(capi.LIB_PATH)
    syms = declared_symbols()
    assert "shb_lowhash0" in syms and "shb_set_markers" in syms
    for s in syms:
        assert hasattr(lib, s), f"{s} is declared in include/ but not exported"


def test_no_cpu_fallback_without_device():
    # Without a GPU the context creation must fail loudly (SHB_ERR_CUDA), never fall back to a CPU path.
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from shasta_b200 import capi
    with pytest.raises(capi.ShastaB200Error):
        capi.Context(0)


def test_product_does_not_import_oracle():
    # The oracle is test infrastructure; nothing under shasta_b200/ may import, include, link or call it.
    forbidden = re.compile(r"\bfrom\s+oracle\b|\bimport\s+oracle\b|oracle/|liboracle|libshasta_ref|\borc_[a-z]|\bref_[a-z]+\(")
    for path in glob.glob(os.path.join(ROOT, "shasta_b200", "**", "*"), recursive=True):
        if os.path.isfile(path) and path.endswith((".py", ".cu", ".cuh", ".cpp", ".h", "Makefile")):
            for line_no, line in enumerate(open(path), 1):
                assert not forbidden.search(line), f"{path}:{line_no}: {line.strip()}"


def declared_parameter_counts():
    counts = {}
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        text = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        for name, params in re.findall(r"\b(shb_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", text, flags=re.S):
            params = params.strip()
            counts[name] = 0 if params in ("", "void") else params.count(",") + 1
    return counts


def test_ctypes_argument_lists_match_the_header():
    """capi.lib() declares the argtypes of every function in include/shasta_b200.h that has parameters when it loads the
    library, and each passes as many arguments as the prototype has."""
    from shasta_b200 import capi
    lib = capi.lib()
    counts = declared_parameter_counts()
    assert counts["shb_lowhash0"] == 8 and counts["shb_last_error"] == 0
    for name, n in counts.items():
        argtypes = getattr(lib, name).argtypes
        if n:
            assert argtypes is not None, f"{name}: no ctypes argument list"
        if argtypes is not None:
            assert len(argtypes) == n, f"{name}: {len(argtypes)} ctypes arguments, {n} in the header"
