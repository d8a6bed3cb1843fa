"""CPU test: the oracle's binding modules declare, when they load their libraries, the ctypes prototype of every function the
oracle's C files (orc_*) and the reference glue (extern "C" ref_*) define. An undeclared function returns a C int, which would
cut a uint64_t or double short without an error, and takes whatever arguments it is given."""
import ctypes as C
import glob
import importlib
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
MODULES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(ORACLE, "*bindings.py")))
RETURN_TYPES = {"void": None, "int": C.c_int, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "double": C.c_double}
DEFINITION = re.compile(r"^([A-Za-z_][\w \t*]*?)\b((?:orc|ref)_\w+)\s*\(([^()]*)\)\s*\{", re.M)


def _source(path):
    text = re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _extern_c(text):
    """The bodies of the extern "C" { ... } blocks of text."""
    blocks = []
    for m in re.finditer(r'extern\s+"C"\s*\{', text):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            i += 1
        blocks.append(text[m.end():i - 1])
    return "\n".join(blocks)


def definitions(text):
    """{name: (return type, parameter count)} of the orc_* / ref_* functions text defines outside any other function."""
    out = {}
    for ret, name, params in DEFINITION.findall(text):
        words = ret.split()
        if "static" in words:
            continue
        params = params.strip()
        out[name] = (" ".join(words), 0 if params in ("", "void") else params.count(",") + 1)
    return out


def glue_by_library():
    """{reference library file name: its glue files}, from oracle/Makefile's <library>_GLUE lists."""
    text = open(os.path.join(ORACLE, "Makefile")).read()
    return {f"lib{lib}.so": [os.path.join(ORACLE, "ref_glue", g + ".cpp") for g in glue.split()]
            for lib, glue in re.findall(r"^(\w+)_GLUE\s*=\s*(.+)$", text, re.M)}


def check(lib, defs):
    for name, (ret, n) in sorted(defs.items()):
        assert ret in RETURN_TYPES, f"{name}: return type {ret} has no ctypes counterpart here"
        f = getattr(lib, name)
        assert f.argtypes is not None, f"{name}: no ctypes argument list"
        assert len(f.argtypes) == n, f"{name}: {len(f.argtypes)} ctypes arguments, {n} in its definition"
        assert f.restype is RETURN_TYPES[ret], f"{name}: restype {f.restype}, defined as returning {ret}"


def test_oracle_prototypes_match_the_definitions():
    defs = {}
    for path in glob.glob(os.path.join(ORACLE, "*.c")):
        defs.update(definitions(_source(path)))
    assert {"orc_lowhash0", "orc_murmurhash64a", "orc_histogram2_threshold", "orc_create_marker_graph_edges"} <= set(defs)
    assert defs["orc_murmurhash64a"] == ("uint64_t", 3) and defs["orc_get_dp_policy"] == ("int", 0)
    mods = [importlib.import_module("oracle." + m) for m in MODULES]
    libs = {id(lib): lib for lib in (mod.oracle_lib() for mod in mods if hasattr(mod, "oracle_lib"))}
    assert len(libs) == 1, "every binding module shares one liboracle.so handle"
    check(*libs.values(), defs)


def test_every_glue_file_belongs_to_a_reference_library():
    listed = {g for files in glue_by_library().values() for g in files}
    assert listed == set(glob.glob(os.path.join(ORACLE, "ref_glue", "*.cpp")))


@pytest.mark.parametrize("module", MODULES)
def test_reference_prototypes_match_the_glue(module):
    mod = importlib.import_module("oracle." + module)
    if not mod.have_ref():
        pytest.skip(f"{mod.REF_SO} is absent")
    defs = {}
    for path in glue_by_library()[os.path.basename(mod.REF_SO)]:
        defs.update(definitions(_extern_c(_source(path))))
    assert defs and all(name.startswith("ref_") for name in defs)
    check(mod.ref_lib(), defs)
