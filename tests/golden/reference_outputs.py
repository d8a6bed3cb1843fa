"""Outputs of the unmodified reference build (oracle/_ref) that the tests compare against, stored in
tests/golden/reference_<group>.npz so that the comparisons run where the reference build is absent.

A test calls `recorded(group, key, fn, *args)` where it would call the reference. Normally the value stored under `key`
is returned and fn is not called. With SHB_RECORD_REFERENCE=1 (and oracle/_ref built from a shasta source tree by
`make -C oracle ref SHASTA_REF_SRC=<shasta>/src`), fn is called, its value returned, and the files are rewritten when
the process exits:

    SHB_RECORD_REFERENCE=1 SHASTA_REF_SRC=<shasta>/src python -m pytest tests -m "not gpu"

fn returns an array, a scalar, a string or a dict of those; the inputs of every recorded call are built from fixed seeds.

The reference's overlap DP comes from SeqAn, which oracle/_ref does not have: its Align4.cpp is compiled against a shim that
forwards the DP to this project's oracle/align_oracle.c. So the recorded `align4_*` alignments pin the reference's Align4
front end (cells, components, bands, selection) around the project's own DP, not the DP itself; the `info_*`, `compress_*`
and every other recorded output come from the reference's code alone.
"""
import atexit
import hashlib
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
RECORD = os.environ.get("SHB_RECORD_REFERENCE") == "1"

_loaded = {}
_pending = {}


def _path(group):
    return os.path.join(HERE, f"reference_{group}.npz")


def _save():
    for group, values in _pending.items():
        out = {}
        if os.path.exists(_path(group)):
            with np.load(_path(group)) as z:
                out.update(z)
        for key, v in values.items():
            out = {k: a for k, a in out.items() if k != key and not k.startswith(key + "/")}
            if isinstance(v, dict):
                out.update({f"{key}/{name}": np.asarray(x) for name, x in v.items()})
            else:
                out[key] = np.asarray(v)
        np.savez_compressed(_path(group), **out)


def shrink(a, limit):
    """An array as it is recorded: itself, or the SHA-256 of its bytes when it has more than `limit` elements. A test
    compares with a recording by the limit that made it."""
    a = np.ascontiguousarray(a)
    return np.frombuffer(hashlib.sha256(a.tobytes()).digest(), np.uint8) if a.size > limit else a


def _unpack(a):
    return a.item() if a.ndim == 0 else a


def recorded(group, key, fn, *args, **kwargs):
    if RECORD:
        from oracle import bindings as B
        assert B.have_ref(), "SHB_RECORD_REFERENCE=1 needs the reference build oracle/_ref"
        value = fn(*args, **kwargs)
        if not _pending:
            atexit.register(_save)
        _pending.setdefault(group, {})[key] = value
        return value
    return _stored(group, key)


def stored(group, key):
    """The value under `key` without calling the reference: the one recorded in this process under
    SHB_RECORD_REFERENCE=1, else the one in the file."""
    if key in _pending.get(group, {}):
        return _pending[group][key]
    return _stored(group, key)


def _stored(group, key):
    if group not in _loaded:
        with np.load(_path(group)) as z:
            _loaded[group] = dict(z)
    z = _loaded[group]
    if key in z:
        return _unpack(z[key])
    prefix = key + "/"
    parts = {k[len(prefix):]: _unpack(a) for k, a in z.items() if k.startswith(prefix)}
    assert parts, f"no recorded reference output {key!r} in {_path(group)}"
    return parts
