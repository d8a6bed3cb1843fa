"""TEST INFRASTRUCTURE — how every oracle binding module opens its libraries (oracle/_build/liboracle.so, oracle/_ref/*.so).

Each binding module keeps one prototype table per library, {name: (restype, argtypes)}, next to its wrappers, and gets the
library through load(), which declares every function the table names when it first sees the table. take() copies a block
that a library function allocated and frees it.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_libs = {}
_declared = {}


def load(path, protos):
    """The library at path, opened once per process, with restype and argtypes set from protos for every function it names.
    A name the library does not export is skipped: a prebuilt library older than a function's glue then raises
    AttributeError when that function is called, as it would without the table."""
    lib = _libs.get(path)
    if lib is None:
        lib = _libs[path] = C.CDLL(path)
    if (path, id(protos)) not in _declared:
        for name, (restype, argtypes) in protos.items():
            f = getattr(lib, name, None)
            if f is not None:
                f.restype, f.argtypes = restype, argtypes
        _declared[(path, id(protos))] = protos
    return lib


def have(path):
    return os.path.exists(path)


def take(ptr, count, dtype, free):
    """A copy of the count dtype elements at ptr, a block a library function returned, which free then releases. An empty
    array for count == 0 or a null pointer."""
    p = ptr.value if isinstance(ptr, C.c_void_p) else ptr
    dtype = np.dtype(dtype)
    if count and p:
        out = np.ctypeslib.as_array((C.c_uint8 * (count * dtype.itemsize)).from_address(p)).view(dtype).copy()
    else:
        out = np.zeros(0, dtype)
    if p:
        free(p)
    return out
