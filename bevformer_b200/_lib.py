"""ctypes binding of ``libbevformer_b200.so``, derived from the C ABI in ``include/bevformer_b200.h``.

The header is the one statement of the ABI: every ``BEVF_API`` prototype is bound with the ctypes types of its C
types, and ``ABI_VERSION`` and the enum codes (``ENUMS``) are read from it.  There is no fallback: if the library is
missing and cannot be built, importing an op raises.
"""
from __future__ import annotations

import ctypes
import os
import re
import threading

from . import build as _build

_lock = threading.Lock()
_lib = None

# the scalar C types the header passes by value; every pointer is a c_void_p.  Any other type raises at import, so a
# new entry point with a new scalar type cannot bind wrongly.
_SCALARS = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "float": ctypes.c_float,
            "double": ctypes.c_double}


def _ctype(decl: str, named: bool = True):
    """ctypes type of a C parameter declaration (``named``: it ends in the parameter's name) or return type."""
    if "*" in decl:
        return ctypes.c_void_p
    words = [w for w in decl.split() if w != "const"]
    scalar = " ".join(words[:-1] if named else words)
    if scalar not in _SCALARS:
        raise RuntimeError(f"bevformer_b200: no ctypes type for the C type of {decl!r} in {_build.HEADER}")
    return _SCALARS[scalar]


def _parse_header(path: str):
    with open(path) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    signatures = {}
    for ret, name, args in re.findall(r"BEVF_API\s+([\w\s\*]+?)\b(bevf_\w+)\s*\(([^)]*)\)\s*;", text):
        restype = ctypes.c_char_p if "".join(ret.split()) == "constchar*" else _ctype(ret, named=False)
        params = [] if args.strip() == "void" else args.split(",")
        signatures[name] = (restype, [_ctype(p) for p in params])
    version = int(re.search(r"#define\s+BEVF_ABI_VERSION\s+(\d+)", text).group(1))
    enums = {}
    for body in re.findall(r"\benum\s+\w+\s*\{([^}]*)\}", text):
        for item in filter(str.strip, body.split(",")):
            key, value = item.split("=")              # every enumerator has an explicit integer value
            enums[key.strip()] = int(value)
    return signatures, version, enums


# name -> (restype, argtypes) of every entry point; the ABI version; enumerator name -> code
SIGNATURES, ABI_VERSION, ENUMS = _parse_header(_build.HEADER)


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True):
    """Load (building first if the in-tree .so is absent or stale and nvcc exists)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        path = _build.LIB_PATH
        if build_if_missing:
            try:
                path = _build.build()
            except Exception as e:  # no nvcc on this box: use the prebuilt .so if there is one
                if not os.path.exists(path):
                    raise RuntimeError(
                        "bevformer_b200: the CUDA library is missing and could not be built "
                        f"({e}); there is no CPU fallback") from e
        if not os.path.exists(path):
            raise RuntimeError(f"bevformer_b200: {path} not found; there is no CPU fallback")
        lib = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)   # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        have = lib.bevf_version()
        if have != ABI_VERSION:
            raise RuntimeError(f"bevformer_b200: ABI mismatch (library {have}, binding {ABI_VERSION})")
        _lib = lib
    return _lib


def check(status: int, lib=None) -> None:
    """Non-zero status -> RuntimeError carrying the library's message (what mmcv's TORCH_CHECK
    failures look like from Python)."""
    if status != 0:
        lib = lib or load()
        raise RuntimeError(lib.bevf_last_error().decode() or f"bevformer_b200 error {status}")


def launch_count() -> int:
    return int(load().bevf_launch_count())
