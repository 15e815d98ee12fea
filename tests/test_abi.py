"""The C-ABI library loads on a GPU-less host and exports exactly what include/*.h declares.
No compute is launched here (there is no GPU in the dev container)."""
import ctypes
import os
import re

import pytest

from bevformer_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "bevformer_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.findall(r"BEVF_API\s+[\w\s\*]+?\b(bevf_\w+)\s*\(", text)


def test_header_declares_something():
    syms = declared_symbols()
    assert "bevf_msda_forward" in syms and "bevf_msda_backward" in syms and len(syms) >= 5


def test_library_builds_and_exports_every_declared_symbol():
    path = build.build()
    lib = ctypes.CDLL(path)
    for s in declared_symbols():
        assert hasattr(lib, s), f"{s} declared in the header but not exported"


# type code of each ctypes type of the binding, and the C++ template that spells the same code for a C type
_CODES = {ctypes.c_void_p: "p", ctypes.c_char_p: "s", ctypes.c_int: "i", ctypes.c_int64: "q", ctypes.c_uint64: "Q",
          ctypes.c_float: "f", ctypes.c_double: "d"}
_TYPE_CODES_CPP = r"""
#include <cstdio>
#include <string>
#include "bevformer_b200.h"
template <class T> struct code;                       // a type without a code does not compile
template <class T> struct code<T *> { static constexpr char c = 'p'; };
template <> struct code<int> { static constexpr char c = 'i'; };
template <> struct code<int64_t> { static constexpr char c = 'q'; };
template <> struct code<uint64_t> { static constexpr char c = 'Q'; };
template <> struct code<float> { static constexpr char c = 'f'; };
template <> struct code<double> { static constexpr char c = 'd'; };
template <class T> struct ret : code<T> {};
template <> struct ret<const char *> { static constexpr char c = 's'; };
template <class F> struct sig;
template <class R, class... A> struct sig<R (*)(A...)> {
    static std::string str() { return std::string(1, ret<R>::c) + std::string{code<A>::c...}; }
};
int main() {
"""


def test_binding_covers_header_exactly(tmp_path):
    """The binding has exactly the header's entry points, with the return and argument types the C++ compiler sees
    in the header's prototypes."""
    import shutil
    import subprocess
    assert sorted(_lib.SIGNATURES) == sorted(declared_symbols())
    cxx = shutil.which("c++") or shutil.which("g++")
    if not cxx:
        pytest.skip("no host C++ compiler on PATH")
    src = tmp_path / "type_codes.cpp"
    src.write_text(_TYPE_CODES_CPP + "".join(f'    std::printf("{n} %s\\n", sig<decltype(&{n})>::str().c_str());\n'
                                             for n in _lib.SIGNATURES) + "}\n")
    exe = tmp_path / "type_codes"
    subprocess.run([cxx, "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    compiled = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                            check=True).stdout.splitlines())
    bound = {n: _CODES[res] + "".join(_CODES[a] for a in args) for n, (res, args) in _lib.SIGNATURES.items()}
    assert bound == compiled


def test_version_and_error_channel():
    lib = _lib.load()
    assert lib.bevf_version() == _lib.ABI_VERSION
    assert lib.bevf_msda_forward(None, 0, None, None, None, None, None, 0, 1, 1, 1, 1, 1, 1, 1,
                                 None) != 0
    assert b"null pointer" in lib.bevf_last_error()
    with pytest.raises(RuntimeError, match="null pointer"):
        _lib.check(1, lib)
    # too many levels is rejected before any launch
    assert lib.bevf_msda_forward(16, 0, 16, 16, 16, 16, 16, 0, 1, 1, 1, 32, 1, 17, 1, None) != 0
    assert b"16 levels" in lib.bevf_last_error()


def test_ops_refuse_cpu_tensors():
    import torch
    from bevformer_b200 import ops
    v = torch.zeros(1, 4, 1, 32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.msda_forward(v, torch.tensor([[2, 2]]), torch.tensor([0]), torch.zeros(1, 1, 1, 1, 1, 2),
                         torch.zeros(1, 1, 1, 1, 1))


def test_sass_has_vector_reductions():
    """The scatter is built on 16-byte fp32 reductions (REDG.E.ADD.F32x4), not scalar atomics."""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    sass = subprocess.run(["cuobjdump", "-sass", build.build()], capture_output=True,
                          text=True).stdout
    assert "REDG.E.ADD.F32x4" in sass
