"""The C ABI as Python sees it: the ctypes bindings of fast3r_b200.lib and the ctypes structs against the prototypes and
structs of include/fast3r_b200.h, the CPU emulator (tests/abi_emulator.py) against the ops wrappers it stands in for,
and the library's exports and argument checks.  ctypes passes whatever its argtypes say without comparing them to the
C prototype, so a binding that disagrees with the header would only show up later, as a wrong answer or a GPU fault."""
import ctypes as C
import inspect
import os
import re

import pytest

from tests.conftest import ROOT


def _header() -> str:
    """include/fast3r_b200.h without comments and preprocessor lines."""
    with open(os.path.join(ROOT, "include", "fast3r_b200.h")) as f:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", "", f.read(), flags=re.S)
    return re.sub(r"^\s*#[^\n]*", "", src, flags=re.M)


def _c_kind(decl: str) -> str:
    """Argument-passing kind of a C type, optionally followed by a name.  size_t and uint64_t share one kind: ctypes has
    one type for both (c_size_t is c_uint64 on LP64)."""
    if "*" in decl:
        return "ptr"
    base = re.sub(r"\b(const|struct)\b", "", decl).split()[0]
    return {"int": "i32", "int32_t": "i32", "size_t": "u64", "uint64_t": "u64", "float": "f32", "void": "void"}[base]


def _ctypes_kind(t) -> str:
    if t is None:
        return "void"
    if t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer):
        return "ptr"
    return {C.c_int32: "i32", C.c_uint64: "u64", C.c_float: "f32"}[t]


def _prototypes() -> dict:
    """name -> (return kind, [argument kinds]) of every f3r_* prototype, in header order."""
    protos = {}
    for ret, name, args in re.findall(r"([\w\s*]+?)\b(f3r_\w+)\s*\(([^()]*)\)\s*;", _header()):
        args = [a for a in args.split(",") if a.strip() not in ("", "void")]
        protos[name] = (_c_kind(ret), [_c_kind(a) for a in args])
    return protos


def _struct_fields(name: str) -> list:
    """[(field, kind)] of `typedef struct name {...} name;`, in declaration order (`int32_t n, k, taps;` is three)."""
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), _header(), re.S).group(1)
    fields = []
    for decl in filter(str.strip, body.split(";")):
        ctype, names = re.fullmatch(r"\s*(.*?[\s*])(\w+(?:\s*,\s*\w+)*)\s*", decl, re.S).groups()
        fields += [(n.strip(), _c_kind(ctype)) for n in names.split(",")]
    return fields


def test_bindings_match_header_prototypes():
    """fast3r_b200.lib binds every prototype of the header, with the same arity, argument kinds and return kind."""
    from fast3r_b200 import lib as L
    protos = _prototypes()
    assert list(L._API) == list(protos)
    for name, (restype, argtypes) in L._API.items():
        assert (_ctypes_kind(restype), [_ctypes_kind(t) for t in argtypes]) == protos[name], name


@pytest.mark.parametrize("c_name,py_name", [("f3r_gemm_desc", "GemmDesc")])
def test_structs_match_header(c_name, py_name):
    from fast3r_b200 import lib as L
    fields = [(n, _ctypes_kind(t)) for n, t in getattr(L, py_name)._fields_]
    assert fields == _struct_fields(c_name)


def test_emulator_signatures_match_ops():
    """Every function of the CPU emulator exists in ops with the same parameters (names, kinds, defaults): a keyword
    that only the emulator accepted would pass the CPU host tests and fail on the GPU."""
    from fast3r_b200 import ops
    from tests import abi_emulator as E
    names = [n for n, f in vars(E).items() if inspect.isfunction(f) and f.__module__ == E.__name__ and n[0] != "_"]
    assert "gemm" in names and "focal_weiszfeld" in names
    params = lambda f: [(p.name, p.kind, p.default) for p in inspect.signature(f).parameters.values()]  # noqa: E731
    for name in names:
        assert inspect.isfunction(getattr(ops, name, None)), name
        assert params(getattr(E, name)) == params(getattr(ops, name)), name


def test_cabi_exports_every_declared_symbol():
    from fast3r_b200 import lib as L
    from fast3r_b200.build import build
    build()
    hdr = open(os.path.join(ROOT, "include", "fast3r_b200.h")).read()
    declared = set(re.findall(r"\b(f3r_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(L.EXPORTS), declared ^ set(L.EXPORTS)
    lib = C.CDLL(L.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert L.load().f3r_abi_version() == L.ABI_VERSION == 3
    assert L.load().f3r_gemm_desc_size() == C.sizeof(L.GemmDesc) == 208


def test_cabi_rejects_bad_arguments_before_any_cuda_call():
    """Argument validation of the C ABI runs before the first CUDA call, so it is checkable without a GPU: every entry
    point returns non-zero and leaves a message naming itself in f3r_last_error()."""
    from fast3r_b200 import lib as L
    lib = L.load()
    f = C.c_float
    cases = [
        ("f3r_conf_quantile", (None, 1, 10, f(0.5), None, None), "null operand"),
        ("f3r_conf_quantile", (8, 1, 10, f(1.5), 8, None), "q must be in [0, 1]"),
        ("f3r_conf_quantile", (8, 1, 1 << 25, f(0.5), 8, None), "bad shape"),
        ("f3r_similarity_fit", (8, 8, 8, None, None, 1, 10, 8, 8, 10 ** 6, None), "conf and thr must be given together"),
        ("f3r_similarity_fit", (8, 8, None, None, None, 1, 10, 8, 8, 16, None), "workspace too small"),
        ("f3r_similarity_fit", (8, 8, None, None, None, 1, 10, 8, 9, 10 ** 6, None), "not 8-byte aligned"),
        ("f3r_similarity_fit", (8, 8, None, None, None, 70000, 10, 8, 8, 10 ** 9, None), "bad shape"),
        ("f3r_similarity_apply", (8, None, 8, 1, 10, None), "null operand"),
        ("f3r_focal_weiszfeld", (8, None, None, None, 1, 4, 4, -1, 8, 8, 10 ** 6, None), "bad iteration count"),
        ("f3r_focal_weiszfeld", (8, 8, None, None, 1, 4, 4, 10, 8, 8, 10 ** 6, None), "conf and thr must be given together"),
        ("f3r_focal_weiszfeld", (8, None, None, None, 1, 4, 4, 10, 8, 8, 16, None), "workspace too small"),
        ("f3r_layernorm", (None, None, None, None, 0, 1, 1024, f(1e-6), None), "null operand"),
        ("f3r_attention", (None, 0, None, 0, None, 0, None, 1, 16, 128, 128, f(0.125), None), "null operand"),
    ]
    for name, args, msg in cases:
        assert getattr(lib, name)(*args) != 0, name
        err = lib.f3r_last_error().decode()
        assert err.startswith(name) and msg in err, (name, err)
    # workspace queries are pure host functions
    assert lib.f3r_similarity_fit_workspace(0) == 0 and lib.f3r_similarity_fit_workspace(3) % 8 == 0
    assert lib.f3r_focal_workspace(2) == 2 * 2 * 256 * 3 * 8
    with pytest.raises(RuntimeError, match="f3r_conf_quantile failed"):
        L.check(lib.f3r_conf_quantile(None, 1, 10, f(0.5), None, None), "f3r_conf_quantile")
