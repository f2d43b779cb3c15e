"""ctypes binding of libactionmesh_b200.so.

The C header include/actionmesh_b200.h is the only declaration of the ABI: when this module is imported it reads every
`int amb_*(...)` / `const char* amb_*(...)` prototype and the `typedef struct ... amb_*_args` bodies from it, and
load_library() sets each function's argtypes and restype from that parse.  The types form a closed set: int, int32_t,
int64_t, uint64_t and float bind as their ctypes equivalents; every pointer (device or host) and amb_stream_t binds as
c_void_p, which takes raw addresses, None, ctypes arrays and byref(...).  Any other type is an AmbError at import.

There is no CPU fallback: if the shared library is missing or a call fails the error is raised.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libactionmesh_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "actionmesh_b200.h")

ABI_VERSION = 17


class AmbError(RuntimeError):
    pass


_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float,
            "amb_stream_t": C.c_void_p}
_POINTEES = {"void", "float", "double", "int", "uint8_t", "int32_t", "int64_t", "uint64_t", "amb_gemm_args", "amb_attn_args"}
_RESTYPES = {"int": C.c_int, "const char*": C.c_char_p}
# one parameter or struct member line: [const] type [*] name[, name ...]
_DECL = re.compile(r"(?:const\s+)?(\w+)(?:\s*(\*)\s*|\s+)(\w+(?:\s*,\s*\w+)*)")


def _decl(text: str, where: str) -> tuple[list[str], type]:
    """'const float* gamma' or 'int32_t m, n, k' -> (names, ctypes type)."""
    m = _DECL.fullmatch(text.strip())
    if m is None or m[1] not in (_POINTEES if m[2] else _SCALARS):
        raise AmbError(f"{where}: `{' '.join(text.split())}` is outside the types the binding maps")
    return re.split(r"\s*,\s*", m[3]), C.c_void_p if m[2] else _SCALARS[m[1]]


def parse_header(path: str = HEADER_PATH) -> tuple[dict, dict]:
    """-> ({function: (restype, argtypes)}, {struct typedef: _fields_}) in declaration order."""
    with open(path) as f:
        text = re.sub(r"/\*.*?\*/|^\s*#.*?$", " ", f.read(), flags=re.S | re.M)
    prototypes = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\s*\b(amb_\w+)\s*\(([^()]*)\)\s*;", text):
        restype = _RESTYPES.get(re.sub(r"\s*\*", "*", " ".join(ret.split())))
        if restype is None:
            raise AmbError(f"{name}: return type `{ret.strip()}` is outside the types the binding maps")
        argtypes = [] if params.strip() == "void" else [_decl(p, name)[1] for p in params.split(",")]
        prototypes[name] = (restype, argtypes)
    structs = {}
    for body, name in re.findall(r"typedef\s+struct\s+\w*\s*\{([^}]*)\}\s*(\w+)\s*;", text):
        fields = []
        for member in filter(str.strip, body.split(";")):
            names, ctype = _decl(member, name)
            fields += [(n, ctype) for n in names]
        structs[name] = fields
    return prototypes, structs


_PROTOTYPES, _STRUCTS = parse_header()
EXPORTS = list(_PROTOTYPES)


class GemmArgs(C.Structure):
    _fields_ = _STRUCTS["amb_gemm_args"]


class AttnArgs(C.Structure):
    _fields_ = _STRUCTS["amb_attn_args"]


_lib = None


def load_library() -> C.CDLL:
    """Load the CUDA extension; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AmbError(
            f"{LIB_PATH} not found: the sm_90a CUDA extension has not been built. "
            "Run `python __graft_entry__.py` (there is no CPU fallback)."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.amb_abi_version() != ABI_VERSION:
        raise AmbError(f"ABI mismatch: library {lib.amb_abi_version()} != binding {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load_library().amb_last_error().decode(errors="replace")
        raise AmbError(f"{what} failed (code {rc}): {msg}")


@functools.lru_cache(maxsize=256)
def scan_scratch_ints(n_items: int) -> int:
    """amb_scan_scratch_ints: the int32 scan scratch a kernel over n_items needs; its last entry receives the total."""
    nints = C.c_int64()
    check(load_library().amb_scan_scratch_ints(int(n_items), C.byref(nints)), "amb_scan_scratch_ints")
    return nints.value
