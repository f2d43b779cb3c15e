"""C-ABI checks that need no GPU: the library loads, exports every symbol include/actionmesh_b200.h declares, the
ctypes binding read from that header has its signatures and struct layouts, and argument validation fails loudly with
an error code + message (no compute calls)."""
import ctypes as C
import os
import re
import subprocess

import pytest

from conftest import ROOT


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "actionmesh_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(amb_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_expected_entry_points():
    names = _declared_functions()
    for n in ("amb_gemm_bf16", "amb_flash_attn_fwd", "amb_cfg_euler_step", "amb_layernorm", "amb_last_error"):
        assert n in names


def test_library_exports_every_declared_symbol(amb_lib):
    for name in _declared_functions():
        assert hasattr(amb_lib, name), f"{name} declared in the header but not exported"


def test_binding_matches_header(amb_lib):
    from actionmesh_b200 import _lib

    assert sorted(_lib.EXPORTS) == _declared_functions()
    text = open(os.path.join(ROOT, "include", "actionmesh_b200.h")).read()
    ver = int(re.search(r"#define AMB_ABI_VERSION (\d+)", text).group(1))
    assert amb_lib.amb_abi_version() == ver == _lib.ABI_VERSION


def test_struct_layouts_match_header(tmp_path):
    """Every field offset and the size of the ctypes structs equal the C compiler's offsetof / sizeof for the header."""
    from actionmesh_b200 import _lib

    structs = (("amb_gemm_args", _lib.GemmArgs), ("amb_attn_args", _lib.AttnArgs))
    prints = [f'printf("%zu\\n", sizeof({cname}));' for cname, _ in structs]
    prints += [f'printf("%zu\\n", offsetof({cname}, {f}));' for cname, cls in structs for f, _ in cls._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "actionmesh_b200.h"\nint main(void) {\n'
                   + "\n".join(prints) + "\nreturn 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    want = [C.sizeof(cls) for _, cls in structs] + [getattr(cls, f).offset for _, cls in structs for f, _ in cls._fields_]
    assert got == want


def test_binding_maps_every_parameter(amb_lib):
    """The header parse binds every declared function with one ctypes type per declared parameter, and load_library
    applies exactly those types."""
    from actionmesh_b200 import _lib

    prototypes, _ = _lib.parse_header(_lib.HEADER_PATH)
    assert sorted(prototypes) == _declared_functions()
    text = re.sub(r"/\*.*?\*/", "", open(_lib.HEADER_PATH).read(), flags=re.S)
    for name, (restype, argtypes) in prototypes.items():
        params = re.search(r"\b%s\s*\(([^)]*)\)" % name, text).group(1).strip()
        assert len(argtypes) == (0 if params == "void" else params.count(",") + 1), name
        fn = getattr(amb_lib, name)
        assert tuple(fn.argtypes) == tuple(argtypes) and fn.restype is restype, name
    P = C.c_void_p
    assert prototypes["amb_cfg_euler_step"] == (C.c_int, [P, P, C.c_int, P, C.c_float, P, C.c_int, C.c_int64, C.c_int64,
                                                          C.c_int64, C.c_int64, P])
    assert prototypes["amb_mesh_collapse_apply"][1][6] is C.c_uint64
    assert prototypes["amb_last_error"] == (C.c_char_p, [])


@pytest.mark.parametrize("decl", [
    "int amb_bad(const float* x, double scale, amb_stream_t stream);",      # unknown scalar
    "int amb_bad(const size_t* x, amb_stream_t stream);",                  # unknown pointee
    "int amb_bad(const float** x, amb_stream_t stream);",                  # pointer to pointer
    "void amb_bad(int n);",                                                # unknown return type
    "typedef struct amb_bad_args { int32_t m; long n; } amb_bad_args;",    # unknown member type
])
def test_header_parse_refuses_unknown_types(tmp_path, decl):
    from actionmesh_b200 import _lib

    header = tmp_path / "bad.h"
    header.write_text("/* comment */\nint amb_ok(int n, amb_stream_t stream);\n" + decl + "\n")
    with pytest.raises(_lib.AmbError, match="amb_bad"):
        _lib.parse_header(str(header))


def test_argument_validation_fails_loudly(amb_lib):
    from actionmesh_b200 import _lib

    g = _lib.GemmArgs()
    rc = amb_lib.amb_gemm_bf16(C.byref(g), None)
    assert rc < 0 and b"null pointer" in amb_lib.amb_last_error()
    g.a, g.w, g.c = 16, 16, 16  # fake non-null pointers: validation must stop before any launch
    g.m, g.n, g.k = 128, 100, 64
    g.lda = g.ldw = g.ldc = 64
    rc = amb_lib.amb_gemm_bf16(C.byref(g), None)
    assert rc < 0 and b"multiple of 64" in amb_lib.amb_last_error()
    a = _lib.AttnArgs()
    a.q = a.k = a.v = a.o = 16
    a.batch = a.heads = 1
    a.sq = a.sk = 64
    a.head_dim = 96
    rc = amb_lib.amb_flash_attn_fwd(C.byref(a), None)
    assert rc < 0 and b"head_dim" in amb_lib.amb_last_error()
    rc = amb_lib.amb_layernorm(None, 0, 0, None, None, None, 0, 0, 1, 2048, 1e-5, None)
    assert rc < 0


def test_product_path_has_no_cpu_fallback():
    """Ops refuse CPU tensors, and nothing under actionmesh_b200/ imports the oracle."""
    import torch

    from actionmesh_b200 import AmbError, ops

    with pytest.raises(AmbError):
        ops.layernorm(torch.zeros(4, 2048, dtype=torch.bfloat16), torch.ones(2048), torch.zeros(2048), 1e-5)
    pkg = os.path.join(ROOT, "actionmesh_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("# oracle", ""), f"{fn} references the oracle"


def test_missing_library_raises(monkeypatch, tmp_path):
    from actionmesh_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.AmbError):
        _lib.load_library()


def test_argument_validation_of_widened_entry_points(amb_lib):
    """Stage-II helpers and the preprocessing kernels validate their geometry before any launch (fake non-null pointers)."""
    P = 16
    err = lambda: amb_lib.amb_last_error().decode()
    assert amb_lib.amb_split3_bf16(None, 0, 1, 128, 128, 0, None, 0, None) < 0 and "null pointer" in err()
    assert amb_lib.amb_split3_bf16(P, 128, 1, 128, 96, 0, P, 384, None) < 0 and "bad geometry" in err()     # cols % seg != 0
    assert amb_lib.amb_split3_bf16(P, 128, 1, 128, 128, 0, P, 256, None) < 0 and "bad geometry" in err()    # ld_dst < 3*cols
    assert amb_lib.amb_softmax_split3(P, 128, 1, 130, 128, 1.0, P, 384, None) < 0 and "bad geometry" in err()  # n > n_pad
    assert amb_lib.amb_softmax_split3(P, 64, 1, 100, 128, 1.0, P, 384, None) < 0                               # ld_s < n_pad
    assert amb_lib.amb_alpha_rows(0.0, 1.0, 511, P, 1024, 1, None) < 0 and "alpha_rows" in err()               # odd size
    assert amb_lib.amb_point_embedding(P, 4, 6, 3, 8, 0, P, 32, None) < 0 and "bad geometry" in err()          # kpad too small
    assert amb_lib.amb_point_embedding(P, 4, 5, 3, 8, 0, P, 64, None) < 0                                      # in_dim != 3 + extra
    assert amb_lib.amb_displacement_out(P, 2, 4, 3, P, None) < 0                                               # ld < out_dim
    assert amb_lib.amb_resize_h_u8(P, 1, 64, 64, 2, 0, 64, P, P, 9, 32, P, None) < 0 and "bad geometry" in err()  # 2 channels
    assert amb_lib.amb_resize_h_u8(P, 1, 64, 64, 3, 60, 8, P, P, 9, 32, P, None) < 0 and "outside the image" in err()
    m = (C.c_float * 3)(0, 0, 0)
    assert amb_lib.amb_resize_v_normalize(P, 1, 0, 0, 32, P, P, 9, 32, P, m, m, P, None, None) < 0 and "bad geometry" in err()
    assert amb_lib.amb_resize_v_normalize(P, 1, 8, 0, 32, P, P, 9, 32, None, m, m, P, None, None) < 0 and "null pointer" in err()
    # zero-size work is a successful no-op without a launch
    assert amb_lib.amb_split3_bf16(P, 128, 0, 128, 128, 0, P, 384, None) == 0
    assert amb_lib.amb_softmax_split3(P, 128, 0, 100, 128, 1.0, P, 384, None) == 0
    assert amb_lib.amb_resize_h_u8(P, 0, 64, 64, 3, 0, 64, P, P, 9, 32, P, None) == 0


@pytest.mark.parametrize("src,dst", [(16 + 4, 16), (16 + 8, 16), (16, 16 + 2), (16, 16 + 4), (16 + 4, 16 + 2)])
def test_split_operands_refuse_misaligned_pointers(amb_lib, src, dst):
    """split3 reads float4 and writes 4-element bf16 vectors, softmax_split3 the same: a source that is not 16-byte
    aligned or a destination that is not 8-byte aligned (a column-offset view such as x[:, 1:]) is refused before any
    launch, naming the argument; zero rows do not skip the check (fake non-null pointers)."""
    err = lambda: amb_lib.amb_last_error().decode()
    name = "src" if src % 16 else "dst"
    for rows in (1, 0):
        assert amb_lib.amb_split3_bf16(src, 128, rows, 128, 128, 0, dst, 384, None) < 0
        assert f"split3: {name} must be" in err()
        assert amb_lib.amb_softmax_split3(src, 128, rows, 100, 128, 1.0, dst, 384, None) < 0
        assert f"softmax_split3: {'scores' if name == 'src' else 'dst'} must be" in err()


def test_split_operands_accept_aligned_pointers(amb_lib):
    """The smallest alignments the kernels need pass validation: 16-byte sources, 8-byte destinations (zero rows: no
    launch)."""
    assert amb_lib.amb_split3_bf16(32, 128, 0, 128, 128, 0, 24, 384, None) == 0
    assert amb_lib.amb_softmax_split3(32, 128, 0, 100, 128, 1.0, 24, 384, None) == 0
    assert amb_lib.amb_split3_bf16(16, 128, 0, 128, 128, 0, 8, 384, None) == 0
