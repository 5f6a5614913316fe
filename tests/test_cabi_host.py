"""No-GPU checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/*.h
declares, the ctypes structs generated from the header have the C layout, and the host-side mirror
rejects what the reference's wrappers reject. No compute calls (there is no GPU here)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    from gssdf_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "gssdf_b200.h")).read()
    declared = set(re.findall(r"\b(gssdf_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/gssdf_b200.h but not exported"
    assert set(_lib.FUNCS) == declared
    assert b"sm_90a" in L.gssdf_version()


def test_struct_layout_matches_c_compiler(tmp_path):
    """sizeof/offsetof from gcc == the ctypes structs parsed out of the header."""
    from gssdf_b200 import _lib
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "gssdf_b200.h"', 'int main(void){']
    for name, S in _lib.STRUCTS.items():
        src.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f, _ in S._fields_:
            src.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    src.append('return 0;}')
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for name, S in _lib.STRUCTS.items():
        assert ctypes.sizeof(S) == int(out[name]), name
        for f, _ in S._fields_:
            assert getattr(S, f).offset == int(out[f"{name}.{f}"]), f"{name}.{f}"


def test_header_is_plain_c():
    """The boundary must be bindable from C / cgo / JNI: the header compiles as C99 with no C++ or torch types."""
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c",
                           os.path.join(ROOT, "include", "gssdf_b200.h")])
    from gssdf_b200 import _lib
    code = _lib._strip_comments(open(os.path.join(ROOT, "include", "gssdf_b200.h")).read())
    assert "Tensor" not in code and "std::" not in code and "torch" not in code


def test_argument_errors_without_gpu():
    """Validation that happens before any CUDA call returns the documented codes + message."""
    from gssdf_b200 import _lib
    L = _lib.lib()
    assert L.gssdf_project2dgs_fwd(None, None) == -1
    assert b"null args" in L.gssdf_last_error()
    a = _lib.make_args("gssdf_raster2dgs_fwd_args", C=1, image_width=32, image_height=32, tile_size=16, channels=5)
    assert L.gssdf_raster2dgs_fwd(ctypes.byref(a), None) == -3  # GSSDF_EUNSUPPORTED
    assert b"Unsupported number of color channels: 5" in L.gssdf_last_error()
    a = _lib.make_args("gssdf_raster2dgs_fwd_args", C=1, image_width=32, image_height=32, tile_size=16, channels=0)
    assert L.gssdf_raster2dgs_fwd(ctypes.byref(a), None) == -1  # std::invalid_argument in the reference
    a = _lib.make_args("gssdf_tile_encode_args", C=0, image_width=32, image_height=32, tile_size=16)
    assert L.gssdf_tile_encode(ctypes.byref(a), None) == -1
    a = _lib.make_args("gssdf_view_colors_fwd_args", N=4, C=1, K=4, sh_degree=3, cap=4)
    assert L.gssdf_view_colors_fwd(ctypes.byref(a), None) == -1
    assert b"Invalid coeffs shape" in L.gssdf_last_error()
    assert L.gssdf_tile_encode_workspace_bytes(1, 1920, 1080, 16, 1 << 20) >= (1 << 23)
    with pytest.raises(KeyError):
        _lib.make_args("gssdf_tile_encode_args", not_a_field=1)


def test_mirror_api_rejects_bad_shapes_on_cpu():
    torch = pytest.importorskip("torch")
    from gssdf_b200 import ops
    z = torch.zeros
    with pytest.raises(ValueError, match="Invalid scales size"):
        ops.fully_fused_projection_2dgs(z(10, 3), z(10, 4), z(10, 2), z(1, 4, 4), z(1, 3, 3), 32, 32, packed=True)
    with pytest.raises(ValueError, match="Unsupported number of color channels"):
        ops.rasterize_to_pixels_2dgs(z(4, 2), z(4, 3, 3), z(4, 0), z(4), z(4, 3), z(4, 2), 32, 32, 16,
                                     z(1, 2, 2, dtype=torch.int32), z(0, dtype=torch.int32), packed=True)
    with pytest.raises(ValueError, match="Invalid shape for opacities"):
        ops.rasterize_to_pixels_2dgs(z(4, 2), z(4, 3, 3), z(4, 3), z(5), z(4, 3), z(4, 2), 32, 32, 16,
                                     z(1, 2, 2, dtype=torch.int32), z(0, dtype=torch.int32), packed=True)
    with pytest.raises(ValueError, match="CUDA tensor"):  # CHECK_CUDA: no CPU path exists (SURVEY 0.5)
        ops.fully_fused_projection_2dgs(z(10, 3), z(10, 4), z(10, 3), z(1, 4, 4), z(1, 3, 3), 32, 32, packed=True)


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under gs-sdf_b200/ may import, link or call it."""
    pkg = os.path.join(ROOT, "gs-sdf_b200")
    for dp, _, fs in os.walk(pkg):
        if "build" in dp.split(os.sep):
            continue
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "oracle" not in txt.lower() or f == "scene.py", f"{f} mentions the oracle"
