"""The C declarations of libl3d_b200.so against what it exports and what Python assumes (include/l3d_capi.h, include/l3dpp_capi.h): both
headers compile as C and C++, the library exports exactly the declared functions, every struct mirror in Python has the C layout, and the
prototypes capi.lib() binds from the headers reject a wrongly typed argument.  No GPU needed."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from line3dpp_b200 import build, capi, line3d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")

# every struct the two headers pass, and its Python mirror (ctypes.Structure or numpy dtype)
MIRRORS = {"l3d_view_desc": capi.ViewDesc, "l3d_undistort_desc": capi.UndistortDesc, "l3d_image_prep_desc": capi.ImagePrepDesc,
           "l3d_match_rec": capi.REC_DT, "l3d_match": capi.MATCH_DT, "l3dpp_stats_block": line3d.Stats, "l3dpp_seg3d": line3d.SEG3D_DT,
           "l3dpp_residual": line3d.RESID_DT, "l3dpp_bin_line": line3d.LINE_DT, "l3dpp_bin_seg": line3d.BIN_SEG_DT,
           "l3dpp_bin_res": line3d.RESID_DT}


def _declared():
    return {n for h in capi.HEADERS for n in capi.declarations(h)}


def _tool(name):
    path = shutil.which(name)
    if path is None:
        pytest.skip(f"no {name}")
    return path


@pytest.mark.parametrize("lang", ["c", "c++"])
@pytest.mark.parametrize("header", ["l3d_capi.h", "l3dpp_capi.h"])
def test_header_compiles(lang, header):
    cc = _tool("gcc" if lang == "c" else "g++")
    std = "-std=c99" if lang == "c" else "-std=c++17"
    r = subprocess.run([cc, "-fsyntax-only", "-x", lang, std, "-Wall", "-Wextra", "-pedantic", "-Werror", os.path.join(INCLUDE, header)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_exports_exactly_the_declared_functions():
    r = subprocess.run([_tool("nm"), "-D", "--defined-only", build.build()], capture_output=True, text=True, check=True)
    exported = {f[2] for f in (line.split() for line in r.stdout.splitlines())
                if len(f) == 3 and f[1] == "T" and re.fullmatch(r"l3d(pp)?_\w+", f[2])}
    declared = _declared()
    assert len(declared) > 100
    assert exported == declared, (sorted(exported - declared), sorted(declared - exported))


def _layout(mirror):
    """[(C field name, offset, size)] and the size of a ctypes.Structure or numpy dtype"""
    if isinstance(mirror, np.dtype):
        fields = [(n, mirror.fields[n][1], mirror.fields[n][0].itemsize) for n in mirror.names]
        size = mirror.itemsize
    else:
        fields = [(n, getattr(mirror, n).offset, getattr(mirror, n).size) for n, _ in mirror._fields_]
        size = ctypes.sizeof(mirror)
    return [(n.lstrip("_"), o, s) for n, o, s in fields], size


def test_struct_mirrors_match_the_headers(tmp_path):
    lines = []
    for name, mirror in MIRRORS.items():
        fields, _ = _layout(mirror)
        lines.append(f'    printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'    printf("{name}.{f} %zu %zu\\n", offsetof({name}, {f}), sizeof((({name}*)0)->{f}));' for f, _, _ in fields]
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "l3d_capi.h"\n#include "l3dpp_capi.h"\nint main(void)\n{\n'
                   + "\n".join(lines) + "\n    return 0;\n}\n")
    exe = tmp_path / "layout"
    r = subprocess.run([_tool("gcc"), "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    c = dict((w[0], tuple(int(x) for x in w[1:])) for w in (line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines()))
    for name, mirror in MIRRORS.items():
        fields, size = _layout(mirror)
        assert c[name] == (size,), name
        for f, off, sz in fields:
            assert c[f"{name}.{f}"] == (off, sz), (name, f)


def test_bound_prototypes_reject_a_wrong_argument_type():
    """in a fresh interpreter: loading the library binds every declared function, so a float for an unsigned int raises before the call,
    and a 64-bit count is returned whole whatever was called before"""
    code = ("import ctypes\n"
            "from line3dpp_b200 import capi\n"
            "L = capi.lib()\n"
            "assert L.l3d_get_view_matches.restype is ctypes.c_longlong and L.l3dpp_segcache_count.restype is ctypes.c_longlong\n"
            "out = (ctypes.c_uint * 4)()\n"
            "assert L.l3dpp_sequential_neighbors(3, 10, 4, out, 4) == 4\n"
            "try:\n"
            "    L.l3dpp_sequential_neighbors(3.0, 10, 4, out, 4)\n"
            "except ctypes.ArgumentError as e:\n"
            "    print('ArgumentError', e)\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("ArgumentError argument 1"), r.stdout


def test_sfm_open_rejects_an_unknown_kind(tmp_path):
    defines = dict(re.findall(r"#define L3DPP_SFM_(\w+) (\d+)", open(os.path.join(INCLUDE, "l3dpp_capi.h")).read()))
    assert {k: int(v) for k, v in defines.items()} == {k[4:]: v for k, v in vars(line3d).items() if k.startswith("SFM_")}
    err = ctypes.create_string_buffer(256)
    for kind in (-1, 6, 99):
        assert capi.lib().l3dpp_sfm_open(kind, str(tmp_path).encode(), b"", err, 256) is None
        assert err.value.decode() == f"unknown model kind {kind}"
    with pytest.raises(capi.L3DError, match="unknown model kind 7"):
        line3d._read_sfm(7, tmp_path)
