"""CPU checks of the ctypes side of the C ABI (vins_mono_b200/_abi.py) against include/vinsb200/*.h: one signature entry per
declared function with the prototype's arity and parameter / return kinds, struct mirrors with the C sizes and offsets,
and no signature assigned anywhere else in the package.  ctypes itself checks none of this: a double passed where an int
is declared arrives as garbage, and a pointer returned through the default int restype is cut to 32 bits."""
import ctypes as C
import os
import re
import subprocess

from test_abi import declared_functions

from vins_mono_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include", "vinsb200")
PROTO = re.compile(r"^[ \t]*((?:const\s+)?\w+\s*\**)\s*\b(v[terp]_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", re.M)
STRUCTS = {"vt_config": _abi.TrackerConfig, "ve_config": _abi.EstimatorConfig, "vp_config": _abi.PoseGraphConfig,
           "vp_loop_config": _abi.LoopConfig, "vp_loop_result": _abi.LoopResult, "vr_sequence": _abi.ReplaySequence}


def prototypes():
    """name -> (return type, [parameter types]) of every function declared in the headers."""
    out = {}
    for f in sorted(os.listdir(INC)):
        src = re.sub(r"/\*.*?\*/", "", open(os.path.join(INC, f)).read(), flags=re.S)
        for ret, name, params in PROTO.findall(src):
            params = [] if params.strip() in ("", "void") else [re.sub(r"\s*\b\w+\s*$", "", p) for p in params.split(",")]
            out[name] = (ret, params)
    return out


def c_kind(t):
    t = " ".join(t.replace("const", " ").replace("*", " * ").split())
    return "char*" if t == "char *" else "pointer" if "*" in t else t


def ctypes_kind(t):
    if t is None:
        return "void"
    if t is C.c_char_p:
        return "char*"
    if t is C.c_void_p or issubclass(t, C._Pointer):
        return "pointer"
    return {C.c_int: "int", C.c_size_t: "size_t", C.c_longlong: "long long", C.c_double: "double", C.c_float: "float"}[t]


def test_table_covers_exactly_the_declared_functions():
    protos = prototypes()
    assert sorted(protos) == declared_functions()
    assert sorted(_abi.SIGNATURES) == sorted(protos)


def test_signatures_match_the_prototypes():
    bad = []
    for name, (ret, params) in prototypes().items():
        restype, argtypes = _abi.SIGNATURES[name]
        want = (c_kind(ret), [c_kind(p) for p in params])
        got = (ctypes_kind(restype), [ctypes_kind(a) for a in argtypes])
        if want != got:
            bad.append(f"{name}: header {want}, table {got}")
    assert not bad, "\n".join(bad)


def test_struct_mirrors_match_the_headers(tmp_path):
    lines = []
    for cname, mirror in STRUCTS.items():
        lines.append(f'    std::printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for field, _ in mirror._fields_:
            lines.append(f'    std::printf("{cname} {field} %zu %zu\\n", offsetof({cname}, {field}), sizeof((({cname}*)0)->{field}));')
    src = tmp_path / "struct_layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "vinsb200/loop_camera.h"\n#include "vinsb200/replay.h"\n'
                   "int main() {\n" + "\n".join(lines) + "\n}\n")
    exe = tmp_path / "struct_layout"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    want = []
    for cname, mirror in STRUCTS.items():
        want.append(f"{cname} sizeof {C.sizeof(mirror)}")
        want += [f"{cname} {field} {getattr(mirror, field).offset} {getattr(mirror, field).size}" for field, _ in mirror._fields_]
    assert got == want


def test_signatures_are_assigned_only_in_the_abi_module():
    pkg = os.path.join(ROOT, "vins_mono_b200")
    hits = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith(".py") and path != os.path.join(pkg, "_abi.py"):
                hits += [f"{path}:{i}" for i, line in enumerate(open(path), 1) if re.search(r"\.(argtypes|restype)\s*=", line)]
    assert not hits, hits
