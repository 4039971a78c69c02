"""CPU checks of the batched key-frame attach's ABI (include/vinsb200/loop_attach.h): the ctypes mirror of vp_attach_job
has the C struct's size and offsets, the header declares the one entry the library exports, and the packed stage's job
table keeps every staging block 16-byte aligned."""
import ctypes as C
import os
import re
import subprocess

from vins_mono_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_attach_job_mirror_matches_the_header(tmp_path):
    mirror = _abi.AttachJob
    lines = ['    std::printf("sizeof %zu\\n", sizeof(vp_attach_job));']
    for field, _ in mirror._fields_:
        lines.append(f'    std::printf("{field} %zu %zu\\n", offsetof(vp_attach_job, {field}), sizeof(((vp_attach_job*)0)->{field}));')
    src = tmp_path / "attach_job.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "vinsb200/loop_attach.h"\nint main() {\n' + "\n".join(lines) + "\n}\n")
    exe = tmp_path / "attach_job"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    want = [f"sizeof {C.sizeof(mirror)}"] + [f"{f} {getattr(mirror, f).offset} {getattr(mirror, f).size}" for f, _ in mirror._fields_]
    assert got == want


def test_header_declares_the_batched_attach():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vinsb200", "loop_attach.h")).read(), flags=re.S)
    assert sorted(set(re.findall(r"\b(vp_[a-z0-9_]+)\s*\(", src))) == ["vp_batch_attach_keyframes"]
    assert _abi.SIGNATURES["vp_batch_attach_keyframes"] == (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p])


def test_attach_job_table_keeps_blocks_aligned(tmp_path):
    src = tmp_path / "jobs.cpp"
    src.write_text('#include <cstdio>\n#include "lv_layout.h"\nint main() {\n'
                   "    for (int n = 1; n <= 70; n++)\n"
                   '        std::printf("%d %zu\\n", n, vb::lv_attach_jobs_bytes(n));\n}\n')
    exe = tmp_path / "jobs"
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "vins_mono_b200", "csrc"), str(src),
                           "-o", str(exe)])
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        n, b = map(int, line.split())
        assert b % 16 == 0 and 8 * n <= b < 8 * n + 16, (n, b)
