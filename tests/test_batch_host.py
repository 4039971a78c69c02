"""Host-side check of the batch skeleton every batched handle family shares (csrc/batch_host.h), compiled with g++ over a
dummy member type: the member(k) bounds, the last-error rule (the member's own text, else its batch's), the "member k:"
roll-up of the first failing member, the refusal of a per-handle call on a member of an explicit batch, and that
destroying a member destroys its batch only when the batch is stand-alone.  The library's three families answer a NULL
handle through it the same way."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECKS = ["member_bounds", "last_error", "roll_up", "refuse_member", "standalone", "kernel_times"]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("batchhost") / "libbatchhost.so"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           "-I", os.path.join(ROOT, "vins_mono_b200", "csrc"),
                           os.path.join(ROOT, "tests", "hostlib", "batch_host_check.cpp"), "-o", str(out)])
    return ctypes.CDLL(str(out))


@pytest.mark.parametrize("name", CHECKS)
def test_batch_skeleton(lib, name):
    fn = getattr(lib, "check_" + name)
    fn.argtypes = [ctypes.c_char_p, ctypes.c_int]
    msg = ctypes.create_string_buffer(256)
    assert fn(msg, len(msg)) == 0, msg.value.decode()


@pytest.mark.parametrize("family", ["vt", "ve", "vp"])
def test_null_handles_name_what_is_missing(family):
    from vins_mono_b200 import load_library
    lib = load_library()
    assert getattr(lib, family + "_last_error")(None) == b"null handle"
    assert getattr(lib, family + "_batch_last_error")(None) == b"null batch"
    assert getattr(lib, family + "_batch_member")(None, 0) is None
    assert getattr(lib, family + "_batch_size")(None) == -1
