"""CPU checks of pose-graph reuse: the saved-map format (vins_mono_b200/csrc/pg_map.cpp, compiled with g++ through
tests/hostlib/pg_map_host.cpp, and the numpy twin tests/pose_graph_map_twin.py) on the committed fixture
tests/golden/pose_graph_map/, its rejection of malformed maps, and the restatement with a loaded map on a two-session
run."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle.pose_graph as opg
import pose_graph_map_twin as tw
from harness import pose_graph_synth as pgs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "pose_graph_map") + os.sep
INVALID, CAPACITY = -1, -4
F = r"-?\d+\.\d{6}"
ROW_RE = re.compile(r"^ \d+ " + " ".join([F] * 15) + r" -?\d+ " + " ".join([F] * 8) + r" \d+\n$")


@pytest.fixture(scope="module")
def mod(tmp_path_factory):
    out = tmp_path_factory.mktemp("pgmap") / "libpgmap.so"
    csrc = os.path.join(ROOT, "vins_mono_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I", csrc, "-I", os.path.join(ROOT, "include"),
                           os.path.join(csrc, "pg_map.cpp"), os.path.join(ROOT, "tests", "hostlib", "pg_map_host.cpp"), "-o", str(out)])
    lib = C.CDLL(str(out))
    lib.pgmap_copy.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
    lib.pgmap_read.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    return lib


def copy(mod, src, dst, with_points=1, max_kf=100, max_corners=100):
    msg = C.create_string_buffer(512)
    rc = mod.pgmap_copy(str(src).encode(), str(dst).encode(), with_points, max_kf, max_corners, msg, 512)
    return rc, msg.value.decode()


def read(mod, src, with_points=1, max_kf=100, max_corners=100):
    rows, pts, desc = np.zeros((100, 26)), np.zeros((400, 4), np.float32), np.zeros((400, 4), np.uint64)
    msg = C.create_string_buffer(512)
    n = mod.pgmap_read(str(src).encode(), with_points, max_kf, max_corners, rows.ctypes.data, 100, pts.ctypes.data, desc.ctypes.data, 400,
                       msg, 512)
    assert n >= 0, msg.value
    return rows[:n], pts[:int(rows[:n, 25].sum())], desc[:int(rows[:n, 25].sum())]


def files(prefix, n):
    names = ["pose_graph.txt"] + [f"{i}_{s}" for i in range(n) for s in ("keypoints.txt", "briefdes.dat")]
    return {f: open(prefix + f, "rb").read() for f in names}


def test_fixture_lines_follow_the_reference_format_strings():
    lines = open(FIX + "pose_graph.txt").read().splitlines(keepends=True)
    assert len(lines) == 4 and all(ROW_RE.match(l) for l in lines)
    kfs = tw.read_map(FIX)
    assert [k["n"] for k in kfs] == [3, 0, 2, 1] and [k["loop_index"] for k in kfs] == [-1, -1, 0, -1]
    assert os.path.getsize(FIX + "1_keypoints.txt") == 0 and os.path.getsize(FIX + "1_briefdes.dat") == 0
    for i in range(4):
        for l in open(FIX + f"{i}_keypoints.txt").read().splitlines(keepends=True):
            assert re.match(r"^" + " ".join([F] * 4) + r"\n$", l)
    # bit order: bit 255 is the first character, bit 0 the last
    d0 = open(FIX + "0_briefdes.dat").read().split("\n")[0]
    assert d0[0] == "1" and d0[255] == "1" and int(kfs[0]["desc"][0, 3]) >> 63 == 1 and int(kfs[0]["desc"][0, 0]) & 1 == 1
    d1 = open(FIX + "0_briefdes.dat").read().split("\n")[1]
    assert d1 == "01" + "0" * 254 and kfs[0]["desc"][1].tolist() == [0, 0, 0, 1 << 62]


def test_twin_and_module_write_the_fixture_back_byte_for_byte(mod, tmp_path):
    want = files(FIX, 4)
    a = tw.scratch_prefix(str(tmp_path), "twin")
    kfs = tw.read_map(FIX)
    tw.write_map(a, [dict(k, kp=k["kp"], kpn=k["kpn"], desc=k["desc"]) for k in kfs])
    assert files(a, 4) == want
    b = tw.scratch_prefix(str(tmp_path), "module")
    rc, msg = copy(mod, FIX, b)
    assert rc == 4, msg
    assert files(b, 4) == want


def test_module_and_twin_read_the_same_values(mod, tmp_path):
    rows, pts, desc = read(mod, FIX)
    kfs = tw.read_map(FIX)
    for r, k in zip(rows, kfs):
        assert r[0] == k["index"] and r[1] == k["stamp"] and r[16] == k["loop_index"] and r[25] == k["n"]
        assert np.array_equal(r[2:5], k["vio_T"]) and np.array_equal(r[5:8], k["pg_T"])
        assert np.array_equal(r[8:12], k["vio_Q"]) and np.array_equal(r[12:16], k["pg_Q"]) and np.array_equal(r[17:25], k["loop_info"])
    assert np.array_equal(pts, np.concatenate([np.hstack([k["kp"], k["kpn"]]) for k in kfs]))
    assert np.array_equal(desc, np.concatenate([k["desc"] for k in kfs]))
    # a round trip through the module and then the twin keeps every value
    b = tw.scratch_prefix(str(tmp_path), "rt")
    assert copy(mod, FIX, b)[0] == 4
    again = tw.read_map(b)
    for k, m in zip(kfs, again):
        for key in ("vio_T", "pg_T", "vio_Q", "pg_Q", "loop_info", "kp", "kpn", "desc"):
            assert np.array_equal(k[key], m[key])
    # without points only pose_graph.txt is read; the copy lists no keypoints
    rows2, _, _ = read(mod, FIX, with_points=0)
    assert np.array_equal(rows2, rows)
    c = tw.scratch_prefix(str(tmp_path), "nopts")
    assert copy(mod, FIX, c, with_points=0)[0] == 4
    assert [k["n"] for k in tw.read_map(c)] == [0, 0, 0, 0]


def _broken(tmp_path, name, edit):
    d = tmp_path / name
    shutil.copytree(FIX, d)
    edit(str(d) + os.sep)
    return str(d) + os.sep


def _rewrite(path, fn):
    s = open(path).read()
    open(path, "w").write(fn(s))


CASES = {
    "missing pose_graph.txt": (lambda p: os.remove(p + "pose_graph.txt"), INVALID, "pose_graph.txt"),
    "truncated line": (lambda p: _rewrite(p + "pose_graph.txt", lambda s: s.replace(" 0.000000 0\n", "\n", 1)), INVALID, "pose_graph.txt:2"),
    "unparsable field": (lambda p: _rewrite(p + "pose_graph.txt", lambda s: s.replace("1403636580.350000", "14036x6580.35", 1)), INVALID,
                         "pose_graph.txt:2"),
    "rows out of order": (lambda p: _rewrite(p + "pose_graph.txt", lambda s: s.replace(" 3 1403636581", " 4 1403636581", 1)), INVALID,
                          "pose_graph.txt:4"),
    "loop onto a later key frame": (lambda p: _rewrite(p + "pose_graph.txt", lambda s: s.replace(" 0 0.120000", " 2 0.120000", 1)), INVALID,
                                    "pose_graph.txt:3"),
    "short descriptor line": (lambda p: _rewrite(p + "2_briefdes.dat", lambda s: s[1:]), INVALID, "2_briefdes.dat"),
    "descriptor character": (lambda p: _rewrite(p + "3_briefdes.dat", lambda s: "2" + s[1:]), INVALID, "3_briefdes.dat:1"),
    "fewer keypoints than listed": (lambda p: _rewrite(p + "0_keypoints.txt", lambda s: s.split("\n", 1)[1]), INVALID, "0_keypoints.txt"),
    "more keypoints than listed": (lambda p: _rewrite(p + "3_keypoints.txt", lambda s: s + s), INVALID, "3_keypoints.txt"),
    "more descriptors than listed": (lambda p: _rewrite(p + "3_briefdes.dat", lambda s: s + s), INVALID, "3_briefdes.dat"),
    "missing keypoint file": (lambda p: os.remove(p + "2_keypoints.txt"), INVALID, "2_keypoints.txt"),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_malformed_maps_are_rejected_and_nothing_is_written(mod, tmp_path, case):
    edit, status, where = CASES[case]
    src = _broken(tmp_path, "src", edit)
    dst = tw.scratch_prefix(str(tmp_path), "dst")
    rc, msg = copy(mod, src, dst)
    assert rc == status and where in msg, (rc, msg)
    assert os.listdir(dst) == []


def test_capacities_and_unwritable_destination(mod, tmp_path):
    dst = tw.scratch_prefix(str(tmp_path), "dst")
    rc, msg = copy(mod, FIX, dst, max_kf=3)
    assert rc == CAPACITY and "pose_graph.txt:4" in msg
    rc, msg = copy(mod, FIX, dst, max_corners=2)
    assert rc == CAPACITY and "pose_graph.txt:1" in msg
    assert copy(mod, FIX, dst, with_points=0, max_corners=0)[0] == 4  # keypoint counts are not checked without points
    rc, msg = copy(mod, FIX, str(tmp_path / "no" / "such" / "dir") + os.sep)
    assert rc == INVALID and "pose_graph.txt" in msg


# ---- the restatement with a loaded map
@pytest.fixture(scope="module")
def sessions(tmp_path_factory):
    ev1, ev2, gt1, gt2 = tw.two_sessions()
    g1 = tw.MapOraclePoseGraph()
    pgs.feed(g1, ev1)
    pre = tw.scratch_prefix(str(tmp_path_factory.mktemp("map")))
    tw.write_map(pre, g1.saved())
    return tw.read_map(pre), ev2, gt1, gt2


def test_oracle_two_sessions_merge_onto_the_map(sessions):
    m, ev2, gt1, gt2 = sessions
    n = len(m)
    g = tw.MapOraclePoseGraph()
    g.load(m)
    P0 = np.array([k["P"] for k in g.kfs])
    R0 = [k["R"].copy() for k in g.kfs]
    first = None
    for _, stamp, P, Q, l, li in ev2:
        g.add_keyframe(stamp, P, Q, l, li)
        if l >= 0 and first is None:
            first = len(g.kfs) - 1
            # the first loop onto the map shifts the new session onto it (pose_graph.cpp:96-124)
            kf, old = g.kfs[first], g.kfs[l]
            w_R = old["vio_R"] @ opg.quat_to_R(li[3:7])
            assert abs(opg.R2ypr(kf["vio_R"])[0] - opg.R2ypr(w_R)[0]) < 1e-9
            assert np.linalg.norm(kf["vio_P"] - (old["vio_R"] @ li[:3] + old["vio_P"])) < 0.1
            assert np.linalg.norm(ev2[first - n][2] - kf["vio_P"]) > 1.0 and g.sequence_loop[1] == 1
        if l >= 0:
            g.optimize()
    # the map does not move: P to the last bit, R = ypr2R(R2ypr(R)) over the optimised range
    assert np.array_equal(np.array([k["P"] for k in g.kfs[:n]]), P0)
    for i in range(n):
        want = opg.ypr2R(opg.R2ypr(opg.quat_to_R(opg.R_to_quat(R0[i])))) if i >= g.earliest else R0[i]
        assert np.abs(g.kfs[i]["R"] - want).max() < 1e-14
    P2 = np.array([k["P"] for k in g.kfs[n:]])
    alone = tw.MapOraclePoseGraph()
    tw.feed_session(alone, [(e[0], e[1], e[2], e[3], -1, None) for e in ev2], 0)
    P_alone = np.array([k["P"] for k in alone.kfs])
    assert tw.ate(P2, gt2) < tw.ate(P_alone, gt2)


def test_oracle_loop_between_map_key_frames_is_not_in_the_minimiser(sessions):
    m, ev2, _, _ = sessions
    m2 = [dict(k) for k in m]
    j = max(i for i, k in enumerate(m2) if k["loop_index"] == -1 and i > m2[-1]["index"] // 2 and i > 10)
    m2[j] = dict(m2[j], loop_index=j - 10, loop_info=np.r_[5.0, -3.0, 1.0, 1.0, 0, 0, 0, 25.0])  # far from the map's poses
    runs = []
    for mm in (m, m2):
        g = tw.MapOraclePoseGraph()
        g.load(mm)
        tw.feed_session(g, ev2[:40], len(mm))
        runs.append(g)
    a, b = runs
    assert a.last["cost0"] == b.last["cost0"] and a.last["cost"] == b.last["cost"]
    assert np.array_equal(a.last["x"], b.last["x"]) and a.last["iterations"] == b.last["iterations"]
