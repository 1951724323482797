"""CPU tests of the LAS writer (DESIGN.md §9.13): the ctypes layouts against the C header; the restatement's files
(tests/las_write_restatement.py) read back through the reference's own loader (stored digests where it has not been
built), read_las_header and oracle.decode_las; hand-made quantisation cases; simlod_files_box against the reload()
restatement and insert_files' errors; and the kernel set of las_write.cu."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

import files_restatement as fr
import las_write_restatement as W
import oracle
import reference_golden as golden
from conftest import ROOT
from simlod_b200 import api, data, files_box, read_las_header
from simlod_b200 import build as B
from test_las_files_cpu import insert_files_no_context, las_file

F = np.float32
SIMLOD_ERR_INVALID = -2


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_las_write_structs_match_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    body = ""
    for name, s in (("SimlodLasWriteParams", api.LasWriteParams), ("SimlodLasWriteInfo", api.LasWriteInfo)):
        body += 'printf("%%zu\\n", sizeof(%s));\n' % name
        body += "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, f) for f, _ in s._fields_)
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' + body + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for s in (api.LasWriteParams, api.LasWriteInfo):
        want += [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out == want
    assert C.sizeof(api.LasWriteParams) == 80 and C.sizeof(api.LasWriteInfo) == 96
    lib = api.load_library()
    for name in ("simlod_write_las", "simlod_files_box"):
        assert name in api.EXPORTS and hasattr(lib, name)


def test_python_params_defaults():
    p = api.las_write_params(0.01, None, (1.0, 2.0, 3.0), 4)
    assert tuple(p.scale) == (0.01,) * 3 and tuple(p.offset) == (1.0, 2.0, 3.0) == tuple(p.translation) and p.writer_threads == 4
    p = api.las_write_params((0.5, 0.25, 2.0), (7.0, 8.0, 9.0))
    assert tuple(p.scale) == (0.5, 0.25, 2.0) and tuple(p.offset) == (7.0, 8.0, 9.0) and tuple(p.translation) == (0.0,) * 3
    assert p.writer_threads == 8
    s, o, t = W.params(0.01, None, (1.0, 2.0, 3.0))
    assert list(s) == [0.01] * 3 and list(o) == list(t) == [1.0, 2.0, 3.0]


# ---- the restatement's files, read back ------------------------------------------------------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "las_write_reference.json")
_stored = None


def reference(key, run):
    """What the reference's own loader reads from a restated file: live where oracle/_ref/libref_las.so has been built
    (checked against the stored value, or stored with SIMLOD_RECORD_GOLDEN=1), else the stored value."""
    global _stored
    if _stored is None:
        _stored = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    if oracle.ref_las() is None:
        assert key in _stored, "no stored reference result for %r in %s" % (key, GOLDEN)
        return _stored[key]
    value = json.loads(json.dumps(run()))
    if os.environ.get("SIMLOD_RECORD_GOLDEN"):
        _stored[key] = value
        with open(GOLDEN, "w") as f:
            json.dump(_stored, f, indent=1, sort_keys=True)
    elif key in _stored:
        assert _stored[key] == value, "reference result for %r differs from the stored one" % key
    return value


def all_colours(n):
    """n samples whose colour bytes run through all 256 values on every channel, alpha varied (it is dropped)."""
    k = np.arange(n, dtype=np.uint32)
    return (k & 0xFF) | (((k * 7 + 3) & 0xFF) << 8) | (((k * 13 + 5) & 0xFF) << 16) | ((k * 29 & 0xFF) << 24)


def terrain_samples(n=5000):
    pts = fr.shifted_terrain(n)
    pts["color"] = all_colours(n)
    return pts


# name: (samples, scale, offset, translation)
CASES = {
    "terrain_mm": (lambda: terrain_samples(), 0.001, None, (0.0, 0.0, 0.0)),
    "terrain_translated": (lambda: terrain_samples(), 0.001, (600000.0, 5200000.0, 0.0), (601234.5, 5207890.25, 312.0)),
    "terrain_odd_scale": (lambda: terrain_samples(), (0.003, 0.007, 0.0025), (100.0, -50.0, 3.0), (0.0, 0.0, 0.0)),
}


def write_case(tmp_path, name):
    make, scale, offset, translation = CASES[name]
    pts = make()
    buf, bad = W.file_bytes(pts, scale, offset, translation)
    assert bad is None
    path = str(tmp_path / (name + ".las"))
    open(path, "wb").write(buf)
    return path, pts, W.params(scale, offset, translation)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restated_file_reads_back(tmp_path, name):
    path, pts, (s, o, t) = write_case(tmp_path, name)
    buf = open(path, "rb").read()
    h, rec = W.decode(buf)
    n = len(pts)
    q, valid = W.quantise(pts, s, o, t)
    assert valid.all()
    # header fields as the library's reader (the reference's loadHeader restated) reads them
    got = read_las_header(path).as_dict()
    assert got["version_major"] == 1 and got["version_minor"] == 2 and got["header_size"] == 227
    assert got["offset_to_point_data"] == 227 and got["format"] == 2 and got["bytes_per_point"] == 26 and got["num_points"] == n
    assert got["scale"] == tuple(s) and got["offset"] == tuple(o)
    assert got["min"] == tuple(q.min(axis=0) * s + o) and got["max"] == tuple(q.max(axis=0) * s + o)
    assert h["signature"] == b"LASF" and h["software"] == b"simlod_b200".ljust(32, b"\0") and h["day_year"] == (0, 0)
    assert h["num_vlrs"] == 0 and h["by_return"] == (n, 0, 0, 0, 0) and len(buf) == 227 + 26 * n
    # the bounds bound the records exactly
    back = rec["xyz"].astype(np.float64) * s + o
    assert (back.min(axis=0) == np.array(got["min"])).all() and (back.max(axis=0) == np.array(got["max"])).all()
    # decoded with a translation t' (as insert_files applies one): xyz = float(q * s + (o + t')), colours exact
    t2 = np.array([-1000.0, -2000.0, -50.0])
    dec = oracle.decode_las(np.frombuffer(buf, np.uint8, offset=227), n, 26, 2, s, o, t2)
    want = (q.astype(np.float64) * s + (o + t2)).astype(F)
    for k, ax in enumerate("xyz"):
        assert dec[ax].tobytes() == want[:, k].tobytes(), ax
    assert (dec["color"] == ((pts["color"] & np.uint32(0xFFFFFF)) | np.uint32(0xFF000000))).all()
    for k in range(3):
        assert len(np.unique((pts["color"] >> np.uint32(8 * k)) & np.uint32(0xFF))) == 256
    # the reference's own loader reads the same header and points
    ref = reference("header/" + name, lambda: {k: list(v) if isinstance(v, tuple) else v for k, v in fr.ref_las_header(path).items()})
    assert ref == {"num_points": n, "bytes_per_point": 26, "format": 2, "offset_to_point_data": 227, "scale": list(s),
                   "offset": list(o), "min": list(got["min"]), "max": list(got["max"])}
    want_pts = golden.points(dec)
    assert reference("points/" + name, lambda: golden.points(oracle.ref_las_load(path, 0, n, t2))) == want_pts


# ---- hand-made quantisation cases ----------------------------------------------------------------------------------

def samples_at(x, y=None, z=None, color=0):
    x = np.atleast_1d(np.asarray(x, dtype=F))
    pts = np.zeros(len(x), dtype=W.POINT_DTYPE)
    pts["x"] = x
    pts["y"] = x if y is None else y
    pts["z"] = x if z is None else z
    pts["color"] = color
    return pts


def test_half_way_ties_round_to_even():
    p = samples_at([0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.25, -3.75])
    q, valid = W.quantise(p, np.ones(3), np.zeros(3), np.zeros(3))
    assert valid.all() and list(q[:, 0]) == [0, 2, 2, 0, -2, -2, 3, -4]
    # a tie reached through the translation and offset, and a scale that is not a power of two
    q, _ = W.quantise(samples_at([1.0]), np.full(3, 0.5), np.full(3, 0.25), np.full(3, 0.0))
    assert q[0, 0] == 2                                          # (1 - 0.25) / 0.5 = 1.5 -> 2
    q, _ = W.quantise(samples_at([0.0]), np.full(3, 0.5), np.zeros(3), np.full(3, 1.25))
    assert q[0, 0] == 2                                          # 1.25 / 0.5 = 2.5 -> 2


def test_negative_coordinates():
    p = samples_at([-1.0, -123.456, -0.0004, -0.125, -0.375, -0.625])
    q, valid = W.quantise(p, np.full(3, 0.25), np.zeros(3), np.zeros(3))
    assert valid.all() and list(q[:, 0]) == [-4, -494, 0, 0, -2, -2]      # -493.824, -0.0016, ties -0.5, -1.5, -2.5
    q, _ = W.quantise(p, np.full(3, 0.001), np.zeros(3), np.zeros(3))
    assert (q[:, 0] == np.rint(p["x"].astype(np.float64) / 0.001)).all() and q[0, 0] == -1000


@pytest.mark.parametrize("t,ok", [(2.0 ** 31 - 1, True), (2.0 ** 31, False), (-(2.0 ** 31 - 1), True), (-(2.0 ** 31), True),
                                  (-(2.0 ** 31) - 1, False)])
def test_int32_range_edges(t, ok):
    p = samples_at([0.0, 0.0])
    q, valid = W.quantise(p, np.ones(3), np.zeros(3), np.array([t, 0.0, 0.0]))
    assert valid.all() == ok
    buf, bad = W.file_bytes(p, 1.0, (0.0, 0.0, 0.0), (t, 0.0, 0.0))
    if ok:
        assert bad is None and W.decode(buf)[1]["xyz"][0, 0] == int(t)
    else:
        assert buf is None and bad == 0


def test_non_finite_coordinates_are_invalid():
    p = samples_at([1.0, 2.0, 3.0, 4.0, 5.0])
    p["y"][2] = np.inf
    p["z"][3] = np.nan
    p["x"][4] = -np.inf
    _, valid = W.quantise(p, np.ones(3), np.zeros(3), np.zeros(3))
    assert list(valid) == [True, True, False, False, False]
    assert W.file_bytes(p, 1.0) == (None, 2)


def test_empty_file():
    buf, bad = W.file_bytes(np.zeros(0, dtype=W.POINT_DTYPE), 0.01, (1.0, 2.0, 3.0))
    h, rec = W.decode(buf)
    assert bad is None and len(buf) == 227 and len(rec) == 0 and h["num_points"] == 0 and h["by_return"] == (0,) * 5
    assert h["min"] == (0.0,) * 3 and h["max"] == (0.0,) * 3 and h["offset"] == (1.0, 2.0, 3.0)


def test_a_scale_that_is_not_a_power_of_two():
    p = samples_at(np.linspace(-10.0, 10.0, 101, dtype=F), color=0x00FF8001)
    s = np.array([0.003, 0.01, 0.1])
    q, valid = W.quantise(p, s, np.zeros(3), np.zeros(3))
    with np.errstate(all="ignore"):
        want = np.rint(np.stack([p["x"], p["y"], p["z"]], axis=1).astype(np.float64) / s)
    assert valid.all() and (q == want).all()
    buf, _ = W.file_bytes(p, s, (0.0, 0.0, 0.0))
    h, rec = W.decode(buf)
    assert h["max"] == tuple(q.max(axis=0) * s) and h["min"] == tuple(q.min(axis=0) * s)
    assert (rec["rgb"] == np.array([257, 128 * 257, 255 * 257])).all() and (rec["flags"] == 9).all()


# ---- simlod_files_box ------------------------------------------------------------------------------------------------

def test_files_box_is_the_reload_box(tmp_path):
    a = las_file(tmp_path / "a.las", 2000, scale=(0.001, 0.001, 0.001), offset=(1000.0, 2000.0, 0.0))
    b = las_file(tmp_path / "b.las", 10)
    s = str(tmp_path / "c.simlod")
    data.write_simlod(s, fr.shifted_terrain(10), (-5.0, 7.0, 1.0), (8000.0, 9000.0, 400.0))
    e = str(tmp_path / "e.las")
    data.write_las(e, np.zeros(0, dtype=oracle.POINT_DTYPE), fmt=0)
    for paths in ([a], [b, a], [a, s], [e, a, s, b], [s]):
        mn, mx = files_box(paths)
        want_mn, want_mx, _, _ = fr.reload(paths)
        assert mn.tobytes() == want_mn.tobytes() and mx.tobytes() == want_mx.tobytes(), paths


def test_files_box_refuses_what_insert_files_refuses(tmp_path):
    good = las_file(tmp_path / "good.las")
    lib = api.load_library()

    def box_rc(paths):
        arr = (C.c_char_p * max(1, len(paths)))(*[os.fsencode(str(p)) for p in paths])
        mn, mx = (C.c_float * 3)(), (C.c_float * 3)()
        rc = lib.simlod_files_box(arr, len(paths), mn, mx)
        return rc, lib.simlod_last_error().decode()
    missing = str(tmp_path / "missing.las")
    laz = tmp_path / "scan.laz"
    laz.write_bytes(open(good, "rb").read())
    other = tmp_path / "scan.xyz"
    other.write_bytes(b"1 2 3\n")
    short = tmp_path / "short.simlod"
    short.write_bytes(b"\0" * 23)
    for paths in ([], [missing], [good, str(laz)], [str(other), good], [good, str(short)]):
        rc, msg = box_rc(paths)
        assert (rc, msg) == insert_files_no_context(paths) and rc == SIMLOD_ERR_INVALID, (paths, msg)
    with pytest.raises(api.SimlodError) as e:
        files_box([good, missing])
    assert e.value.code == SIMLOD_ERR_INVALID and missing in str(e.value)


# ---- las_write.cu: the exact set of kernels, none using local memory ---------------------------------------------------

def test_las_write_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "las_write.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("las_write", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "las_write.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_las_encode"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    sass = subprocess.run([os.path.join(B.CUDA, "bin", "cuobjdump"), "-sass", cubin], stdout=subprocess.PIPE, text=True).stdout
    assert "LDL" not in sass and "STL" not in sass
    assert "UBLKCP.G.S" in sass                              # the full tiles' shared -> global bulk store
    assert "las_write" in B.PROGRAMS
