"""CPU-only: the pick's layout, its restatement (pick_restatement) against a brute-force loop on hand-made samples, and
the resource use of pick.cu's kernels. The GPU pick is pinned to kernel_render's frame and to this restatement in
test_pick_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import pick_restatement as P
from conftest import ROOT
from simlod_b200 import api
from simlod_b200 import build as B

W, H = 40, 24


def test_pick_info_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    s = api.SimlodPickInfo
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' +
                   'printf("%zu\\n", sizeof(SimlodPickInfo));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodPickInfo, %s));\n' % f for f, _ in s._fields_) + "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert out == [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert C.sizeof(s) == 40 and hasattr(api.load_library(), "simlod_pick") and "simlod_pick" in api.EXPORTS


def test_uniform_offsets_of_the_restatement():
    u = api.Uniforms()
    u.width, u.height, u.showPoints, u.colorByNode, u.colorByLOD, u.useHighQualityShading, u.pointSize = 7.0, 5.0, 1, 2, 3, 4, -6
    u.transform = api.mat4_to_struct(np.arange(16, dtype=np.float32).reshape(4, 4))
    got = P.uniforms_from_bytes(bytes(bytearray(u)))
    assert (got["width"], got["height"], got["showPoints"], got["colorByNode"], got["colorByLOD"], got["useHighQualityShading"],
            got["pointSize"]) == (7.0, 5.0, 1, 2, 3, 4, -6)
    assert (got["transform"] == np.arange(16).reshape(4, 4)).all()


def test_node_color_id():
    # Node::getID(): 'r' -> 1, then 3 bits per child index; % 127. Names of the shallow levels by the plain formula.
    def plain(name):
        ident = 1
        for k, c in enumerate(name[1:], start=1):
            ident |= (c - 48) << (3 * k)
        return ident
    for name in (b"r0", b"r7", b"r01234567", b"r7654321"):
        full = plain(name)
        # the bytes after the name are 0: digit -48 of every later position, as kernel_render reads them
        for k in range(len(name), 19):
            v = ((-48) << (3 * k)) & 0xFFFFFFFF if k <= 9 else ((-48) << (30 + 3 * (k - 10) - (1 if k == 18 else 0))) & ((1 << 64) - 1)
            if k <= 9 and v >= 1 << 31:
                v = (v - (1 << 32)) & ((1 << 64) - 1)
            full |= v
        assert P.node_color_id(name) == full % 127


# ---- hand-made views ---------------------------------------------------------------------------------------------------

def uniforms(transform, **kw):
    u = api.Uniforms()
    u.width, u.height, u.showPoints, u.pointSize = float(W), float(H), 1, 1
    u.transform = api.mat4_to_struct(np.asarray(transform, dtype=np.float32))
    for k, v in kw.items():
        setattr(u, k, v)
    return P.uniforms_from_bytes(bytes(bytearray(u)))


# w = 2z, ndc = (x, y) / 2z: a sample at (x, y, z) lands at pixel ((x/2z + 1) W / 2, (y/2z + 1) H / 2) with depth 2z. A
# huge finite z overflows w to +inf while x and y stay finite (ndc 0: the centre).
PERSPECTIVE = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 2, 0]]


def view(samples, names=(b"r", b"r3")):
    """Two records: the root's voxels (first half of the samples) and a level-1 leaf's points (the rest)."""
    s = np.asarray(samples, dtype=object)
    pts = api.make_points(np.array([r[:3] for r in s], dtype=np.float32), [int(r[3]) for r in s])
    rec = np.zeros(2, dtype=api.EXPORT_NODE_DTYPE)
    half = len(pts) // 2
    rec["level"] = [0, 1]
    rec["name"] = list(names)
    rec["sample_offset"] = [0, half]
    rec["num_voxels"] = [half, 0]
    rec["num_points"] = [0, len(pts) - half]
    return rec, pts


SAMPLES = [
    (0.0, 0.0, 1.0, 0x00AA0000),            # the frame's centre, depth 2
    (0.0, 0.0, 1.0, 0x00AA0000),            # duplicate: the same key, the lower index wins
    (0.0, 0.0, 1.0, 0x00110000),            # same depth, smaller colour: wins the centre
    (0.0, 0.0, 1.5, 0x00000001),            # farther: loses
    (0.5, 0.5, 3e38, 0x00000001),           # depth +inf below the clear colour: a candidate with depth +inf
    (0.5, -0.5, 3e38, 0x00FFFFFF),          # depth +inf at or above it: not a candidate
    (-0.5, 0.5, -2.0, 0x00000005),          # negative depth: its key is above the clear value (and HQS wants depth > 0)
    (-0.5, -0.5, float("nan"), 0x00000005), # NaN depth: not inside
    (1.74, 1.6, 1.0, 0x00000007),           # the last inside pixel (37, 21): pointSize 5 wraps at x == W and drops rows
    (0.5, 0.5, 1.0, 0x00000009),
]


def check(rec, pts, u, expect_hits=None):
    got = P.pick_frame(rec, pts, u, W, H)
    want = P.brute_force(rec, pts, u, W, H)
    assert got.shape == (H, W) and np.array_equal(got, want)
    if expect_hits is not None:
        assert int((got >= 0).sum()) == expect_hits
    return got


def test_restatement_equals_brute_force():
    rec, pts = view(SAMPLES)
    for kw in ({}, {"pointSize": 2}, {"pointSize": 3}, {"pointSize": 5}, {"colorByLOD": 1}, {"colorByNode": 1},
               {"useHighQualityShading": 1}, {"useHighQualityShading": 1, "pointSize": 3}):
        got = check(rec, pts, uniforms(PERSPECTIVE, **kw))
        assert (got >= 0).any(), kw


def test_ties_go_to_the_lower_index():
    rec, pts = view(SAMPLES)
    got = check(rec, pts, uniforms(PERSPECTIVE))
    assert got[H // 2, W // 2] == 2                                     # smaller colour at the same depth
    rec2, pts2 = view(SAMPLES[:2] + SAMPLES[3:])                        # without it: the duplicates tie, index 0 wins
    assert check(rec2, pts2, uniforms(PERSPECTIVE))[H // 2, W // 2] == 0
    # colorByNode: every sample of a record has the same colour, so equal depths tie on the key
    got = check(rec, pts, uniforms(PERSPECTIVE, colorByNode=1))
    assert got[H // 2, W // 2] == 0


def test_depths_at_the_edges():
    rec, pts = view(SAMPLES)
    x, y, w, cand, key = P.sample_keys(rec, pts, uniforms(PERSPECTIVE), W, H)
    assert cand[4] and not cand[5] and not cand[6] and not cand[7]
    assert int(key[4]) >> 32 == 0x7F800000
    hqs = P.sample_keys(rec, pts, uniforms(PERSPECTIVE, useHighQualityShading=1), W, H)[3]
    assert not hqs[4] and not hqs[6] and hqs[0]                          # HQS: depth bits below +inf and depth > 0


def test_point_size_5_wraps_and_drops():
    rec, pts = view(SAMPLES)
    u = uniforms(PERSPECTIVE, pointSize=5)
    x, y, _, _, _ = P.sample_keys(rec, pts, u, W, H)
    assert x[8] + 4 > W and y[8] + 4 > H                                # the corner sample's square crosses both edges
    got = check(rec, pts, u).reshape(-1)
    # clamp(x + ox, 0, W) == W is pixel 0 of the next row, and rows >= H are dropped
    assert got[W * (int(y[8]) + 1)] == 8
    flat = P.pick_frame(rec, pts, u, W, H)
    assert flat.shape == (H, W)


def test_show_points_off():
    rec, pts = view(SAMPLES)
    assert (check(rec, pts, uniforms(PERSPECTIVE, showPoints=0), expect_hits=0) == -1).all()


def test_frame_key():
    rec, pts = view(SAMPLES)
    u = uniforms(PERSPECTIVE)
    got = P.pick_frame(rec, pts, u, W, H)
    k = P.frame_key(rec, pts, u, got)
    assert k[H // 2, W // 2] == (0x40000000 << 32) | 0x00110000         # depth 2.0, colour of sample 2
    assert (k[got < 0] == P.CLEAR).all()


# ---- pick.cu: no kernel uses local memory -----------------------------------------------------------------------------

def test_pick_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "pick.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("pick", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "pick.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_pick_clear", "simlod_pick_key", "simlod_pick_index", "simlod_pick_write"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "pick" in B.PROGRAMS
