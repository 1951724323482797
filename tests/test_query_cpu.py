"""CPU-only: the region query's layouts, its restatement (query_restatement) on an oracle-built octree against a
brute-force filter of the source points, and the resource use of query.cu's kernels. The GPU query is pinned byte for
byte to this restatement in test_query_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import oracle
import query_restatement as Q
from conftest import ROOT
from simlod_b200 import Region, api, data
from simlod_b200 import build as B
from test_export_cpu import sorted_points


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_region_structs_match_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    structs = (("SimlodRegion", api.SimlodRegion), ("SimlodQueryInfo", api.SimlodQueryInfo))
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' +
                   "".join('printf("%%zu\\n", sizeof(%s));\n' % n + "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (n, f) for f, _ in s._fields_)
                           for n, s in structs) +
                   'printf("%d %d %d %d\\n", SIMLOD_REGION_BOX, SIMLOD_REGION_SPHERE, SIMLOD_REGION_PLANES, SIMLOD_REGION_MAX_PLANES);return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for _, s in structs:
        want += [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out[:-4] == want
    assert out[-4:] == [api.REGION_BOX, api.REGION_SPHERE, api.REGION_PLANES, api.REGION_MAX_PLANES] == [Q.BOX, Q.SPHERE, Q.PLANES, 16]
    assert C.sizeof(api.SimlodRegion) == 304 and C.sizeof(api.SimlodQueryInfo) == 40
    assert hasattr(api.load_library(), "simlod_query_region")


def test_region_constructors():
    r = Region.planes([[1, 0, 0, -2], [0, -1, 0, 5]])
    assert (r.kind, r.num_planes) == (api.REGION_PLANES, 2) and list(r.planes[1]) == [0.0, -1.0, 0.0, 5.0]
    b = Region.box((1, 2, 3), (4, 5, 6))
    assert b.kind == api.REGION_BOX and list(b.box_min) == [1.0, 2.0, 3.0] and list(b.box_max) == [4.0, 5.0, 6.0]
    s = Region.sphere((1, 2, 3), 0.5)
    assert s.kind == api.REGION_SPHERE and list(s.center) == [1.0, 2.0, 3.0] and s.radius == 0.5
    for bad in (np.zeros((0, 4)), np.zeros((17, 4)), np.zeros((3, 3))):
        with pytest.raises(ValueError):
            Region.planes(bad)


# ---- the predicates --------------------------------------------------------------------------------------------------

def pts(*rows):
    return api.make_points(np.array([r[:3] for r in rows], dtype=np.float32), [r[3] for r in rows])


def test_boundaries_are_inside():
    p = pts((1, 2, 3, 0), (4, 5, 6, 1), (4.0000005, 5, 6, 2), (0.9999999, 2, 3, 3))
    assert Q.contains(Region.box((1, 2, 3), (4, 5, 6)), p).tolist() == [True, True, False, False]
    p = pts((105, 100, 100, 0), (100, 100, 95, 1), (103, 104, 100, 2), (103, 104, 100.001, 3))
    assert Q.contains(Region.sphere((100, 100, 100), 5), p).tolist() == [True, True, True, False]
    assert Q.contains(Region.sphere((105, 100, 100), 0), p).tolist() == [True, False, False, False]
    p = pts((40, 0, 0, 0), (39.99999, 0, 0, 1), (40, 7, 0, 2), (40, 7.000001, 0, 3))
    assert Q.contains(Region.planes([[1, 0, 0, -40], [0, -1, 0, 7]]), p).tolist() == [True, False, True, False]


def test_in_cube_is_the_builders_half_open_cube():
    mn, mx = (0.0, 0.0, 0.0), (256.0, 100.0, 50.0)
    p = pts((0, 0, 0, 0), (256, 1, 1, 1), (255.99998, 99, 49, 2), (-1e-6, 1, 1, 3), (1, 255.9999, 1, 4), (1, 1, 256, 5), (float("nan"), 1, 1, 6))
    assert Q.in_cube(p, mn, mx).tolist() == [True, False, True, False, True, False, False]
    with pytest.raises(AssertionError):
        Q.in_cube(p, mn, (300.0, 1.0, 1.0))                  # not a power of two: the device's reciprocal is needed
    assert Q.in_cube(p, mn, (300.0, 1.0, 1.0), rcp=np.float32(1.0) / np.float32(300.0))[0]


# ---- the restatement on an oracle-built octree against brute force ---------------------------------------------------

MARK = 0xABCD0000          # colours of the hand-placed points


@pytest.fixture(scope="module")
def tree():
    cloud, mn, mx = data.uniform_cube(400_000, size=256.0, seed=3)
    placed = pts((256.0, 10.0, 10.0, MARK),                 # exactly on the max face: filed under X = 0, never returned
                 (10.0, 20.0, 30.0, MARK + 1), (50.0, 60.0, 70.0, MARK + 2),      # the corners of REGIONS["box_part"]
                 (105.0, 100.0, 100.0, MARK + 3),            # on the sphere
                 (40.0, 200.0, 200.0, MARK + 4))             # on the first plane of the corridor
    points = np.concatenate([cloud[:200_000], placed, cloud[200_000:]])
    box = (mn, (256.0, 256.0, 256.0))
    o = oracle.Oracle(*box)
    for b in np.array_split(points, 3):
        o.add_batch(b)
    canon = o.canon()
    assert int(canon.records["level"].max()) >= 2
    return points, box, canon


REGIONS = {
    "box_part": Region.box((10, 20, 30), (50, 60, 70)),
    "box_everything": Region.box((-1, -1, -1), (257, 257, 257)),
    "box_disjoint": Region.box((300, 0, 0), (400, 256, 256)),
    "sphere": Region.sphere((100, 100, 100), 5),
    "corridor": Region.planes([[1, 0, 0, -40], [-1, 0, 0, 44], [0.6, 0.8, 0, -100], [-0.6, -0.8, 0, 300], [0, 0, 1, -8], [0, 0, -1, 250]]),
}
EXPECT_MARKS = {"box_part": {1, 2}, "box_everything": {1, 2, 3, 4}, "box_disjoint": set(), "sphere": {3}, "corridor": {4}}


@pytest.mark.parametrize("name", list(REGIONS))
def test_restatement_equals_brute_force(tree, name):
    points, box, canon = tree
    region = REGIONS[name]
    want = Q.brute_force(points, region, *box)
    got, n_points, n_voxels = Q.query_export(R.export_canon(canon), region, None, *box)
    assert n_voxels == 0 and n_points == len(got) == len(want)
    assert np.array_equal(sorted_points(got), sorted_points(want))
    marks = {int(c) - MARK for c in got["color"] if MARK <= int(c) < MARK + 16}
    assert marks == EXPECT_MARKS[name]
    if name == "box_everything":                             # all but the point on the max face, which the box contains
        assert len(got) == len(points) - 1 and Q.contains(region, points).all()
    if name == "box_disjoint":
        assert len(got) == 0
    # at or below the deepest level the cut is the point set; above it, the voxels of the cut are filtered by position alone
    top = int(canon.records["level"].max())
    deep, dp, dv = Q.query_export(R.export_canon(canon, top), region, top, *box)
    assert dv == 0 and np.array_equal(sorted_points(deep), sorted_points(want))
    cn, cs, _ = cut = R.export_canon(canon, 1)
    coarse, cp, cv = Q.query_export(cut, region, 1, *box)
    vox = np.zeros(len(cs), dtype=bool)
    for r in range(len(cn)):
        a, p, v = int(cn["sample_offset"][r]), int(cn["num_points"][r]), int(cn["num_voxels"][r])
        vox[a + p:a + p + v] = True
    inside = Q.contains(region, cs)
    assert cv == int((inside & vox).sum()) and cp == int((inside & ~vox & Q.in_cube(cs, *box)).sum()) and cp + cv == len(coarse)


def test_image_restatement_keeps_the_exports_order():
    from test_export_view_cpu import Tree
    t = Tree()
    for depth in (None, 0, 2, 3):
        region = Region.box((0.25, 0, 0), (0.75, 0, 0))      # the hand-made samples have x in [0, 1), y = z = 0
        nodes, samples, _ = R.export_image(*t.image(), depth)
        got, n_p, n_v = Q.query_image(*t.image(), region, depth, (0, 0, 0), (1, 1, 1))
        keep = (samples["x"] >= 0.25) & (samples["x"] <= 0.75)
        if depth is None:                                    # the points of the leaves only
            for r in range(len(nodes)):
                a, p, v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
                keep[a + p:a + p + v] = False
                if not nodes["flags"][r] & R.LEAF:
                    keep[a:a + p] = False
            assert n_v == 0
        assert got.tobytes() == samples[keep].tobytes() and n_p + n_v == len(got) > 0


# ---- query.cu: no kernel uses local memory ----------------------------------------------------------------------------

def test_query_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "query.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("query", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "query.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_query_plan", "simlod_query_count", "simlod_query_scan", "simlod_query_write"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "query" in B.PROGRAMS
