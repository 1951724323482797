"""CPU-only: the height map's layouts, its restatement (heightmap_restatement) against a plain per-sample loop on
hand-made sample sets and on oracle-built octrees, and the resource use of heightmap.cu's kernels. The GPU query is
pinned byte for byte to this restatement in test_heightmap_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import heightmap_restatement as H
import oracle
import query_restatement as Q
from conftest import ROOT
from simlod_b200 import api, data
from simlod_b200 import build as B

F = np.float32


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_heightmap_layouts_match_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    body = ""
    for name, s in (("SimlodHeightmap", api.SimlodHeightmap), ("SimlodHeightmapInfo", api.SimlodHeightmapInfo)):
        body += 'printf("%%zu\\n", sizeof(%s));\n' % name
        body += "".join('printf("%%zu\\n", offsetof(%s, %s));\n' % (name, f) for f, _ in s._fields_)
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' + body +
                   'printf("%u\\n", SIMLOD_HEIGHTMAP_MAX_CELLS);return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for s in (api.SimlodHeightmap, api.SimlodHeightmapInfo):
        want += [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out[:-1] == want
    assert out[-1] == api.HEIGHTMAP_MAX_CELLS == 1 << 27
    assert C.sizeof(api.SimlodHeightmap) == 24 and C.sizeof(api.SimlodHeightmapInfo) == 56
    assert api.SimlodHeightmapInfo.plan_ms.offset == 44
    assert "simlod_query_heightmap" in api.EXPORTS and hasattr(api.load_library(), "simlod_query_heightmap")


# ---- a plain loop, stated without the restatement's helpers -------------------------------------------------------------

def sample_set(export, depth, box_min, box_max, rcp=None):
    """(index, is voxel) of every sample of the set, in index order."""
    nodes, samples, _ = export
    eligible = Q.in_cube(samples, box_min, box_max, rcp)
    out = []
    for r in range(len(nodes)):
        a, n_p, n_v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
        if depth is not None or nodes["flags"][r] & R.LEAF:
            out += [i for i in range(a, a + n_p) if eligible[i]]
        if depth is not None:
            out += list(range(a + n_p, a + n_p + n_v))
    return sorted(out)


def plain(export, depth, box_min, box_max, origin, cell, shape, rcp=None):
    """Per sample in Python: the float32 cell, then per cell the count, the extremes by sign-aware bits, the top index
    and the fixed-point mean. Returns {cell id: (count, z_min bits, z_max bits, z_mean bits, top)}."""
    _, samples, _ = export
    ny, nx = shape
    size = float(max(F(box_max[a]) - F(box_min[a]) for a in range(3)))
    minz, K = float(F(box_min[2])), 2.0 ** 30 / size
    ox, oy, c = F(origin[0]), F(origin[1]), F(cell)
    cells = {}
    for i in sample_set(export, depth, box_min, box_max, rcp):
        x, y, z = F(samples["x"][i]), F(samples["y"][i]), F(samples["z"][i])
        with np.errstate(all="ignore"):
            u, v = (x - ox) / c, (y - oy) / c
        if not (u >= 0 and v >= 0) or not (np.trunc(u) < nx and np.trunc(v) < ny):
            continue
        key = int(np.trunc(v)) * nx + int(np.trunc(u))
        bits = int(np.asarray(z, dtype=F).view(np.uint32))
        o = bits ^ 0xFFFFFFFF if bits >> 31 else bits | 0x80000000
        q = round((float(z) - minz) * K)                       # Python's round: half to even
        e = cells.setdefault(key, [0, None, None, None, 0])
        e[0] += 1
        e[1] = o if e[1] is None else min(e[1], o)
        if e[2] is None or o > e[2][0] or (o == e[2][0] and i < e[2][1]):
            e[2] = (o, i)
        e[4] += q
    out = {}
    for key, (n, lo, (hi, top), _, S) in cells.items():
        back = [w ^ 0x80000000 if w >> 31 else w ^ 0xFFFFFFFF for w in (lo, hi)]
        mean = F(minz + (float(S) / float(n)) / K)
        out[key] = (n, back[0], back[1], int(np.asarray(mean).view(np.uint32)), top)
    return out


def check(export, depth, box, origin, cell, shape, rcp=None):
    """The restatement's sparse and dense forms against the plain loop; returns the dense results."""
    want = plain(export, depth, *box, origin, cell, shape, rcp)
    ids, count, z_min, z_max, z_mean, top = H.binned(export, depth, *box, origin, cell, shape, rcp)
    got = {int(k): (int(n), int(a.view(np.uint32)), int(b.view(np.uint32)), int(m.view(np.uint32)), int(t))
           for k, n, a, b, m, t in zip(ids, count, z_min, z_max, z_mean, top)}
    assert got == want
    if shape[0] * shape[1] > 1 << 20:
        return None
    dense = H.heightmap(export, depth, *box, origin, cell, shape, rcp)
    flat = [a.reshape(-1) for a in dense]
    empty = np.ones(shape[0] * shape[1], dtype=bool)
    empty[list(want)] = False
    assert (flat[0][empty] == 0).all() and (flat[4][empty] == -1).all()
    for z in flat[1:4]:
        assert (z[empty].view(np.uint32) == H.NAN_BITS).all()
    assert not flat[5][empty].tobytes().strip(b"\0")
    for k, (n, lo, hi, mean, t) in want.items():
        assert (flat[0][k], flat[4][k]) == (n, t)
        assert [int(flat[a][k:k + 1].view(np.uint32)[0]) for a in (1, 2, 3)] == [lo, hi, mean]
        assert flat[5][k].tobytes() == export[1][t].tobytes()
    return dense


BOX = ((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))


def one_record(points, voxels=(), leaf=True):
    """An export with the root as its only record: `points` then `voxels`, in this order."""
    xyz = np.asarray(list(points) + list(voxels), dtype=F).reshape(-1, 3)
    samples = api.make_points(xyz, np.arange(len(xyz), dtype=np.uint32)).view(R.POINT_DTYPE)
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["flags"] = (R.LEAF if leaf else 0) | R.SAMPLED
    nodes["parent"], nodes["first_child"] = -1, -1
    nodes["num_points"], nodes["num_voxels"] = len(points), len(voxels)
    return nodes, samples, R.ExportInfo(1, 0, len(samples), len(points), len(voxels))


def test_cell_borders_and_the_far_edge():
    below = float(np.nextafter(F(4.0), F(0.0)))
    xyz = [[0, 0, 1], [1, 1, 2], [2, 0, 3], [1.999999, 0.5, 4], [4.0, 4.0, 5], [below, 3.5, 6], [3.5, below, 7],
           [6.0, 1.0, 1.5], [5.999999, 1.0, 1.25], [1.0, 6.0, 0.5], [7.9999995, 7.9999995, 7.0]]
    export = one_record(xyz)
    # 2 x 2 cells of 2 m from (0, 0): the grid ends at 4 (x - ox == nx * cell is excluded), 3.9999998 is inside
    dense = check(export, None, BOX, (0.0, 0.0), 2.0, (2, 2))
    assert dense[0].tolist() == [[3, 1], [0, 2]] and dense[4].tolist() == [[3, 2], [-1, 6]]
    # 3 x 4 cells of 2 m from (0, 0), and of 1.5 m from (0.5, -1): borders at multiples of the cell
    check(export, None, BOX, (0.0, 0.0), 2.0, (3, 4))
    check(export, None, BOX, (0.5, -1.0), 1.5, (7, 5))
    check(export, None, BOX, (0.0, 0.0), 1.0, (8, 8))


def test_negative_origin_and_grids_partly_or_wholly_outside_the_cube():
    rng = np.random.default_rng(2)
    export = one_record(rng.uniform(0, 8, (500, 3)).astype(F))
    for origin, cell, shape in [((-3.0, -5.0), 0.75, (9, 12)), ((-8.0, -8.0), 2.0, (4, 4)), ((6.0, 6.0), 0.5, (10, 10)),
                                ((100.0, -100.0), 1.0, (3, 3)), ((-1e6, -1e6), 1e5, (21, 21)), ((-0.25, 7.5), 0.1, (30, 90))]:
        dense = check(export, None, BOX, origin, cell, shape)
        if origin[0] == 100.0:
            assert dense[0].sum() == 0                         # wholly outside: every cell empty


def test_one_cell_and_the_largest_grid():
    rng = np.random.default_rng(3)
    export = one_record(rng.uniform(0, 8, (300, 3)).astype(F))
    dense = check(export, None, BOX, (0.0, 0.0), 8.0, (1, 1))
    assert dense[0][0, 0] == 300
    # 2^27 cells: the sparse form only (the dense one would take 3.5 GB here)
    assert check(export, None, BOX, (0.0, 0.0), 8.0 / 8192, (1 << 13, 1 << 14)) is None
    assert check(export, None, BOX, (0.0, 0.0), 8.0 / (1 << 26), (2, 1 << 26)) is None


def test_equal_z_and_signed_zeros_in_one_cell():
    xyz = [[1, 1, 2.5], [1.5, 1.5, 2.5], [0.5, 0.5, 1.0], [1.2, 1.2, 2.5], [5, 5, 0.0], [5.5, 5.5, -0.0], [5.2, 5.2, 0.0]]
    export = one_record(xyz)
    box = ((0.0, 0.0, -4.0), (8.0, 8.0, 4.0))                  # z below 0 is in this cube
    dense = check(export, None, box, (0.0, 0.0), 4.0, (2, 2))
    assert dense[4][0, 0] == 0 and dense[2][0, 0] == F(2.5)     # three at z = 2.5: the smallest index
    assert dense[4][1, 1] == 4                                 # +0 above -0: the first +0
    assert dense[1][1, 1].view(np.uint32) == 0x80000000 and dense[2][1, 1].view(np.uint32) == 0


def test_max_face_below_box_min_and_voxels_at_a_depth():
    pts = [[8.0, 1.0, 1.0], [1.0, 8.0, 1.0], [1.0, 1.0, 8.0], [-1e-6, 2.0, 2.0], [1.0, 1.0, 1.0]]
    vox = [[0.5, 0.5, 7.5], [1.5, 1.5, 0.5], [7.5, 7.5, 7.5]]
    assert Q.in_cube(one_record(pts)[1], *BOX).tolist() == [False, False, False, False, True]
    dense = check(one_record(pts), None, BOX, (-1.0, -1.0), 10.0, (1, 1))
    assert dense[0][0, 0] == 1                                 # only the point inside the cube
    inner = one_record(pts, vox, leaf=False)                   # the root cut at depth 0: its points and voxels
    dense = check(inner, 0, BOX, (0.0, 0.0), 4.0, (2, 2))
    assert dense[0].tolist() == [[3, 0], [0, 1]] and dense[2][0, 0] == F(7.5)
    dense = check(inner, None, BOX, (0.0, 0.0), 4.0, (2, 2))  # depth None: not a leaf, nothing
    assert dense[0].sum() == 0


# ---- the restatement on an oracle-built octree ------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tree():
    cloud, mn, mx = data.uniform_cube(60_000, size=256.0, seed=9)
    on_face = api.make_points(np.array([[256.0, 10.0, 10.0]], dtype=F), [7])
    points = np.concatenate([cloud[:600], cloud[:100], on_face, cloud[600:]])
    box = (mn, (256.0, 256.0, 256.0))
    o = oracle.Oracle(*box)
    for b in np.array_split(points, 2):
        o.add_batch(b)
    canon = o.canon()
    assert int(canon.records["level"].max()) >= 1
    return points, box, canon


@pytest.mark.parametrize("depth", [None, 0, "deepest"])
def test_restatement_on_an_oracle_octree(tree, depth):
    points, box, canon = tree
    if depth == "deepest":
        depth = int(canon.records["level"].max())
    export = R.export_canon(canon, depth)
    for origin, cell, shape in [((0.0, 0.0), 32.0, (8, 8)), ((-10.0, 50.0), 7.0, (40, 30)), ((100.0, 100.0), 1.0, (64, 64))]:
        dense = check(export, depth, box, origin, cell, shape)
        assert dense[0].sum() > 0
    if depth is None:                                          # every inserted point in the cube, once
        dense = check(export, None, box, (0.0, 0.0), 256.0, (1, 1))
        assert dense[0][0, 0] == int(Q.in_cube(points, *box).sum())


# ---- heightmap.cu: the exact set of kernels, none using local memory --------------------------------------------------

def test_heightmap_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "heightmap.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("heightmap", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "heightmap.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_heightmap_accumulate", "simlod_heightmap_finalize"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "heightmap" in B.PROGRAMS
