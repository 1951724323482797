"""CPU-only: the radius query's layouts, its restatement (radius_restatement) against a plain per-sample loop over the
record tree and against the k-nearest restatement on hand-made sample sets and on oracle-built octrees, and the resource
use of radius.cu's kernels. The GPU query is pinned byte for byte to this restatement in test_radius_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import nearest_restatement as N
import oracle
import query_restatement as Q
import radius_restatement as S
from conftest import ROOT
from simlod_b200 import api, data
from simlod_b200 import build as B

F = np.float32
INF = float("inf")
NAN = float("nan")


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_radius_info_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    s = api.SimlodRadiusInfo
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' +
                   'printf("%zu\\n", sizeof(SimlodRadiusInfo));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodRadiusInfo, %s));\n' % f for f, _ in s._fields_) +
                   'printf("%u\\n", SIMLOD_RADIUS_MAX_QUERIES);return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert out[:-1] == [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out[-1] == api.RADIUS_MAX_QUERIES == 1 << 24
    assert C.sizeof(s) == 64 and s.num_queries.offset == 32 and s.plan_ms.offset == 48
    assert "simlod_query_radius" in api.EXPORTS and hasattr(api.load_library(), "simlod_query_radius")


# ---- a plain statement: the record tree walked depth first in octant order, one sample at a time ----------------------

def plain(export, queries, radius, depth, box_min, box_max, rcp=None):
    """For each query: the terminal records in the walk's order (children by octant), each record's samples in export
    order, the float32 key of each one scalar at a time, kept when <= fl(r * r)."""
    nodes, samples, _ = export
    eligible = Q.in_cube(samples, box_min, box_max, rcp)
    order = []                                                # terminal records, depth first, children in octant order
    stack = [0] if len(nodes) else []
    while stack:
        r = stack.pop()
        fc = int(nodes["first_child"][r])
        if fc < 0:
            order.append(r)
        else:
            stack.extend(range(fc + 7, fc - 1, -1))
    with np.errstate(over="ignore"):
        rr = F(radius) * F(radius)
    offsets, index, dist2 = [0], [], []
    for q in np.asarray(queries, dtype=F)[:, :3]:
        if np.isfinite(q).all():
            for r in order:
                a, n_p, n_v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
                for i in range(a, a + n_p + (0 if depth is None else n_v)):
                    if i < a + n_p and not eligible[i]:
                        continue
                    with np.errstate(over="ignore", under="ignore"):
                        dx, dy, dz = F(samples["x"][i]) - q[0], F(samples["y"][i]) - q[1], F(samples["z"][i]) - q[2]
                        d2 = (dx * dx + dy * dy) + dz * dz
                    if d2 <= rr:
                        index.append(i)
                        dist2.append(d2)
        offsets.append(len(index))
    return np.array(offsets, dtype=np.int64), np.array(index, dtype=np.int64), np.array(dist2, dtype=F)


def check(export, queries, radius, depth, box, rcp=None, loop=True):
    got = S.radius(export, queries, radius, depth, *box, rcp=rcp)
    brute = S.brute_force(export, queries, radius, depth, *box, rcp=rcp)
    wants = [("brute_force", brute)] + ([("plain", plain(export, queries, radius, depth, *box, rcp=rcp))] if loop else [])
    for name, want in wants:
        for part, g, w in zip(("offsets", "index", "dist2"), got, want):
            assert g.tobytes() == w.tobytes(), "%s: %s\n%r\n%r" % (name, part, g, w)
    if S._rr(radius) != INF:                                  # nearest_restatement bounds its superset by the radius itself
        nearest_agrees(export, queries, radius, depth, box, got, rcp)
    return got


def nearest_agrees(export, queries, radius, depth, box, got, rcp=None):
    """Each query with <= 32 neighbours: its segment sorted by (d2, index) is the filled slots of the 32 nearest within r."""
    offsets, index, dist2 = got
    ni, nd = N.nearest(export, queries, 32, depth, *box, rcp=rcp, max_radius=radius)
    for t in range(len(offsets) - 1):
        a, b = int(offsets[t]), int(offsets[t + 1])
        if b - a > 32:
            continue
        o = np.lexsort((index[a:b], dist2[a:b]))
        filled = ni[t] >= 0
        assert int(filled.sum()) == b - a, t
        assert index[a:b][o].tolist() == ni[t][filled].tolist() and dist2[a:b][o].tobytes() == nd[t][filled].tobytes(), t


def one_leaf(xyz, box=((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))):
    """An export with the root as its only (leaf) record, holding `xyz` as points in this order."""
    samples = api.make_points(np.asarray(xyz, dtype=F).reshape(-1, 3), np.arange(len(xyz), dtype=np.uint32))
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["flags"], nodes["parent"], nodes["first_child"] = R.LEAF | R.SAMPLED, -1, -1
    nodes["num_points"] = len(samples)
    info = R.ExportInfo(1, 0, len(samples), len(samples), 0)
    return (nodes, samples, info), box


# ---- hand-made sets ---------------------------------------------------------------------------------------------------

def test_duplicates_and_samples_exactly_at_the_radius():
    grid = np.array([[x, y, z] for x in range(4) for y in range(4) for z in range(4)], dtype=F)
    xyz = np.concatenate([grid[::-1], grid[:5], grid[:5]])     # every point of grid[:5] three times
    export, box = one_leaf(xyz)
    queries = np.array([[1.0, 1.0, 1.0], [0.0, 0.0, 0.0], [1.5, 1.5, 1.5], [3.0, 3.0, 3.0]], dtype=F)
    offsets, index, d2 = check(export, queries, 1.0, None, box)
    # the query on a grid point: itself and its 6 axis neighbours at d2 == fl(1 * 1) exactly, in export order
    seg = slice(offsets[0], offsets[1])
    assert offsets[1] - offsets[0] == 7 and sorted(d2[seg].tolist()).count(1.0) == 6 and index[seg].tolist() == sorted(index[seg])
    # the origin, stored three times: the duplicates all count
    seg = slice(offsets[1], offsets[2])
    assert (d2[seg] == 0).sum() == 3
    # the 8 corners of a cell are at d2 = 0.75 from its centre: radius sqrt(0.75) rounds so that they are or are not in
    r = float(np.sqrt(np.float64(0.75)))
    o2, i2, _ = check(export, queries[2:3], r, None, box)
    assert o2[1] == (8 if F(r) * F(r) >= F(0.75) else 0)


def test_radius_zero_and_non_finite_and_outside_queries():
    rng = np.random.default_rng(5)
    xyz = rng.uniform(0, 8, (300, 3)).astype(F)
    export, box = one_leaf(xyz)
    queries = np.concatenate([xyz[:10], [[NAN, 1, 1], [1, INF, 1], [-INF, 0, 0], [100.0, -50.0, 3.0], [-1.0, 4.0, 4.0]]]).astype(F)
    offsets, index, d2 = check(export, queries, 0.0, None, box)
    assert np.diff(offsets)[:10].tolist() == [1] * 10 and index[:10].tolist() == list(range(10)) and (d2 == 0).all()
    assert offsets[-1] == 10
    offsets, index, d2 = check(export, queries, 1.5, None, box)
    assert (np.diff(offsets)[10:13] == 0).all() and np.diff(offsets)[14] > 0     # non-finite empty; outside finds
    assert (d2 <= F(1.5) * F(1.5)).all()


def test_max_face_and_below_box_min_points_are_never_neighbours():
    xyz = [[8.0, 1.0, 1.0], [1.0, 8.0, 1.0], [7.9, 7.9, 7.9], [1.0, 1.0, 1.0], [-0.0, 0.0, 0.0], [-1e-6, 2.0, 2.0]]
    export, box = one_leaf(xyz)
    assert Q.in_cube(export[1], *box).tolist() == [False, False, True, True, True, False]
    queries = np.array([[8.0, 1.0, 1.0], [1.0, 8.0, 1.0], [0.0, 2.0, 2.0], [4, 4, 4]], dtype=F)
    offsets, index, d2 = check(export, queries, 20.0, None, box)
    assert not np.isin(index, [0, 1, 5]).any() and np.diff(offsets).tolist() == [3, 3, 3, 3]


def test_a_radius_whose_square_overflows_takes_every_sample():
    export, box = one_leaf([[1, 1, 1], [2, 2, 2], [3, 3, 3]])
    queries = np.array([[3e38, 0, 0], [-3e38, 3e38, 0], [1, 1, 1]], dtype=F)
    offsets, index, d2 = check(export, queries, 2e19, None, box)
    assert np.diff(offsets).tolist() == [3, 3, 3] and index.tolist() == [0, 1, 2] * 3 and np.isinf(d2[:6]).all()
    offsets, _, _ = check(export, queries, 1e18, None, box)   # finite r * r: the overflowed keys are out
    assert np.diff(offsets).tolist() == [0, 0, 3]


def two_level_tree():
    """Root (with points of its own, not candidates at depth None) -> 8 children at level 1; child 0 -> 8 children at
    level 2. Breadth-first records: 0 root, 1..8 level 1, 9..16 level 2 inside record 1. Each leaf holds 3 points in its
    box. In Z-order records 9..16 precede 2..8, so the output order is not ascending index."""
    box = ((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))
    rng = np.random.default_rng(3)
    nodes = np.zeros(17, dtype=R.EXPORT_NODE_DTYPE)
    nodes["parent"][1:9], nodes["parent"][9:] = 0, 1
    nodes["first_child"] = -1
    nodes["first_child"][0], nodes["first_child"][1] = 1, 9
    pts, offset = [], 0
    for r in range(17):
        level, o = (0, 0) if r == 0 else (1, r - 1) if r < 9 else (2, r - 9)
        X, Y, Z = (o >> 2) & 1, (o >> 1) & 1, o & 1
        nodes["level"][r], nodes["X"][r], nodes["Y"][r], nodes["Z"][r] = level, X, Y, Z
        nodes["flags"][r] = R.SAMPLED | (R.LEAF if r not in (0, 1) else 0)
        size = 8.0 / (1 << level)
        n = 2 if r in (0, 1) else 3
        pts.append(np.array([X, Y, Z], dtype=np.float64) * size + rng.uniform(0.05, 0.95, (n, 3)) * size)
        nodes["sample_offset"][r], nodes["num_points"][r] = offset, n
        offset += n
    xyz = np.concatenate(pts).astype(F)
    samples = api.make_points(xyz, np.arange(len(xyz), dtype=np.uint32))
    return (nodes, samples, R.ExportInfo(17, 2, len(xyz), len(xyz), 0)), box


def test_leaves_at_different_levels_come_in_z_order():
    export, box = two_level_tree()
    queries = np.array([[4.0, 4.0, 4.0], [2.0, 2.0, 2.0], [0.5, 6.0, 0.5], [9.0, 9.0, 9.0]], dtype=F)
    offsets, index, d2 = check(export, queries, 5.0, None, box)
    seg = index[offsets[0]:offsets[1]]
    assert not np.isin(seg, np.arange(0, 4)).any()            # the inner records' points are not candidates
    assert (np.diff(seg) < 0).any(), "Z-order must differ from index order here: %r" % seg
    offsets, index, _ = check(export, queries, 100.0, None, box)
    nodes = export[0]
    zk = S.zkeys(nodes)
    leaves = [r for r in range(17) if nodes["first_child"][r] < 0]
    walk = sorted(leaves, key=lambda r: int(zk[r]))
    assert walk[:9] == [9, 10, 11, 12, 13, 14, 15, 16, 2]
    expect = np.concatenate([np.arange(nodes["sample_offset"][r], nodes["sample_offset"][r] + 3) for r in walk])
    assert index[offsets[0]:offsets[1]].tolist() == expect.tolist()


# ---- the restatement on an oracle-built octree ------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tree():
    cloud, mn, mx = data.uniform_cube(150_000, size=256.0, seed=9)
    on_face = api.make_points(np.array([[256.0, 10.0, 10.0]], dtype=F), [7])
    points = np.concatenate([cloud[:1000], cloud[:200], on_face, cloud[1000:]])       # 200 exact duplicates
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
    rng = np.random.default_rng(4)
    stored = np.stack([points["x"], points["y"], points["z"]], axis=1)[rng.choice(len(points), 12)]
    queries = np.concatenate([stored, stored + rng.normal(0, 1.0, stored.shape), rng.uniform(-20, 276, (12, 3)),
                              [[256.0, 10.0, 10.0], [NAN, 0, 0]]]).astype(F)
    for radius in (0.0, 3.0, 12.0):
        offsets, index, d2 = check(export, queries, radius, depth, box, loop=False)
        assert offsets[-1] == len(index) and (d2 <= F(radius) * F(radius)).all()
    if depth is None:                                         # the stored points find themselves
        offsets, index, d2 = S.radius(export, stored.astype(F), 0.0, None, *box)
        assert (np.diff(offsets) >= 1).all() and (d2 == 0).all()


# ---- radius.cu: the exact set of kernels, none using local memory -----------------------------------------------------

def test_radius_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "radius.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("radius", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "radius.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_radius_count", "simlod_radius_reduce", "simlod_radius_scan",
                                      "simlod_radius_write"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "radius" in B.PROGRAMS
