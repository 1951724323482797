"""CPU-only: the k-nearest query's layouts, its restatement (nearest_restatement) against a plain brute force on
hand-made sample sets and on oracle-built octrees, and the resource use of nearest.cu's kernels. The GPU query is pinned
byte for byte to this restatement in test_nearest_gpu.py."""
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
from conftest import ROOT
from simlod_b200 import api, data
from simlod_b200 import build as B

F = np.float32
INF = float("inf")
NAN = float("nan")


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_nearest_info_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    s = api.SimlodNearestInfo
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' +
                   'printf("%zu\\n", sizeof(SimlodNearestInfo));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodNearestInfo, %s));\n' % f for f, _ in s._fields_) +
                   'printf("%d %u\\n", SIMLOD_NEAREST_MAX_K, SIMLOD_NEAREST_MAX_QUERIES);return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert out[:-2] == [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out[-2:] == [api.NEAREST_MAX_K, api.NEAREST_MAX_QUERIES] == [32, 1 << 24]
    assert C.sizeof(s) == 64 and s.plan_ms.offset == 48
    assert "simlod_query_nearest" in api.EXPORTS and hasattr(api.load_library(), "simlod_query_nearest")


# ---- a plain brute force, stated without the restatement's helpers ----------------------------------------------------

def plain(export, queries, k, depth, box_min, box_max, rcp=None, max_radius=None):
    """For each query: every sample of the set, its float32 key, a full sort by (d2, index), the first k."""
    nodes, samples, _ = export
    members = []                                              # (export index, is voxel) of the sample set
    for r in range(len(nodes)):
        a, n_p, n_v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
        full = depth is None
        if not full or nodes["flags"][r] & R.LEAF:
            members.append((np.arange(a, a + n_p), np.zeros(n_p, dtype=bool)))
        if not full:
            members.append((np.arange(a + n_p, a + n_p + n_v), np.ones(n_v, dtype=bool)))
    idx = np.concatenate([m[0] for m in members] + [np.zeros(0, dtype=np.int64)]).astype(np.int64)
    vox = np.concatenate([m[1] for m in members] + [np.zeros(0, dtype=bool)])
    idx = idx[vox | Q.in_cube(samples[idx], box_min, box_max, rcp)]
    x, y, z = (samples[c][idx].astype(F) for c in ("x", "y", "z"))
    rr = F(INF if max_radius is None else max_radius)
    with np.errstate(over="ignore"):
        rr = rr * rr
    out_i = np.full((len(queries), k), -1, dtype=np.int64)
    out_d = np.full((len(queries), k), INF, dtype=F)
    for t, q in enumerate(np.asarray(queries, dtype=F)):
        if not np.isfinite(q[:3]).all():
            continue
        with np.errstate(over="ignore", under="ignore"):
            dx, dy, dz = x - q[0], y - q[1], z - q[2]
            d2 = (dx * dx + dy * dy) + dz * dz
        keep = d2 <= rr
        order = np.lexsort((idx[keep], d2[keep]))[:k]
        out_i[t, :len(order)], out_d[t, :len(order)] = idx[keep][order], d2[keep][order]
    return out_i, out_d


def check(export, queries, k, depth, box, max_radius=None, rcp=None):
    want = plain(export, queries, k, depth, *box, rcp=rcp, max_radius=max_radius)
    got = N.nearest(export, queries, k, depth, *box, rcp=rcp, max_radius=max_radius)
    brute = N.brute_force(export, queries, k, depth, *box, rcp=rcp, max_radius=max_radius)
    for name, res in (("restatement", got), ("brute_force", brute)):
        assert res[0].tobytes() == want[0].tobytes(), "%s: index\n%r\n%r" % (name, res[0], want[0])
        assert res[1].tobytes() == want[1].tobytes(), "%s: d2" % name
    return got


# ---- hand-made sets: one leaf (the root), so that the export's order is the insertion order ---------------------------

def one_leaf(xyz, box=((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))):
    """An export with the root as its only (leaf) record, holding `xyz` as points in this order."""
    samples = api.make_points(np.asarray(xyz, dtype=F).reshape(-1, 3), np.arange(len(xyz), dtype=np.uint32))
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["flags"], nodes["parent"], nodes["first_child"] = R.LEAF | R.SAMPLED, -1, -1
    nodes["num_points"] = len(samples)
    info = R.ExportInfo(1, 0, len(samples), len(samples), 0)
    return (nodes, samples, info), box


def test_duplicates_and_equidistant_grid_points_tie_by_index():
    grid = np.array([[x, y, z] for x in range(4) for y in range(4) for z in range(4)], dtype=F)
    xyz = np.concatenate([grid[::-1], grid[:5], grid[:5]])     # every point of grid[:5] three times
    export, box = one_leaf(xyz)
    queries = np.array([[1.5, 1.5, 1.5], [0.0, 0.0, 0.0], [0.5, 0.5, 0.5], [3.0, 3.0, 3.0]], dtype=F)
    index, d2 = check(export, queries, 12, None, box)
    # the 8 corners of the cell around (1.5, 1.5, 1.5) are equidistant: by index, which follows grid[::-1]
    corners = sorted(int(i) for i in np.nonzero(N.key(N._xyz(export[1]), queries[0]) == F(0.75))[0])
    assert len(corners) == 8 and index[0, :8].tolist() == corners and (d2[0, :8] == F(0.75)).all()
    # the query on a stored point finds it with its two duplicates first, at d2 = 0, ascending indices
    zero = [int(i) for i in np.nonzero((xyz == 0).all(axis=1))[0]]
    assert len(zero) == 3 and index[1, :3].tolist() == zero and (d2[1, :3] == 0).all() and d2[1, 3] > 0


def test_ineligible_points_outside_queries_and_non_finite_queries():
    xyz = [[8.0, 1.0, 1.0], [1.0, 8.0, 1.0], [7.9, 7.9, 7.9], [1.0, 1.0, 1.0], [-0.0, 0.0, 0.0], [-1e-6, 2.0, 2.0]]
    export, box = one_leaf(xyz)
    assert Q.in_cube(export[1], *box).tolist() == [False, False, True, True, True, False]
    queries = np.array([[8.0, 1.0, 1.0], [100.0, -50.0, 3.0], [NAN, 1.0, 1.0], [1.0, INF, 1.0], [-INF, 0, 0], [4, 4, 4]], dtype=F)
    index, d2 = check(export, queries, 4, None, box)
    assert not np.isin(index, [0, 1, 5]).any()               # the max-face points and the one below boxMin
    assert (index[2:5] == -1).all() and np.isinf(d2[2:5]).all()
    assert (index[[0, 1, 5], 3] == -1).all() and (index[[0, 1, 5], :3] >= 0).all()   # three eligible points: k = 4 is more


def test_max_radius_zero_and_small():
    rng = np.random.default_rng(5)
    xyz = rng.uniform(0, 8, (300, 3)).astype(F)
    export, box = one_leaf(xyz)
    queries = np.concatenate([xyz[:20], rng.uniform(-1, 9, (20, 3)).astype(F)])
    index, d2 = check(export, queries, 8, None, box, max_radius=0.0)
    assert (index[:20, 0] == np.arange(20)).all() and (index[:20, 1:] == -1).all() and (index[20:] == -1).all()
    index, d2 = check(export, queries, 8, None, box, max_radius=0.7)
    assert (d2[index >= 0] <= F(0.7) * F(0.7)).all() and (index == -1).any() and (index[:, 1] >= 0).any()


def test_k_larger_than_the_set():
    export, box = one_leaf([[1, 1, 1], [2, 2, 2], [3, 3, 3]])
    index, d2 = check(export, np.array([[0, 0, 0], [2.6, 2.6, 2.6]], dtype=F), 32, None, box)
    assert index[0, :3].tolist() == [0, 1, 2] and index[1, :3].tolist() == [2, 1, 0] and (index[:, 3:] == -1).all()
    assert np.isinf(d2[:, 3:]).all()
    empty, _ = one_leaf(np.zeros((0, 3)))
    index, d2 = check(empty, np.array([[1, 1, 1]], dtype=F), 5, None, box)
    assert (index == -1).all()


def test_keys_that_overflow_tie_by_index():
    export, box = one_leaf([[1, 1, 1], [2, 2, 2], [3, 3, 3]])
    index, d2 = check(export, np.array([[3e38, 0, 0], [-3e38, 3e38, 0]], dtype=F), 2, None, box)
    assert np.isinf(d2).all() and index.tolist() == [[0, 1], [0, 1]]


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
    queries = np.concatenate([stored, rng.uniform(-20, 276, (12, 3)), [[256.0, 10.0, 10.0], [NAN, 0, 0]]]).astype(F)
    for k, radius in ((1, None), (8, None), (32, 4.0)):
        check(export, queries, k, depth, box, max_radius=radius)
    if depth is None:                                         # the stored points are found at d2 = 0
        index, d2 = N.nearest(export, stored.astype(F), 1, None, *box)
        assert (d2[:, 0] == 0).all()


# ---- nearest.cu: the exact set of kernels, none using local memory ----------------------------------------------------

def test_nearest_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "nearest.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("nearest", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "nearest.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_nearest_locate", "simlod_nearest_scan", "simlod_nearest_scatter",
                                      "simlod_nearest_search"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "nearest" in B.PROGRAMS
