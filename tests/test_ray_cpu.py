"""CPU-only: the ray query's layouts, its restatement (ray_restatement: the grid superset against its brute force and
against a plain per-sample loop) on hand-made sample sets and on oracle-built octrees, and the resource use of ray.cu's
kernels. The GPU query is pinned byte for byte to this restatement in test_ray_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import oracle
import query_restatement as Q
import ray_restatement as Y
from conftest import ROOT
from simlod_b200 import api, data
from simlod_b200 import build as B

F = np.float32
INF = float("inf")
NAN = float("nan")


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_ray_info_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    s = api.SimlodRayInfo
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n' +
                   'printf("%zu\\n", sizeof(SimlodRayInfo));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodRayInfo, %s));\n' % f for f, _ in s._fields_) +
                   'printf("%u\\n", SIMLOD_RAY_MAX_RAYS);return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert out[:-1] == [C.sizeof(s)] + [getattr(s, f).offset for f, _ in s._fields_]
    assert out[-1] == api.RAY_MAX_RAYS == 1 << 24
    assert C.sizeof(s) == 56 and s.plan_ms.offset == 44 and s.num_rays.offset == 32
    assert "simlod_query_ray" in api.EXPORTS and hasattr(api.load_library(), "simlod_query_ray")


# ---- a plain loop, stated without the restatement's helpers -------------------------------------------------------------

def plain(export, rays, radius, depth, box_min, box_max, rcp=None):
    """For each ray and each sample of the set, one float32 operation at a time; the least (t, index) among the hits."""
    nodes, samples, _ = export
    members = []
    for r in range(len(nodes)):
        a, n_p, n_v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
        if depth is not None or nodes["flags"][r] & R.LEAF:
            members += [(i, False) for i in range(a, a + n_p)]
        if depth is not None:
            members += [(i, True) for i in range(a + n_p, a + n_p + n_v)]
    eligible = Q.in_cube(samples, box_min, box_max, rcp)
    rr = np.multiply(F(radius), F(radius), dtype=F)
    out_i = np.full(len(rays), -1, dtype=np.int64)
    out_t = np.full(len(rays), INF, dtype=F)
    out_h = np.full(len(rays), INF, dtype=F)
    for k, ray in enumerate(np.asarray(rays, dtype=F)):
        o, tmin, d, tmax = ray[0:3], ray[3], ray[4:7], ray[7]
        if not (np.isfinite(o).all() and np.isfinite(d).all() and (d != 0).any() and np.isfinite(tmin) and tmin >= 0
                and tmax >= tmin):
            continue
        dd = [float(v) for v in d]
        length = ((dd[0] * dd[0] + dd[1] * dd[1]) + dd[2] * dd[2]) ** 0.5
        u = [F(v / length) for v in dd]
        best = None
        for i, voxel in members:
            if not voxel and not eligible[i]:
                continue
            p = [F(samples[c][i]) for c in ("x", "y", "z")]
            with np.errstate(all="ignore"):
                w = [p[a] - o[a] for a in range(3)]
                t = ((w[0] * u[0] + w[1] * u[1]) + w[2] * u[2]) + F(0)
                c = [w[1] * u[2] - w[2] * u[1], w[2] * u[0] - w[0] * u[2], w[0] * u[1] - w[1] * u[0]]
                h2 = (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]
            if tmin <= t <= tmax and h2 <= rr and (best is None or (int(t.view(np.uint32)), i) < best[0]):
                best = ((int(t.view(np.uint32)), i), t, h2)
        if best is not None:
            out_i[k], out_t[k], out_h[k] = best[0][1], best[1], best[2]
    return out_i, out_t, out_h


def check(export, rays, radius, depth, box, rcp=None, loop=True):
    got = Y.trace(export, rays, radius, depth, *box, rcp=rcp)
    brute = Y.brute_force(export, rays, radius, depth, *box, rcp=rcp)
    results = [("brute_force", brute)] + ([("plain", plain(export, rays, radius, depth, *box, rcp=rcp))] if loop else [])
    for name, want in results:
        for a, b, what in zip(got, want, ("index", "t", "h2")):
            assert a.tobytes() == b.tobytes(), "%s: %s\n%r\n%r" % (name, what, a, b)
    return got


# ---- hand-made sets: one leaf (the root), so that the export's order is the insertion order ---------------------------

BOX = ((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))


def one_leaf(xyz):
    """An export with the root as its only (leaf) record, holding `xyz` as points in this order."""
    samples = api.make_points(np.asarray(xyz, dtype=F).reshape(-1, 3), np.arange(len(xyz), dtype=np.uint32))
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["flags"], nodes["parent"], nodes["first_child"] = R.LEAF | R.SAMPLED, -1, -1
    nodes["num_points"] = len(samples)
    return nodes, samples, R.ExportInfo(1, 0, len(samples), len(samples), 0)


def test_duplicates_and_equal_t_tie_by_index():
    xyz = [[6, 4, 4], [2, 4.25, 4], [2, 4, 4], [2, 3.75, 4], [2, 4, 4], [2, 4, 4.25], [1, 4, 5]]
    export = one_leaf(xyz)
    r = Y.rays([[0, 4, 4], [0, 4, 4.25], [8, 4, 4]], [[1, 0, 0], [1, 0, 0], [-1, 0, 0]])
    index, t, h2 = check(export, r, 0.5, None, BOX)
    assert index.tolist() == [1, 1, 0] and t.tolist() == [2.0, 2.0, 2.0]     # five samples at t = 2: the lowest index
    index, t, h2 = check(export, r[:1], 0.0, None, BOX)
    assert index.tolist() == [2] and h2[0] == 0                               # radius 0: the duplicates on the ray
    # the grid superset splits these into different cells: the order of the cells must not matter
    grid = np.array([[x, y, z] for x in range(8) for y in range(8) for z in range(8)], dtype=F)
    export = one_leaf(np.concatenate([grid[::-1], grid]))
    r = Y.rays([[3, 3, -1], [-1, 2.5, 2.5], [7.5, 7.5, 7.5]], [[0, 0, 1], [1, 0, 0], [-1, -1, -1]])
    index, t, _ = check(export, r, 0.75, None, BOX, loop=False)
    assert (index >= 0).all()


def test_at_radius_tmin_and_tmax_and_minus_zero():
    xyz = [[3, 4.5, 4], [2, 4.5000005, 4], [5, 4, 4], [7, 4, 4], [1, 4, 4]]
    export = one_leaf(xyz)
    r = Y.rays([[0, 4, 4]] * 4, [[1, 0, 0]] * 4, [0, 3, 5, 7.5], [INF, 4, 7, INF])
    index, t, h2 = check(export, r, 0.5, None, BOX)
    # h2 == r*r hits; 4.5000005 is beyond; t == tmin hits; t == tmax hits
    assert index.tolist() == [4, 0, 2, -1] and h2[1] == F(0.25)
    r = Y.rays([[0, 4, 4]], [[1, 0, 0]], 7.0, 7.0)
    assert check(export, r, 0.5, None, BOX)[0].tolist() == [3]
    # a sample at the origin of a ray whose direction is negative on every axis: t = -0 + 0 = +0
    export = one_leaf([[4, 4, 4], [5, 5, 5]])
    index, t, h2 = check(export, Y.rays([[4, 4, 4]], [[-1, -1, -1]]), 0.0, None, BOX)
    assert index.tolist() == [0] and t.view(np.uint32).tolist() == [0]


def test_axis_parallel_rays_origins_on_faces_inside_outside_and_far():
    rng = np.random.default_rng(3)
    xyz = np.concatenate([rng.integers(0, 8, (300, 3)).astype(F), rng.uniform(0, 8, (300, 3)).astype(F)])
    export = one_leaf(xyz)
    origins, dirs = [], []
    for a in range(3):                                          # along each axis, from on a face, from inside, from outside
        for start in (0.0, 4.0, -3.0, 8.0):
            for off in ((2.0, 3.0), (4.0, 4.0), (0.0, 7.0)):
                o = [off[0], off[1]]
                o.insert(a, start)
                d = [0.0, 0.0]
                d.insert(a, 1.0 if start != 8.0 else -1.0)
                origins.append(o)
                dirs.append(d)
    origins += [[-8e6, 4.0, 4.0], [-8e6, -8e6, 4.0], [4.0, 4.0, 8e6], [20, 20, 20], [-1, -1, -1]]
    dirs += [[1, 0, 0], [1, 1, 0.0000001], [0.001, -0.002, -1], [1, 1, 1], [-1, -1, -1]]
    r = Y.rays(origins, dirs)
    for radius in (0.0, 0.3, 2.0):
        index, t, h2 = check(export, r, radius, None, BOX)
        assert index[-1] == -1 and index[-2] == -1               # pointing away from the cube
    assert (check(export, r, 0.0, None, BOX)[0][:36] >= 0).sum() >= 12   # integer rays through integer points


def test_ineligible_points_are_never_hit():
    xyz = [[8.0, 1.0, 1.0], [1.0, 8.0, 1.0], [-1e-6, 2.0, 2.0], [1.0, 1.0, 1.0], [1.0, 8.0, 8.0]]
    export = one_leaf(xyz)
    assert Q.in_cube(export[1], *BOX).tolist() == [False, False, False, True, False]
    r = Y.rays([[9, 1, 1], [1, 9, 1], [-1, 2, 2], [0, 1, 1], [1, 9, 9]], [[-1, 0, 0], [0, -1, 0], [1, 0, 0], [1, 0, 0], [0, -1, -1]])
    index, _, _ = check(export, r, 0.1, None, BOX)
    assert index.tolist() == [3, 3, -1, 3, 3]                   # each ray passes an ineligible point first


def test_every_kind_of_invalid_ray():
    export = one_leaf([[1, 1, 1], [2, 2, 2]])
    o, d = [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]
    cases = [(("o", 0, NAN)), ("o", 1, INF), ("o", 2, -INF), ("d", 0, NAN), ("d", 1, INF), ("zero", 0, 0), ("tmin", 0, NAN),
             ("tmin", 0, -1.0), ("tmin", 0, INF), ("tmax", 0, NAN), ("tmax", 0, 0.5)]
    rows = []
    for what, a, v in cases:
        oo, dd, tmin, tmax = list(o), list(d), 1.0, INF
        if what == "o":
            oo[a] = v
        elif what == "d":
            dd[a] = v
        elif what == "zero":
            dd = [0.0, 0.0, 0.0]
        elif what == "tmin":
            tmin = v
        else:
            tmax = v
        rows.append(Y.rays([oo], [dd], tmin, tmax)[0])
    # valid edge cases: tmin -0, tmax == tmin, tmax +inf, a denormal direction
    rows += list(Y.rays([o, o, o], [d, d, [1e-45, 0, 0]], [-0.0, 3 ** 0.5, 0.0], [INF, 3 ** 0.5, INF]))
    r = np.array(rows, dtype=F)
    assert Y.valid(r).tolist() == [False] * len(cases) + [True] * 3
    index, t, h2 = check(export, r, 0.1, None, BOX)
    assert (index[:len(cases)] == -1).all() and np.isinf(t[:len(cases)]).all() and np.isinf(h2[:len(cases)]).all()
    assert index[len(cases):].tolist() == [0, 0, -1]


def test_radius_zero():
    rng = np.random.default_rng(5)
    xyz = rng.integers(0, 8, (400, 3)).astype(F)
    export = one_leaf(xyz)
    origins = np.concatenate([xyz[:20] - F(0.5) * np.array([1, 0, 0], dtype=F), rng.uniform(-1, 9, (20, 3)).astype(F)])
    dirs = np.concatenate([np.tile([[1, 0, 0]], (20, 1)), rng.normal(0, 1, (20, 3))]).astype(F)
    index, t, h2 = check(export, Y.rays(origins, dirs), 0.0, None, BOX)
    assert (index[:20] >= 0).all() and (h2[:20] == 0).all() and (t[:20] == F(0.5)).all()


# ---- the restatement on an oracle-built octree ------------------------------------------------------------------------

@pytest.fixture(scope="module")
def tree():
    cloud, mn, mx = data.uniform_cube(60_000, size=256.0, seed=9)
    on_face = api.make_points(np.array([[256.0, 10.0, 10.0]], dtype=F), [7])
    points = np.concatenate([cloud[:1000], cloud[:200], on_face, cloud[1000:]])       # 200 exact duplicates
    box = (mn, (256.0, 256.0, 256.0))
    o = oracle.Oracle(*box)
    for b in np.array_split(points, 2):
        o.add_batch(b)
    canon = o.canon()
    assert int(canon.records["level"].max()) >= 1
    return points, box, canon


def tree_rays(points, rng, n=16):
    xyz = np.stack([points["x"], points["y"], points["z"]], axis=1).astype(np.float64)
    a, b = xyz[rng.choice(len(xyz), n)], xyz[rng.choice(len(xyz), n)]
    origins = [a - 0.25 * (b - a), rng.uniform(-50, 300, (n, 3)), np.tile([[128.0, 64.0, 0.0]], (n, 1))]
    dirs = [b - a, rng.normal(0, 1, (n, 3)), np.tile([[0.0, 0.0, 1.0]], (n, 1))]
    origins[2][:, 0] = rng.choice([0.0, 64.0, 128.0, 192.0, 256.0], n)      # on node faces, axis-parallel
    origins[2][:, 1] = rng.uniform(0, 256, n)
    tmax = [np.full(n, 1.25), np.full(n, np.inf), np.full(n, np.inf)]       # segments between two stored points
    tmax[0] *= np.linalg.norm(b - a, axis=1)
    return Y.rays(np.concatenate(origins), np.concatenate(dirs), 0.0, np.concatenate(tmax))


@pytest.mark.parametrize("depth", [None, 0, "deepest"])
def test_restatement_on_an_oracle_octree(tree, depth):
    points, box, canon = tree
    if depth == "deepest":
        depth = int(canon.records["level"].max())
    export = R.export_canon(canon, depth)
    r = tree_rays(points, np.random.default_rng(4))
    for radius in (0.0, 0.5, 3.0):
        index, t, h2 = check(export, r, radius, depth, box, loop=False)
        if radius == 3.0:
            assert (index >= 0).sum() >= 16
    if depth is None:                                         # a segment between two stored points finds the first one
        index, t, _ = check(export, r[:16], 0.01, None, box, loop=False)
        assert (index >= 0).all()


# ---- ray.cu: the exact set of kernels, none using local memory --------------------------------------------------------

def test_ray_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "ray.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("ray", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "ray.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    assert {f for f, *_ in found} == {"simlod_ray_check", "simlod_ray_trace"}, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
    assert "ray" in B.PROGRAMS
