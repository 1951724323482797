"""CPU-only checks of the oracle (oracle/oracle.cpp) against independent restatements and against
properties the reference's algorithm guarantees, plus the golden digests produced by the
reference's own kernels on an H100 (tests/golden/, see make_golden.py)."""
import os

import numpy as np
import pytest

import oracle
from simlod_b200 import data, make_points


def quantize(pts, size, mn=(0.0, 0.0, 0.0)):
    """numpy restatement of voxels.cu:148-155 for a power-of-two cube (exact reciprocal)."""
    out = []
    for ax, m in zip("xyz", mn):
        d = pts[ax].astype(np.float32) - np.float32(m)
        X = (d * np.float32(1048576.0) * np.float32(1.0 / size))
        P = (d * np.float32(268435456.0) * np.float32(1.0 / size))
        out.append((np.clip(np.floor(X), 0, 2**32 - 1).astype(np.uint64), np.clip(np.floor(P), 0, 2**32 - 1).astype(np.uint64)))
    return out


def build(batches, box, rcp=0.0):
    o = oracle.Oracle(box[0], box[1], rcp)
    for b in batches:
        o.add_batch(b)
    return o


@pytest.fixture(scope="module")
def config1():
    pts, mn, mx = data.uniform_cube(1_000_000)
    o = build([pts], (mn, mx))
    return pts, (mn, mx), o, o.canon()


def test_config1_topology_matches_the_survey_prediction(config1):
    pts, box, o, cn = config1
    s = o.stats()
    # SURVEY.md §8d: root -> 8 -> 64 leaves (73 nodes, 9 inner), ~0.79 M root voxels + ~0.97 M level-1 voxels
    assert (s.numNodes, s.numInner, s.numLeaves, s.numNonemptyLeaves) == (73, 9, 64, 64)
    assert s.numPoints == 1_000_000 and s.numPointsProcessed == 1_000_000 and s.batchletIndex == 1
    root = cn.records[0]
    assert root["name"] == b"r" and 780_000 < root["numVoxels"] < 800_000
    lvl1 = cn.records[cn.records["level"] == 1]
    assert len(lvl1) == 8 and 950_000 < lvl1["numVoxels"].sum() < 990_000
    assert s.numVoxels == root["numVoxels"] + lvl1["numVoxels"].sum()
    assert s.droppedSpilledPoints == 0


def test_leaf_membership_and_voxel_sets_against_numpy(config1):
    pts, (mn, mx), o, cn = config1
    (X, pX), (Y, pY), (Z, pZ) = quantize(pts, 1024.0)
    total = 0
    for k, r in enumerate(cn.records):
        L = int(r["level"])
        sel = ((X >> np.uint64(20 - L)) == r["X"]) & ((Y >> np.uint64(20 - L)) == r["Y"]) & ((Z >> np.uint64(20 - L)) == r["Z"])
        if r["isLeaf"]:
            assert sel.sum() == r["numPoints"] == r["counter"]
            got = cn.samples(k)
            want = np.sort(pts[sel].view("V16"))
            assert (np.sort(got.view("V16")) == want).all()
            total += int(r["numPoints"])
            assert r["chunksPoints"] == -(-int(r["numPoints"]) // 1000)
        else:
            sh = np.uint64(21 - L)
            cells = ((pX[sel] >> sh) & np.uint64(127)) | (((pY[sel] >> sh) & np.uint64(127)) << np.uint64(7)) | (((pZ[sel] >> sh) & np.uint64(127)) << np.uint64(14))
            assert len(np.unique(cells)) == r["numVoxels"] == r["numVoxelsStored"]
            assert r["numPoints"] == 0 and r["chunksVoxels"] == -(-int(r["numVoxels"]) // 1000)
            vox = cn.samples(k, voxels=True)
            # voxel = cell centre (voxels.cu:103-114): exact for a power-of-two cube at this depth
            ns = 1024.0 / 2**L
            cx = np.round((vox["x"].astype(np.float64) - r["X"] * ns) / ns * 128 - 0.5).astype(np.int64)
            assert ((cx >= 0) & (cx < 128)).all()
            assert np.allclose(vox["x"], r["X"] * ns + ns * (cx + 0.5) / 128, rtol=0, atol=0)
    assert total == 1_000_000


def test_chunk_and_heap_accounting_identities(config1):
    _, _, o, cn = config1
    s = o.stats()
    assert s.numAllocatedChunks == s.numChunksPoints == cn.records["chunksPoints"].sum()
    grids = s.numInner if s.numInner else 1
    voxel_chunks = int(cn.records["chunksVoxels"].sum())
    assert s.allocatedBytes_persistent == 16 + 262160 * grids + 16032 * (s.chunkPoolSize + voxel_chunks)


def test_topology_and_leaf_contents_do_not_depend_on_batching():
    pts, mn, mx = data.terrain(600_000)
    pts = pts.copy()
    box = ((0.0, 0.0, 0.0), (8192.0, 8192.0, 8192.0))      # power-of-two cube around the terrain
    a = build([pts], box).canon()
    b = build([pts[:100_000], pts[100_000:100_001], pts[100_001:450_000], pts[450_000:]], box).canon()
    assert len(a.records) == len(b.records)
    for f in ("level", "X", "Y", "Z", "name", "numPoints", "hashPoints", "isLeaf"):
        assert (a.records[f] == b.records[f]).all(), f
    inner = (a.records["isLeaf"] == 0) & (a.records["level"] > 0)
    # the root keeps one voxel per cell per "epoch" (its grid is wiped when it splits), so only
    # non-root inner nodes have batching-independent voxel sets
    assert (a.records["hashVoxelPos"][inner] == b.records["hashVoxelPos"][inner]).all()


def test_leaf_capacity_is_50000_inclusive():
    rng = np.random.default_rng(0)
    xyz = (rng.random((50_001, 3)) * 16).astype(np.float32)
    pts = make_points(xyz, np.full(50_001, 0xFF00FF00, dtype=np.uint32))
    box = ((0.0, 0.0, 0.0), (16.0, 16.0, 16.0))
    o = build([pts[:50_000]], box)
    assert o.stats().numNodes == 1 and o.stats().numPoints == 50_000
    o.add_batch(pts[50_000:])
    s = o.stats()
    assert s.numNodes == 9 and s.numPoints == 50_001 and s.numInner == 1
    # the 50 chunks of the old root went back to the pool and were reused: nothing new on the heap for points
    assert s.chunkPoolSize == max(50, s.numAllocatedChunks)


def test_root_grid_is_wiped_when_the_root_splits():
    # voxels.cu:370-382 clears the grid of every split node, including the root's populated one:
    # the root then holds one voxel per cell from before the split AND one per cell from the re-sampling
    pts, mn, mx = data.uniform_cube(60_000, size=64.0, seed=5)
    o = build([pts[:40_000], pts[40_000:]], (mn, mx))
    cn = o.canon()
    root = cn.records[0]
    (X, pX), (Y, pY), (Z, pZ) = quantize(pts, 64.0)
    sh = np.uint64(21)
    def ncells(sel):
        c = ((pX[sel] >> sh) & np.uint64(127)) | (((pY[sel] >> sh) & np.uint64(127)) << np.uint64(7)) | (((pZ[sel] >> sh) & np.uint64(127)) << np.uint64(14))
        return len(np.unique(c))
    first = np.arange(60_000) < 40_000
    assert root["numVoxels"] == ncells(first) + ncells(np.ones(60_000, bool))


def test_empty_and_single_point_batches():
    box = ((0.0, 0.0, 0.0), (8.0, 8.0, 8.0))
    o = build([np.zeros(0, dtype=oracle.POINT_DTYPE)], box)
    s = o.stats()
    assert s.batchletIndex == 1 and s.numPoints == 0 and s.numNodes == 1 and s.allocatedBytes_persistent == 16 + 262160
    one = make_points(np.array([[1.0, 2.0, 3.0]], dtype=np.float32), np.array([0xFF123456], dtype=np.uint32))
    o.add_batch(one)
    s = o.stats()
    assert s.numPoints == 1 and s.numAllocatedChunks == 1 and s.allocatedBytes_persistent == 16 + 262160 + 2 * 16032
    cn = o.canon()
    assert cn.records[0]["numVoxels"] == 1
    v = cn.samples(0, voxels=True)[0]
    # cell centre of (1,2,3) in an 8-cube with 128 cells per axis: (c + 0.5) / 16
    assert (v["x"], v["y"], v["z"], v["color"]) == (1.03125, 2.03125, 3.03125, 0xFF123456)


def test_out_of_box_points_follow_the_reference_quirks():
    # on the max face X = 2^20: the child bit wraps to 0; negatives saturate to 0 (SURVEY.md §7.3-3)
    box = ((0.0, 0.0, 0.0), (16.0, 16.0, 16.0))
    rng = np.random.default_rng(1)
    xyz = (rng.random((60_000, 3)) * 16).astype(np.float32)
    xyz[0] = [16.0, 1.0, 1.0]
    xyz[1] = [-3.0, 15.0, 15.0]
    pts = make_points(xyz, np.arange(60_000, dtype=np.uint32))
    cn = build([pts], box).canon()
    leaves = cn.records[cn.records["isLeaf"] == 1]
    def leaf_of(color):
        for k, r in enumerate(cn.records):
            if r["isLeaf"] and (cn.samples(k)["color"] == color).any():
                return r
    assert leaf_of(0)["X"] == 0          # 16.0 -> X = 2^20 -> bit 19 is 0 -> low octant
    assert leaf_of(1)["X"] == 0          # negative -> saturates to 0
    assert leaves["numPoints"].sum() == 60_000


GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_kernels.npz")


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="golden digests not generated yet (tests/golden/make_golden.py on a GPU)")
def test_oracle_matches_golden_digests_from_the_reference_kernels():
    import make_golden_cases as cases
    g = np.load(GOLDEN)
    for name, batches, box, _cam in cases.cases():
        if ("%s/rcp" % name) in g:
            rcp = float(g["%s/rcp" % name])
        else:
            rcp = 0.0
        o = build(batches, box, rcp)
        rec = o.canon().records
        ref = g["%s/records" % name]
        assert len(rec) == len(ref), name
        for f in rec.dtype.names:
            if f in ("nodeIndex", "_pad"):
                continue
            assert (rec[f] == ref[f]).all(), (name, f)
        s = o.stats()
        for f, v in zip(oracle.STATS_FIELDS, g["%s/stats" % name]):
            assert int(getattr(s, f)) == int(v), (name, f)
        # the frame the reference's kernel_render drew of that octree (same Uniforms bytes): the LOD cut of the CPU
        # rasteriser must be the reference's, and so must the depth of every pixel — except where a sample sits within
        # an ulp of a pixel edge (1/w is MUFU.RCP on the device, a correctly rounded reciprocal here: DESIGN.md §6).
        # Colours are not compared: which point donates a voxel's colour is a race in the reference.
        H, W = g["%s/framebuffer" % name].shape
        fb, rs, _flags = o.canon().render(g["%s/uniforms" % name].tobytes(), W, H)
        want = g["%s/visible" % name]
        assert [rs.numVisibleNodes, rs.numVisibleInner, rs.numVisibleLeaves, rs.numVisiblePoints, rs.numVisibleVoxels] == [int(v) for v in want], name
        depth_mismatch = float(((fb >> np.uint64(32)) != (g["%s/framebuffer" % name] >> np.uint64(32))).mean())
        assert depth_mismatch < 2e-3, (name, depth_mismatch)
