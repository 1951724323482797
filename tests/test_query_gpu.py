"""GPU tests of the region query (run with -m gpu on an H100): simlod_query_region against its restatement
(query_restatement: the export of the same device image, filtered sample by sample with no hierarchy shortcut, byte
for byte), against a brute-force filter of the source points, and its protocol (size query, capacity, malformed
regions, no writes into the context's buffers)."""
import os

import numpy as np
import pytest

import export_restatement as R
import oracle
import query_restatement as Q
from simlod_b200 import Region, SimLOD, SimlodError, api, camera, data
from test_export_cpu import sorted_points
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def cube(sim, box):
    """(boxMin, boxMax, the device's reciprocal of the cube size) for the restatement."""
    size = float(np.max(np.subtract(box[1], box[0]).astype(np.float32)))
    return box[0], box[1], sim.device_rcp(size)


def frustum_planes(view, proj):
    """The six half-spaces -w <= x, y, z <= w of clip = proj * view * p, as rows (nx, ny, nz, d)."""
    m = (np.asarray(proj, dtype=np.float32) @ np.asarray(view, dtype=np.float32)).astype(np.float32)
    return np.array([m[3] + m[0], m[3] - m[0], m[3] + m[1], m[3] - m[1], m[3] + m[2], m[3] - m[2]], dtype=np.float32)


def regions_of(box, points, full_nodes):
    mn = np.asarray(box[0], dtype=np.float64)
    ext = np.asarray(box[1], dtype=np.float64) - mn
    size = float(ext.max())
    leaves = full_nodes[(full_nodes["flags"] & api.EXPORT_LEAF != 0) & (full_nodes["num_points"] > 0)]
    leaf = leaves[np.argmax(leaves["level"])]
    edge = size / 2.0 ** int(leaf["level"])
    lo = mn + edge * np.array([leaf["X"], leaf["Y"], leaf["Z"]], dtype=np.float64)
    p = points[len(points) // 3]
    stored = (float(p["x"]), float(p["y"]), float(p["z"]))
    c = mn + ext / 2
    s = np.sqrt(0.5)
    along = s * c[0] + s * c[1]                              # the corridor runs along (1, 1, 0) through the centre
    across = s * c[0] - s * c[1]
    w = size / 400.0
    return {
        "inside_leaf": Region.box(lo + 0.02 * edge, lo + 0.98 * edge),
        "tenth": Region.box(mn - 1.0, (mn[0] + 0.1 * ext[0], mn[1] + size + 1.0, mn[2] + size + 1.0)),
        "everything": Region.box(mn - 1.0, mn + size + 1.0),
        "disjoint": Region.box(mn + 2.0 * size, mn + 3.0 * size),
        "degenerate": Region.box(stored, stored),
        "sphere": Region.sphere(stored, size / 50.0),
        "corridor": Region.planes([[s, -s, 0, -(across - w)], [-s, s, 0, across + w], [s, s, 0, -(along - 0.3 * size)], [-s, -s, 0, along + 0.3 * size],
                                   [0, 0, 1, -mn[2]], [0, 0, -1, mn[2] + size]]),
        "frustum": Region.planes(frustum_planes(*camera.autofocus(box[1], 640, 360))),
    }


SMALL = ("inside_leaf", "degenerate", "sphere")


def check_queries(sim, box, points, names=None, depths=None):
    """Every region at every depth: byte-identical to the restatement of the image; at depth None also the brute-force
    filter of the source points as a multiset."""
    image = sim.download_octree()
    cb = cube(sim, box)
    exports = {None: R.export_image(*image)}
    top = exports[None][2].max_level
    regions = regions_of(box, points, exports[None][0])
    total = len(points)
    for depth in (sorted({0, 1, 3, top}) if depths is None else depths):
        exports[depth] = R.export_image(*image, depth)
    for name in names or regions:
        region = regions[name]
        for depth, ex in exports.items():
            label = "%s depth %s" % (name, depth)
            want, n_points, n_voxels = Q.query_export(ex, region, depth, *cb)
            got, info = sim.query_region(region, depth, device="cpu")
            assert (info.num_samples, info.num_points, info.num_voxels) == (len(want), n_points, n_voxels), label
            assert got.tobytes() == want.tobytes(), label
            assert info.max_level == top and info.num_samples <= info.samples_tested <= ex[2].num_samples, label
            if depth is None:
                if len(want) < 10_000_000:                   # larger results: the byte comparison above and the count below
                    assert np.array_equal(sorted_points(got), sorted_points(Q.brute_force(points, region, *cb))), label
                assert info.num_voxels == 0
                if name in SMALL:
                    assert info.samples_tested < total // 4 and info.nodes_visited >= 1, label
                if name == "everything":
                    assert info.samples_tested == total and info.num_samples == int(Q.in_cube(points, *cb).sum())
                if name == "degenerate":
                    assert info.num_samples >= 1
                if name in ("tenth", "everything", "sphere", "corridor"):
                    assert info.num_samples > 0, label
            if name == "disjoint":
                assert (info.num_samples, info.samples_tested, info.nodes_visited) == (0, 0, 0), label


@pytest.mark.parametrize("stream", [uniform_stream, terrain_ragged_stream], ids=["uniform_1m", "terrain_ragged"])
def test_query_equals_the_restatement_and_brute_force(sim, stream):
    batches, box, _ = stream()
    build(sim, batches, box)
    check_queries(sim, box, np.concatenate(batches))


def test_query_of_a_36m_device_generated_terrain_stream(sim):
    n = 36_000_000
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        sim.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.reset()
        sim.insert_device(dptr, n)
        points = sim.memcpy_dtoh(dptr, n * 16).view(api.POINT_DTYPE)
    finally:
        sim.device_free(dptr)
    assert sim.stats().dbg == 0 and sim.stats().numPointsProcessed == n
    check_queries(sim, ((0.0, 0.0, 0.0), data.TERRAIN_EXTENT), points, depths=(3,))


MARK = 0xABCD0000


def test_a_point_on_the_max_face_is_never_returned(sim):
    cloud, mn, mx = data.uniform_cube(400_000, size=256.0, seed=3)
    on_face = api.make_points(np.array([[256.0, 10.0, 10.0], [10.0, 256.0, 10.0]], dtype=np.float32), [MARK, MARK + 1])
    points = np.concatenate([cloud[:100_000], on_face, cloud[100_000:]])
    box = (mn, (256.0, 256.0, 256.0))
    build(sim, [points], box)
    image = sim.download_octree()
    stored = R.export_image(*image, 20)[1]                   # the points of every leaf
    assert (stored["color"] == MARK).sum() == 1              # the builder did store it (under a wrapped coordinate)
    for region in (Region.box((-1, -1, -1), (257, 257, 257)), Region.sphere((128, 128, 128), 1000.0),
                   Region.planes([[0, 0, 1, 5]])):
        got, info = sim.query_region(region, None, device="cpu")
        want, _, _ = Q.query_image(*image, region, None, *cube(sim, box))
        assert got.tobytes() == want.tobytes() and info.num_samples == len(points) - 2
        assert not ((got["color"] == MARK) | (got["color"] == MARK + 1)).any()
        assert Q.contains(region, on_face).all()             # the region does contain both points


def test_protocol(sim):
    torch = pytest.importorskip("torch")
    sim.set_box((0.0, 0.0, 0.0), (64.0, 64.0, 64.0))
    sim.reset()
    got, info = sim.query_region(Region.box((0, 0, 0), (64, 64, 64)), None, device="cpu")   # a fresh octree: an empty leaf root
    assert len(got) == 0 and (info.num_samples, info.samples_tested, info.nodes_visited, info.max_level) == (0, 0, 1, 0)

    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    region = Region.sphere((2400.0, 2100.0, 100.0), 400.0)
    for depth in (None, 3):
        info, _ = sim.query_region_into(region, depth, 0, 0)              # size query
        m = info.num_samples
        assert m > 1000
        a, ia = sim.query_region(region, depth, device="cpu")
        b, ib = sim.query_region(region, depth, device="cpu")
        assert a.tobytes() == b.tobytes() and bytes(ia) == bytes(ib) == bytes(info)
        t, it = sim.query_region(region, depth, device="cuda")
        assert isinstance(t, torch.Tensor) and t.is_cuda and tuple(t.shape) == (m, 4) and t.dtype == torch.float32
        assert t.cpu().numpy().tobytes() == a.tobytes() and bytes(it) == bytes(info)
        guard = 4096
        ds = sim.device_alloc(m * 16 + 2 * guard)
        try:
            pattern = np.full(m * 16 + 2 * guard, 0x5A, dtype=np.uint8)
            sim.memcpy_htod(ds, pattern)
            info0, _ = sim.query_region_into(region, depth, 0, m)         # size query: nothing written
            assert bytes(info0) == bytes(info)
            with pytest.raises(SimlodError) as err:                      # one short: refused, destination untouched
                sim.query_region_into(region, depth, ds + guard, m - 1)
            assert err.value.code == -2
            with pytest.raises(SimlodError) as err:
                sim.query_region_into(region, 21, ds + guard, m)
            assert err.value.code == -2
            with pytest.raises(SimlodError) as err:
                sim.query_region_into(region, depth, ds + guard + 8, m)
            assert err.value.code == -2
            assert (sim.memcpy_dtoh(ds, len(pattern)) == pattern).all()
            info2, ms = sim.query_region_into(region, depth, ds + guard, m)
            assert bytes(info2) == bytes(info) and ms > 0
            back = sim.memcpy_dtoh(ds, len(pattern))
            assert (back[:guard] == 0x5A).all() and (back[guard + m * 16:] == 0x5A).all()
            assert back[guard:guard + m * 16].tobytes() == a.tobytes()
        finally:
            sim.device_free(ds)


def malformed_regions():
    nan, inf = float("nan"), float("inf")
    out = {"kind_0": api.SimlodRegion(kind=0), "kind_4": api.SimlodRegion(kind=4),
           "box_min_above_max": Region.box((0, 5, 0), (1, 4, 1)), "box_nan": Region.box((0, nan, 0), (1, 1, 1)),
           "box_inf": Region.box((0, 0, 0), (1, inf, 1)), "sphere_negative": Region.sphere((0, 0, 0), -1.0),
           "sphere_nan_radius": Region.sphere((0, 0, 0), nan), "sphere_inf_center": Region.sphere((0, -inf, 0), 1.0),
           "plane_nan": Region.planes([[1, 0, 0, 0], [0, nan, 0, 0]])}
    for count in (0, 17):
        r = Region.planes([[1, 0, 0, 0]])
        r.num_planes = count
        out["planes_%d" % count] = r
    return out


def test_malformed_regions_are_refused(sim):
    sim.set_box((0.0, 0.0, 0.0), (64.0, 64.0, 64.0))
    sim.reset()
    launches = sim.launch_info()["launches"]
    for name, region in malformed_regions().items():
        with pytest.raises(SimlodError) as err:
            sim.query_region_into(region, None, 0, 0)
        assert err.value.code == -2, name
    assert sim.launch_info()["launches"] == launches         # refused before any launch
    unused = Region.planes([[1, 0, 0, 0]])
    unused.planes[5][1] = float("nan")                       # beyond num_planes: not part of the region
    sim.query_region_into(unused, None, 0, 0)


def test_query_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], sim.width, sim.height))
    sim.render()
    before = buffer_digests(sim)
    ring = sim.ring_slot(0, 1000).tobytes()
    for depth in (None, 2):
        for region in (Region.box((0, 0, 0), (5000, 5000, 500)), Region.sphere((1000, 1000, 50), 300.0)):
            sim.query_region(region, depth, device="cpu")
    assert buffer_digests(sim) == before and sim.ring_slot(0, 1000).tobytes() == ring
    # a query in the middle of a stream changes nothing that follows
    def run(with_query):
        sim.set_box(*box)
        sim.reset()
        sim.insert_batches(batches[:3])
        if with_query:
            sim.query_region(Region.box((0, 0, 0), (5000, 5000, 500)), None, device="cpu")
        sim.insert_batches(batches[3:])
        return sim.stats(), oracle.canon_from_image(*sim.download_octree())
    st_a, cn_a = run(True)
    st_b, cn_b = run(False)
    diffs = oracle.compare_canon(cn_a, cn_b) + oracle.compare_stats(st_a, st_b)
    assert not diffs, "\n".join(diffs)


def test_query_while_batches_are_pending_sees_the_last_completed_launch(sim):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for b in batches:
        sim.upload_batch(b)
    region = Region.sphere((256, 256, 256), 200.0)
    snapshots = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        done = sim.stats().batchletIndex
        if done < len(batches):
            image = sim.download_octree()
            got, info = sim.query_region(region, None, device="cpu")
            want, _, _ = Q.query_image(*image, region, None, mn, mx)
            assert got.tobytes() == want.tobytes()
            assert np.array_equal(sorted_points(got), sorted_points(Q.brute_force(np.concatenate(batches[:done]), region, mn, mx)))
            snapshots += 1
    assert snapshots >= 1


def test_query_of_the_reference_kernels_octree_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    points = np.concatenate(batches)
    names = ("inside_leaf", "tenth", "corridor", "frustum")
    if all(os.path.exists(p) for p in oracle.REF_CUBINS.values()):
        build(sim, batches, box, reference=True)          # the query reads the ABI only
        check_queries(sim, box, points, names=names, depths=(2,))
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    sim.save_octree(path)
    sim.reset()
    sim.load_octree(path)
    check_queries(sim, box, points, names=names, depths=(2,))
