"""GPU tests of octree files (run with -m gpu on an H100): simlod_save_octree against its restatement and the export,
simlod_load_octree as a round trip (the same octree, exports and frames), resumption (saving after k batches, loading
into a fresh context and inserting the rest equals never stopping), octrees of the reference kernels in both
directions, every validation rule, and the save's promise to write nothing into the context."""
import hashlib
import os

import numpy as np
import pytest

import octree_file_restatement as F
import oracle
from simlod_b200 import SimLOD, SimlodError, api, camera, data
from test_export_gpu import (buffer_digests, export_digest, reference_result, terrain_ragged_stream, uniform_stream,
                             use_reference)

pytestmark = pytest.mark.gpu

HEAP = 12 << 30
RESUME_KEEP = [f for f in oracle.STATS_FIELDS if f not in ("numAllocatedChunks", "chunkPoolSize", "allocatedBytes_persistent")]
SWEEP = ["numNodes", "numInner", "numLeaves", "numNonemptyLeaves", "numPoints", "numVoxels", "numChunksPoints", "numChunksVoxels",
         "batchletIndex", "numPointsProcessed"]


def make_sim(heap=HEAP):
    return SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=heap)


@pytest.fixture(scope="module")
def sim():
    s = make_sim()
    yield s
    s.close()


@pytest.fixture(scope="module")
def other():
    """a second context with a different heap size: loads land at other addresses"""
    s = make_sim(HEAP - (1 << 30))
    yield s
    s.close()


def build(sim, batches, box, reference=False):
    use_reference(sim, reference)
    try:
        sim.set_box(*box)
        sim.reset()
        sim.insert_batches(batches)
    finally:
        use_reference(sim, False)
    assert sim.stats().dbg == 0


def canon(sim):
    return oracle.canon_from_image(*sim.download_octree())


def expected_file(sim):
    st = sim.stats()
    return F.file_bytes(*sim.download_octree(), sim.uniforms.boxMin, sim.uniforms.boxMax, st.batchletIndex, st.numPointsProcessed)


def check_file_is_the_export(sim, path):
    buf = open(path, "rb").read()
    assert buf == expected_file(sim), "saved file differs from the restatement"
    h, nodes, counters, samples = F.decode(buf)
    e = sim.export_octree(None, device="cpu")
    assert nodes.tobytes() == e.nodes.tobytes() and samples.tobytes() == e.samples.tobytes()
    hdr = api.read_octree_header(path)
    assert bytes(hdr.info) == bytes(e.info)
    # the sections are memmap-able at the header's offsets
    mm = np.memmap(path, dtype=api.EXPORT_NODE_DTYPE, mode="r", offset=hdr.records_offset, shape=(hdr.info.num_nodes,))
    assert mm.tobytes() == e.nodes.tobytes()
    return buf


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged"])
def test_saved_file_is_the_export(sim, tmp_path, name):
    batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    info, ms = sim.save_octree(path)
    assert ms > 0 and info.num_nodes == sim.stats().numNodes
    check_file_is_the_export(sim, path)


def frames(sim, box):
    out = []
    for hqs, bbox, by_node in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)):
        sim.set_settings(useHighQualityShading=hqs, showBoundingBox=bbox, colorByNode=by_node)
        for name, (view, proj) in (("autofocus", camera.autofocus(box, sim.width, sim.height)),
                                   ("close", camera.orbit_camera(0.4, -0.3, float(np.linalg.norm(box)) * 0.08,
                                                                 (box[0] * 0.55, box[1] * 0.45, box[2] * 0.3), sim.width, sim.height))):
            sim.set_camera(view, proj)
            sim.render()
            st = sim.stats()
            e = sim.export_view(device="cpu")
            out.append((name, hqs, bbox, by_node, sim.framebuffer().tobytes(), sim.surface().tobytes(),
                        tuple(getattr(st, f) for f in ("numVisibleNodes", "numVisibleInner", "numVisibleLeaves", "numVisiblePoints", "numVisibleVoxels")),
                        e.nodes.tobytes(), e.samples.tobytes()))
    sim.set_settings(useHighQualityShading=0, showBoundingBox=0, colorByNode=0)
    return out


def exports(sim):
    top = sim.export_octree(None, device="cpu")
    out = [(None, top.nodes.tobytes(), top.samples.tobytes(), bytes(top.info))]
    m = top.info.max_level
    for d in sorted({0, 1, 3, m, m + 1}):
        e = sim.export_octree(d, device="cpu")
        out.append((d, e.nodes.tobytes(), e.samples.tobytes(), bytes(e.info)))
    return out


def round_trip(sim, other, batches, box, tmp_path):
    build(sim, batches, box)
    path = str(tmp_path / "a.octree")
    sim.save_octree(path)
    st_a, cn_a = sim.stats(), canon(sim)
    ex_a, fr_a = exports(sim), frames(sim, box[1])
    other.load_octree(path)
    st_b = other.stats()
    assert tuple(other.uniforms.boxMin) == tuple(sim.uniforms.boxMin) and tuple(other.uniforms.boxMax) == tuple(sim.uniforms.boxMax)
    diffs = oracle.compare_canon(canon(other), cn_a) + oracle.compare_stats(st_b, st_a, SWEEP)
    assert not diffs, "\n".join(diffs)
    assert st_b.dbg == 0 and st_b.allocatedBytes_persistent <= st_a.allocatedBytes_persistent
    assert st_b.numAllocatedChunks == st_b.chunkPoolSize == st_b.numChunksPoints
    assert st_b.allocatedBytes_momentary == st_a.allocatedBytes_momentary
    assert exports(other) == ex_a
    fr_b = frames(other, box[1])
    for a, b in zip(fr_a, fr_b):
        assert a == b, "frame %s (hqs %d, box %d, by node %d) differs after the round trip" % a[:4]
    path2 = str(tmp_path / "b.octree")
    other.save_octree(path2)
    assert open(path2, "rb").read() == open(path, "rb").read()


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged"])
def test_round_trip_is_the_same_octree(sim, other, tmp_path, name):
    batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
    round_trip(sim, other, batches, box, tmp_path)


def test_round_trip_of_a_36m_device_generated_terrain(sim, other, tmp_path):
    n = 36_000_000
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        sim.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.reset()
        sim.insert_device(dptr, n)
    finally:
        sim.device_free(dptr)
    assert sim.stats().dbg == 0
    path = str(tmp_path / "t36.octree")
    sim.save_octree(path)
    check_file_is_the_export(sim, path)
    other.load_octree(path)
    diffs = oracle.compare_canon(canon(other), canon(sim)) + oracle.compare_stats(other.stats(), sim.stats(), SWEEP)
    assert not diffs, "\n".join(diffs)
    assert exports(other) == exports(sim)


def far_box_stream():
    """a box far from the origin: neighbouring voxel centres share a float from level 8 on"""
    pts, _, _ = data.uniform_cube(1_500_000, size=1000.0, seed=13)
    pts["x"] += np.float32(500000.0)
    pts["y"] += np.float32(4000000.0)
    box = ((500000.0, 4000000.0, 0.0), (501000.0, 4001000.0, 1000.0))
    return np.split(pts, [700_000, 1_000_000]), box


def deep_cluster_stream():
    """a dense cluster inside a 64-unit box: inner nodes down to level 17 and deeper, where voxel centres collide"""
    rng = np.random.default_rng(17)
    n = 400_000
    from simlod_b200 import make_points
    xyz = np.float32(37.3) + rng.random((n, 3), dtype=np.float32) * np.float32(64.0 / 2 ** 18)
    xyz[: n // 4] = rng.random((n // 4, 3), dtype=np.float32) * np.float32(64.0)
    pts = make_points(xyz, rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32))
    return np.split(pts, [150_000, 250_000]), ((0.0, 0.0, 0.0), (64.0, 64.0, 64.0))


@pytest.mark.parametrize("name", ["far_box", "deep_cluster"])
def test_round_trip_and_resume_where_voxel_centres_collide(sim, other, tmp_path, name):
    batches, box = {"far_box": far_box_stream, "deep_cluster": deep_cluster_stream}[name]()
    build(sim, batches, box)
    if name == "deep_cluster":
        e = sim.export_octree(None, device="cpu")
        assert e.nodes["level"][e.nodes["first_child"] >= 0].max() >= 17
    round_trip(sim, other, batches, box, tmp_path)
    o = oracle.Oracle(box[0], box[1], float(sim.device_rcp(max(np.subtract(box[1], box[0])))))
    for b in batches:
        o.add_batch(b)
    build(sim, batches, box)
    st_full, cn_full = sim.stats(), canon(sim)
    build(sim, batches[:1], box)
    path = str(tmp_path / "k.octree")
    sim.save_octree(path)
    other.load_octree(path)
    other.insert_batches(batches[1:])
    st, cn = other.stats(), canon(other)
    diffs = (oracle.compare_canon(cn, cn_full) + oracle.compare_stats(st, st_full, RESUME_KEEP) +
             oracle.compare_canon(cn, o.canon()) + oracle.compare_stats(st, o.stats(), RESUME_KEEP))
    assert not diffs, "\n".join(diffs)
    # the colour checker finds a voxel's cell from its position, so where centres collide it cannot tell some cells apart:
    # the resumed octree must fare exactly as the uninterrupted one, and with distinct centres both must pass
    full_colors = o.check_voxel_colors(cn_full)
    assert o.check_voxel_colors(cn) == full_colors
    if name == "far_box":
        assert full_colors == 0


def small_batches():
    pts, mn, mx = data.uniform_cube(120_000, size=64.0, seed=5)
    return np.split(pts, np.cumsum([20_000, 20_000, 10_000, 1, 30_000])), (mn, mx)


def resume_cases():
    t, tbox, _ = terrain_ragged_stream()
    s, sbox = small_batches()
    # (terrain, k = 1): leaves loaded with points split later, new voxels land in loaded grids
    # (small batches, k = 2): the root is a leaf with voxels at save time and splits after the load
    return {"terrain_k1": (t, tbox, 1), "terrain_k4": (t, tbox, 4), "small_root_leaf_k2": (s, sbox, 2)}


@pytest.mark.parametrize("case", ["terrain_k1", "terrain_k4", "small_root_leaf_k2"])
def test_resume_equals_never_stopping(sim, other, tmp_path, case):
    batches, box, k = resume_cases()[case]
    # the terrain stream's oracle takes the device's MUFU.RCP of the cube size (as test_export_gpu.py does)
    rcp = float(sim.device_rcp(max(np.subtract(box[1], box[0])))) if case.startswith("terrain") else 0.0
    o = oracle.Oracle(box[0], box[1], rcp)
    for b in batches:
        o.add_batch(b)
    build(sim, batches, box)
    st_full, cn_full = sim.stats(), canon(sim)
    build(sim, batches[:k], box)
    if case.startswith("small"):
        st = sim.stats()
        assert st.numNodes == 1 and st.numVoxels == 0 and sim.export_octree(None, device="cpu").info.num_voxels > 0
    path = str(tmp_path / "k.octree")
    sim.save_octree(path)
    other.load_octree(path)
    other.insert_batches(batches[k:])
    st, cn = other.stats(), canon(other)
    assert st.dbg == 0
    diffs = (oracle.compare_canon(cn, cn_full) + oracle.compare_stats(st, st_full, RESUME_KEEP) +
             oracle.compare_canon(cn, o.canon()) + oracle.compare_stats(st, o.stats(), RESUME_KEEP))
    assert not diffs, "\n".join(diffs)
    assert o.check_voxel_colors(cn) == 0


def test_reference_kernels_octree_saves_loads_and_continues(sim, other, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    k = 2
    o = oracle.Oracle(box[0], box[1], float(sim.device_rcp(max(np.subtract(box[1], box[0])))))
    for b in batches:
        o.add_batch(b)
    # the reference kernels' octree, saved: matches the stored digests of its export
    build(sim, batches, box, reference=True)
    path = str(tmp_path / "ref.octree")
    sim.save_octree(path)
    _, nodes, _, samples = F.decode(open(path, "rb").read())
    ref = reference_result("export_terrain_ragged", lambda: export_digest(nodes, samples))
    got = export_digest(nodes, samples)
    assert got == ref, "saved reference octree vs stored export digests"
    # a prefix built by the reference kernels, loaded and continued by ours
    build(sim, batches[:k], box, reference=True)
    sim.save_octree(path)
    other.load_octree(path)
    other.insert_batches(batches[k:])
    diffs = oracle.compare_canon(canon(other), o.canon()) + oracle.compare_stats(other.stats(), o.stats(), RESUME_KEEP)
    assert not diffs, "\n".join(diffs)
    # our prefix, loaded, continued by the reference kernels
    build(sim, batches[:k], box)
    sim.save_octree(path)
    other.load_octree(path)
    use_reference(other, True)
    try:
        other.insert_batches(batches[k:])
    finally:
        use_reference(other, False)
    diffs = oracle.compare_canon(canon(other), o.canon()) + oracle.compare_stats(other.stats(), o.stats(), RESUME_KEEP)
    assert not diffs, "\n".join(diffs)


def side_table_bytes():
    """the head of the momentary buffer that persists across launches: kernel_construct's control block and its per-node
    side tables (construct_layout.cuh, up to OFF_DIRTYLEAF)"""
    tab, off = 263168, 4096

    def a256(x):
        return (x + 255) & ~255
    for width in (4, 4, 8, 4, 4, 8, 8):            # first child, parent, grid, leaf row, split state, voxel tail, directory
        off = a256(off + tab * width)
    return off


def context_digest(sim):
    b = sim.buffers()
    d = buffer_digests(sim)
    d.pop("momentary")
    d.pop("renderbuffer")
    d["side_tables"] = hashlib.sha256(sim.memcpy_dtoh(b.momentary, side_table_bytes()).tobytes()).hexdigest()
    d["uniforms"] = sim.uniforms_bytes()
    d["ring"] = hashlib.sha256(sim.memcpy_dtoh(b.ring + 2 * api.MAX_BATCH_SIZE * 16, 16 * 1000).tobytes()).hexdigest()
    return d


def mutate(buf, fn):
    h, nodes, counters, samples = F.decode(buf)
    nodes, counters, samples = nodes.copy(), counters.copy(), samples.copy()
    fn(nodes, counters, samples)
    class Info:
        pass
    info = Info()
    info.max_level, info.num_points, info.num_voxels = h["max_level"], h["num_points"], h["num_voxels"]
    return F.encode(nodes, samples, info, counters, h["box_min"], h["box_max"], h["batchlet_index"], h["num_points_processed"])


def first_inner(nodes, level=1):
    return int(np.nonzero((nodes["first_child"] >= 0) & (nodes["level"] == level))[0][0])


def sample_range(nodes, i, voxels):
    a = int(nodes["sample_offset"][i]) + (int(nodes["num_points"][i]) if voxels else 0)
    return a, a + int(nodes["num_voxels"][i] if voxels else nodes["num_points"][i])


def bad_first_child(n, c, s):
    i = first_inner(n)
    n["first_child"][i] += 8


def bad_child_x(n, c, s):
    i = first_inner(n)
    n["X"][int(n["first_child"][i]) + 1] ^= 1


def bad_child_name(n, c, s):
    i = first_inner(n)
    nm = bytearray(n["name"][int(n["first_child"][i]) + 3])
    nm[2] = ord("7")
    n["name"][int(n["first_child"][i]) + 3] = bytes(nm)


def bad_sample_offset(n, c, s):
    n["sample_offset"][5] += 1


def inner_counter_50000(n, c, s):
    c[first_inner(n)] = 50_000


def voxel_one_ulp(n, c, s):
    a, _ = sample_range(n, first_inner(n), True)
    s["x"][a] = np.nextafter(s["x"][a], np.float32(np.inf))


def point_in_sibling(n, c, s):
    leaves = np.nonzero((n["first_child"] < 0) & (n["num_points"] > 0))[0]
    i = int(leaves[0])
    a, _ = sample_range(n, i, False)
    # one leaf edge along x: into the neighbouring leaf at the same level, inside the box
    edge = np.float32(64.0 / (1 << int(n["level"][i])))
    s["x"][a] = s["x"][a] + edge if int(n["X"][i]) % 2 == 0 else s["x"][a] - edge


def duplicated_voxel(n, c, s):
    a, b = sample_range(n, first_inner(n), True)
    s[a + 1] = s[a]


BEFORE_WRITE = {"first_child": bad_first_child, "child_x": bad_child_x, "child_name": bad_child_name,
                "sample_offset": bad_sample_offset, "inner_counter": inner_counter_50000}
SAMPLE_STAGE = {"voxel_ulp": voxel_one_ulp, "point_in_sibling": point_in_sibling, "duplicate_voxel": duplicated_voxel}


@pytest.fixture(scope="module")
def saved(sim, tmp_path_factory):
    """an octree of the uniform 64^3 stream, with inner nodes at level 1 and leaves below, saved"""
    pts, mn, mx = data.uniform_cube(600_000, size=64.0, seed=9)
    build(sim, [pts], (mn, mx))
    path = str(tmp_path_factory.mktemp("saved") / "u.octree")
    sim.save_octree(path)
    return path, (mn, mx)


def test_errors_before_any_write_leave_the_context_unchanged(sim, other, saved, tmp_path):
    path, box = saved
    buf = open(path, "rb").read()
    terrain, tbox, _ = terrain_ragged_stream()
    build(other, terrain[:2], tbox)
    other.upload_batch(terrain[2])                     # a batch waiting in the ring
    before = context_digest(other)
    for name, fn in BEFORE_WRITE.items():
        p = str(tmp_path / (name + ".octree"))
        open(p, "wb").write(mutate(buf, fn))
        with pytest.raises(SimlodError) as e:
            other.load_octree(p)
        assert e.value.code == -2 and p in str(e.value), (name, str(e.value))
        assert context_digest(other) == before, name
    # a heap too small for the image
    small = make_sim(heap=250 << 20)                   # 50 MB above the capacity guard's margin
    try:
        build(sim, terrain, tbox)
        big = str(tmp_path / "big.octree")
        sim.save_octree(big)
        snap = context_digest(small)
        with pytest.raises(SimlodError) as e:
            small.load_octree(big)
        assert e.value.code == -5 and big in str(e.value)
        assert context_digest(small) == snap
    finally:
        small.close()
    # a swapped-in construct module
    use_reference(other, True)
    try:
        with pytest.raises(SimlodError) as e:
            other.load_octree(path)
        assert e.value.code == -4
    finally:
        use_reference(other, False)
    assert context_digest(other) == before
    other.update_octree()                               # the pending batch is still consumed as before
    assert other.stats().batchletIndex == 3


def test_sample_errors_leave_an_empty_octree(other, saved, tmp_path):
    path, box = saved
    buf = open(path, "rb").read()
    pts, mn, mx = data.uniform_cube(200_000, size=64.0, seed=1)
    for name, fn in SAMPLE_STAGE.items():
        p = str(tmp_path / (name + ".octree"))
        open(p, "wb").write(mutate(buf, fn))
        with pytest.raises(SimlodError) as e:
            other.load_octree(p)
        assert e.value.code == -2 and p in str(e.value), (name, str(e.value))
        st = other.stats()
        assert st.numNodes == 1 and st.numPoints == 0 and st.batchletIndex == 0, name
        h = api.read_octree_header(p)
        assert tuple(other.uniforms.boxMax) == tuple(h.box_max)
        other.insert_batches([pts])                     # the empty octree takes new batches
        o = oracle.Oracle(other.uniforms.boxMin, other.uniforms.boxMax)
        o.add_batch(pts)
        diffs = oracle.compare_canon(canon(other), o.canon()) + oracle.compare_stats(other.stats(), o.stats())
        assert not diffs, name + "\n" + "\n".join(diffs)


def test_save_writes_nothing_into_the_context(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    view, proj = camera.autofocus(box[1], sim.width, sim.height)
    sim.set_camera(view, proj)
    sim.render()
    before = buffer_digests(sim)
    sim.save_octree(str(tmp_path / "s.octree"))
    assert buffer_digests(sim) == before


def test_save_refuses_an_octree_with_dropped_samples(sim, tmp_path):
    pts, mn, mx = data.uniform_cube(10_000, size=8.0, seed=2)
    build(sim, [pts], (mn, mx))
    b = sim.buffers()
    st = sim.stats()
    st.dbg = 2
    sim.memcpy_htod(b.stats, np.frombuffer(bytes(st), dtype=np.uint8))
    with pytest.raises(SimlodError) as e:
        sim.save_octree(str(tmp_path / "d.octree"))
    assert e.value.code == -2 and "d.octree" in str(e.value)
    assert not os.path.exists(str(tmp_path / "d.octree"))


def test_a_failed_save_keeps_the_existing_file(sim, tmp_path):
    pts, mn, mx = data.uniform_cube(100_000, size=8.0, seed=3)
    build(sim, [pts], (mn, mx))
    path = tmp_path / "keep.octree"
    sim.save_octree(str(path))
    good = path.read_bytes()
    os.mkdir(str(path) + ".tmp")                       # the temporary file cannot be created
    with pytest.raises(SimlodError) as e:
        sim.save_octree(str(path))
    assert e.value.code == -2 and str(path) in str(e.value)
    assert path.read_bytes() == good
