"""GPU tests of the octree export (run with -m gpu on an H100): simlod_export_octree against its restatement
(export_restatement.export_image of the same device image, byte for byte), against the oracle builder and the
reference kernels, and its protocol (sizes, capacities, guard bytes, no writes into the context's buffers).

What the reference kernels' octree exports to is stored in tests/golden/export_reference.json; with
SIMLOD_RECORD_GOLDEN set the reference runs live and is recorded again (reference_golden.reference)."""
import hashlib
import json
import os

import numpy as np
import pytest

import export_restatement as R
import oracle
import reference_golden as golden
from simlod_b200 import SimLOD, SimlodError, api, camera, data
from test_export_cpu import check_structure, sorted_points

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def use_reference(sim, on):
    for p in (0, 2):
        sim.use_module(p, oracle.REF_CUBINS[p] if on else None)


def build(sim, batches, box, reference=False):
    use_reference(sim, reference)
    try:
        sim.set_box(*box)
        sim.reset()
        sim.insert_batches(batches)
    finally:
        use_reference(sim, False)
    st = sim.stats()
    assert st.dbg == 0
    return st


def image_canon(sim):
    return oracle.canon_from_image(*sim.download_octree())


def uniform_stream():
    pts, mn, mx = data.uniform_cube(1_000_000)
    return [pts], (mn, mx), 0.0


def terrain_ragged_stream():
    n = 3_300_000
    pts, mn, mx = data.terrain(n)
    sizes = [1_000_000, 1_000_000, 7, 0, 900_000, n - 2_900_007]
    return np.split(pts, np.cumsum(sizes)[:-1]), (mn, mx), None     # None: the device's MUFU.RCP of the cube size


STREAMS = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "export_reference.json")


def reference_result(key, run):
    """The reference kernels' result for `key`: run() live (and recorded) with SIMLOD_RECORD_GOLDEN set, else the stored one."""
    if golden.RECORD:
        return golden.reference(key, run)
    with open(GOLDEN) as f:
        stored = json.load(f)
    assert key in stored, "no stored reference result for %r in %s" % (key, GOLDEN)
    return stored[key]


def same_export(got, want, label):
    nodes, samples, info = got
    wn, ws, wi = want
    assert bytes(info) == bytes(wi), "%s: info %r != %r" % (label, tuple(getattr(info, f) for f, _ in info._fields_),
                                                            tuple(getattr(wi, f) for f, _ in wi._fields_))
    assert nodes.tobytes() == wn.tobytes(), "%s: node table differs" % label
    assert samples.tobytes() == ws.tobytes(), "%s: samples differ" % label


def sorted_positions(v):
    """Voxel positions (x, y, z bits) as (N, 3) uint32 rows in a canonical order."""
    a = np.ascontiguousarray(v).view(np.uint32).reshape(-1, 4)[:, :3]
    return a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))]


def device_export(sim, depth):
    e = sim.export_octree(depth, device="cpu")
    return e.nodes, e.samples, e.info


def check_all_depths(sim, points):
    """Full export and the cuts at 0, 1, 3, max_level, max_level + 1, byte-identical to the restatement of the image."""
    image = sim.download_octree()
    full = device_export(sim, None)
    same_export(full, R.export_image(*image), "full")
    check_structure(full[0], full[2])
    top = full[2].max_level
    for depth in sorted({0, 1, 3, top, top + 1}):
        got = device_export(sim, depth)
        same_export(got, R.export_image(*image, depth), "depth %d" % depth)
        if depth >= top:                                    # the deepest node is a leaf: the cut is the point set
            assert got[2].num_voxels == 0 and np.array_equal(sorted_points(got[1]), sorted_points(points))
    return full


@pytest.mark.parametrize("name", list(STREAMS))
def test_export_equals_the_restatement_and_the_oracle_builder(sim, name):
    batches, box, rcp = STREAMS[name]()
    build(sim, batches, box)
    points = np.concatenate(batches)
    nodes, samples, info = check_all_depths(sim, points)
    # the oracle builder on the same stream: identical node table, per node the same points and voxel positions
    o = oracle.Oracle(box[0], box[1], float(sim.device_rcp(max(np.subtract(box[1], box[0])))) if rcp is None else rcp)
    for b in batches:
        o.add_batch(b)
    on, osamp, oi = R.export_canon(o.canon())
    assert bytes(info) == bytes(oi) and nodes.tobytes() == on.tobytes()
    for i in range(len(nodes)):
        a, np_, nv = int(nodes["sample_offset"][i]), int(nodes["num_points"][i]), int(nodes["num_voxels"][i])
        assert np.array_equal(sorted_points(samples[a:a + np_]), sorted_points(osamp[a:a + np_]))
        assert np.array_equal(sorted_positions(samples[a + np_:a + np_ + nv]), sorted_positions(osamp[a + np_:a + np_ + nv]))
    assert o.check_voxel_colors(image_canon(sim)) == 0


def test_export_of_a_36m_device_generated_terrain_stream(sim):
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
    check_all_depths(sim, points)


def export_digest(nodes, samples):
    """sha256 of the node table, of the per-node sorted point sets and of the per-node sorted voxel positions."""
    hp, hv = hashlib.sha256(), hashlib.sha256()
    for i in range(len(nodes)):
        a, np_, nv = int(nodes["sample_offset"][i]), int(nodes["num_points"][i]), int(nodes["num_voxels"][i])
        hp.update(sorted_points(samples[a:a + np_]).tobytes())
        hv.update(sorted_positions(samples[a + np_:a + np_ + nv]).tobytes())
    return {"nodes": golden.sha256(nodes), "points": hp.hexdigest(), "voxel_positions": hv.hexdigest()}


def test_export_of_the_reference_kernels_octree(sim):
    """The export reads the ABI only: the reference kernels' octree of the ragged terrain stream exports to the same
    node table, point sets and voxel positions as ours."""
    batches, box, _ = terrain_ragged_stream()

    def run():
        build(sim, batches, box, reference=True)
        nodes, samples, _ = device_export(sim, None)
        same_export((nodes, samples, _), R.export_image(*sim.download_octree()), "reference kernels' octree vs restatement")
        return export_digest(nodes, samples)
    ref = reference_result("export_terrain_ragged", run)
    build(sim, batches, box)
    nodes, samples, _ = device_export(sim, None)
    golden.assert_same(export_digest(nodes, samples), ref, "export of ours vs of the reference kernels' octree")


def buffer_digests(sim):
    b, st = sim.buffers(), sim.stats()
    heap_used = int(sim.memcpy_dtoh(b.persistent + 8, 8).view(np.uint64)[0])
    return {name: hashlib.sha256(sim.memcpy_dtoh(ptr, size).tobytes()).hexdigest() for name, ptr, size in (
        ("nodes", b.nodes, b.nodes_bytes), ("heap", b.persistent, heap_used), ("momentary", b.momentary, b.momentary_bytes),
        ("renderbuffer", b.renderbuffer, b.renderbuffer_bytes), ("stats", b.stats, 112))}


def test_export_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    view, proj = camera.autofocus(box[1], sim.width, sim.height)
    sim.set_camera(view, proj)
    sim.render()
    before = buffer_digests(sim)
    for depth in (None, 0, 2):
        sim.export_octree(depth, device="cpu")
    assert buffer_digests(sim) == before

    # an export in the middle of a stream changes nothing that follows
    def run(with_export):
        sim.set_box(*box)
        sim.reset()
        sim.insert_batches(batches[:3])
        if with_export:
            sim.export_octree(None, device="cpu")
            sim.export_octree(1, device="cpu")
        sim.insert_batches(batches[3:])
        sim.render()
        return sim.stats(), image_canon(sim), sim.framebuffer()
    st_a, cn_a, fb_a = run(True)
    st_b, cn_b, fb_b = run(False)
    diffs = oracle.compare_canon(cn_a, cn_b) + oracle.compare_stats(st_a, st_b, oracle.STATS_FIELDS + [
        "numVisibleNodes", "numVisibleInner", "numVisibleLeaves", "numVisiblePoints", "numVisibleVoxels", "dbg"])
    assert not diffs, "\n".join(diffs)
    assert ((fb_a >> np.uint64(32)) == (fb_b >> np.uint64(32))).all()
    if st_a.numVisibleVoxels == 0:            # which point colours a voxel is a race in the builder
        assert (fb_a == fb_b).all()


def test_snapshot_while_batches_are_pending(sim):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for b in batches:
        sim.upload_batch(b)
    snapshots = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        if sim.stats().batchletIndex < len(batches):
            image = sim.download_octree()
            same_export(device_export(sim, None), R.export_image(*image), "snapshot after %d batches" % sim.stats().batchletIndex)
            same_export(device_export(sim, 2), R.export_image(*image, 2), "cut snapshot")
            snapshots += 1
    assert snapshots >= 1
    o = oracle.Oracle(mn, mx)
    for b in batches:
        o.add_batch(b)
    st = sim.stats()
    diffs = oracle.compare_canon(image_canon(sim), o.canon()) + oracle.compare_stats(st, o.stats())
    assert not diffs and st.dbg == 0, "\n".join(diffs)
    nodes, _, info = device_export(sim, None)
    on, _, oi = R.export_canon(o.canon())
    assert nodes.tobytes() == on.tobytes() and bytes(info) == bytes(oi)


def test_protocol(sim):
    torch = pytest.importorskip("torch")
    sim.set_box((0.0, 0.0, 0.0), (64.0, 64.0, 64.0))
    sim.reset()
    e = sim.export_octree(None, device="cpu")            # a fresh octree: one leaf root without samples
    assert e.info.num_nodes == 1 and e.info.num_samples == 0 and len(e.samples) == 0
    assert e.nodes["flags"][0] == api.EXPORT_LEAF | api.EXPORT_SAMPLED and e.nodes["parent"][0] == -1 and e.nodes["first_child"][0] == -1
    assert e.nodes["name"][0] == b"r"

    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    for depth in (None, 3):
        info, _ = sim.export_octree_into(depth, 0, 0, 0, 0)           # size query
        n, m = info.num_nodes, info.num_samples
        a = device_export(sim, depth)
        b = device_export(sim, depth)
        same_export(a, b, "two exports")
        assert bytes(a[2]) == bytes(info)
        t = sim.export_octree(depth, device="cuda")
        assert isinstance(t.samples, torch.Tensor) and t.samples.is_cuda and tuple(t.samples.shape) == (m, 4)
        assert t.samples.dtype == torch.float32
        assert t.samples.cpu().numpy().tobytes() == a[1].tobytes() and t.nodes.tobytes() == a[0].tobytes()
        colors = t.samples.view(torch.int32)[:, 3].cpu().numpy().view(np.uint32)
        assert (colors == a[1]["color"]).all()
        # capacities one short: SIMLOD_ERR_INVALID and the guard bytes around both destinations untouched
        guard = 4096
        dn, ds = sim.device_alloc(n * 64 + 2 * guard), sim.device_alloc(m * 16 + 2 * guard)
        try:
            pattern_n = np.full(n * 64 + 2 * guard, 0xA5, dtype=np.uint8)
            pattern_s = np.full(m * 16 + 2 * guard, 0x5A, dtype=np.uint8)
            sim.memcpy_htod(dn, pattern_n)
            sim.memcpy_htod(ds, pattern_s)
            for caps in ((n - 1, m), (n, m - 1), (0, 0)):
                with pytest.raises(SimlodError) as err:
                    sim.export_octree_into(depth, dn + guard, caps[0], ds + guard, caps[1])
                assert err.value.code == -2
                assert (sim.memcpy_dtoh(dn, len(pattern_n)) == pattern_n).all() and (sim.memcpy_dtoh(ds, len(pattern_s)) == pattern_s).all()
            with pytest.raises(SimlodError) as err:
                sim.export_octree_into(21, dn + guard, n, ds + guard, m)
            assert err.value.code == -2
            # exact capacities: the export lands between the guards
            info2, ms = sim.export_octree_into(depth, dn + guard, n, ds + guard, m)
            assert bytes(info2) == bytes(info) and ms > 0
            got_n, got_s = sim.memcpy_dtoh(dn, len(pattern_n)), sim.memcpy_dtoh(ds, len(pattern_s))
            assert (got_n[:guard] == 0xA5).all() and (got_n[guard + n * 64:] == 0xA5).all()
            assert (got_s[:guard] == 0x5A).all() and (got_s[guard + m * 16:] == 0x5A).all()
            assert got_n[guard:guard + n * 64].tobytes() == a[0].tobytes() and got_s[guard:guard + m * 16].tobytes() == a[1].tobytes()
        finally:
            sim.device_free(dn)
            sim.device_free(ds)
