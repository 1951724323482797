"""GPU tests of the view export (run with -m gpu on an H100): simlod_export_view against the LOD cut kernel_render
draws for the same uniforms. The expectation is export_view_restatement.export_view_image of the device image, with the drawn
set that the frame's visible / isLarge flags give (drawn_from_flags), byte for byte; the drawn set is also checked
against the frame's Stats, against the reference's own kernel_render (digests in tests/golden/export_view_reference.json,
recorded again live with SIMLOD_RECORD_GOLDEN set), under a frozen visibility transform, and the protocol (sizes,
capacities, guard bytes, no writes into the context's buffers)."""
import hashlib
import json
import os

import numpy as np
import pytest

import export_restatement as R
import export_view_restatement as V
import oracle
import reference_golden as golden
from simlod_b200 import SimLOD, SimlodError, api, camera, data
from test_export_cpu import check_structure
from test_export_gpu import build, buffer_digests, same_export, terrain_ragged_stream, uniform_stream
from test_parity_gpu import cameras

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
MIN_NODE_SIZES = (16.0, 64.0, 256.0)
# (stream, camera, minNodeSize) cases with a drawn node below a node that is not large (isLarge is not monotone along
# the path once box corners lie behind the camera; the reason the cut is evaluated per node, not by a descent from the
# root), asserted so that they keep being covered. test_view_export_is_the_renderers_cut prints the count for every
# case; none of its cases has one (measured on an H100), so the per-node evaluation is pinned there by the byte-exact
# comparison only, and the case itself by test_export_view_cpu.py's hand-made flags.
NON_MONOTONE_CASES = []


@pytest.fixture(scope="module")
def sim():
    # 3 render blocks per SM: the grid the reference's own kernel_render gets from the occupancy query on sm_90
    s = SimLOD(W, H, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30, render_blocks_per_sm=3)
    yield s
    s.close()


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "export_view_reference.json")


def reference_result(key, run):
    """The reference kernels' result for `key`: run() live (and recorded) with SIMLOD_RECORD_GOLDEN set, else the stored one."""
    if golden.RECORD:
        return golden.reference(key, run)
    with open(GOLDEN) as f:
        stored = json.load(f)
    assert key in stored, "no stored reference result for %r in %s" % (key, GOLDEN)
    return stored[key]


def view_cameras(box_max, terrain):
    cams = list(cameras(box_max, W, H))
    if terrain:
        cams += [("morro_bird", camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD)),
                 ("morro_close", camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE))]
    return cams


def build_generated_terrain(sim, n=36_000_000):
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        sim.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.reset()
        sim.insert_device(dptr, n)
    finally:
        sim.device_free(dptr)
    assert sim.stats().dbg == 0 and sim.stats().numPointsProcessed == n
    return tuple(float(v) for v in data.TERRAIN_EXTENT)


def build_stream(sim, name):
    if name == "terrain_36m":
        return build_generated_terrain(sim), True
    batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
    build(sim, batches, box)
    return box[1], name.startswith("terrain")


def nodes_image(sim):
    st = sim.stats()
    return sim.memcpy_dtoh(sim.buffers().nodes, st.numNodes * 152)


def heap_image(sim):
    b = sim.buffers()
    used = int(sim.memcpy_dtoh(b.persistent + 8, 8).view(np.uint64)[0])
    return sim.memcpy_dtoh(b.persistent, used), int(b.nodes), int(b.persistent)


def device_view(sim):
    e = sim.export_view(device="cpu")
    return e.nodes, e.samples, e.info


def non_monotone(nodes_bytes, drawn):
    """Drawn nodes with an ancestor (by coordinates) that the frame did not flag large."""
    raw = np.ascontiguousarray(nodes_bytes).reshape(-1, 152)
    rec = np.frombuffer(raw.tobytes(), dtype=R.NODE_DTYPE)
    large = raw[:, V.IS_LARGE_BYTE] != 0
    key = {(int(l), int(x), int(y), int(z)): i for i, (l, x, y, z) in enumerate(zip(rec["level"], rec["X"], rec["Y"], rec["Z"]))}
    count = 0
    for i in np.nonzero(drawn)[0]:
        l, x, y, z = int(rec["level"][i]), int(rec["X"][i]), int(rec["Y"][i]), int(rec["Z"][i])
        while l > 0:
            l, x, y, z = l - 1, x >> 1, y >> 1, z >> 1
            if not large[key[(l, x, y, z)]]:
                count += 1
                break
    return count


def check_frame(sim, heap, label):
    """Render, then: the view export == the restatement for the frame's drawn set, and the drawn set matches Stats."""
    sim.render()
    st = sim.stats()
    nb = nodes_image(sim)
    drawn = V.drawn_from_flags(nb)
    got = device_view(sim)
    same_export(got, V.export_view_image(nb, *heap, drawn), label)
    nodes, samples, info = got
    check_structure(nodes, info)
    sampled = (nodes["flags"] & api.EXPORT_SAMPLED) != 0
    assert int(sampled.sum()) == int(drawn.sum()) == st.numVisibleNodes, label
    assert int(nodes["num_points"][sampled].sum()) == st.numVisiblePoints, label
    rec = np.frombuffer(np.ascontiguousarray(nb).tobytes(), dtype=np.dtype({"names": ["numPoints", "numVoxels", "numVoxelsStored"],
                        "formats": ["<u4", "<u4", "<u4"], "offsets": [68, 144, 148], "itemsize": 152}))
    voxel_nodes = drawn & (rec["numPoints"] == 0)
    if (rec["numVoxels"][voxel_nodes] == rec["numVoxelsStored"][voxel_nodes]).all():
        assert int(nodes["num_voxels"][sampled & (nodes["num_points"] == 0)].sum()) == st.numVisibleVoxels, label
    return nb, drawn, got


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged", "terrain_36m"])
def test_view_export_is_the_renderers_cut(sim, name):
    box_max, terrain = build_stream(sim, name)
    heap = heap_image(sim)
    report = []
    for cam, (view, proj) in view_cameras(box_max, terrain):
        sim.set_camera(view, proj)
        for mns in MIN_NODE_SIZES:
            sim.set_settings(minNodeSize=mns)
            label = "%s/%s/minNodeSize %g" % (name, cam, mns)
            nb, drawn, (nodes, _, info) = check_frame(sim, heap, label)
            nm = non_monotone(nb, drawn)
            report.append((cam, mns, info.num_nodes, int(drawn.sum()), info.num_samples, nm))
            if (name, cam, mns) in NON_MONOTONE_CASES:
                assert nm > 0, label
    sim.set_settings(minNodeSize=64.0)
    for r in report:
        print("view export %s: camera %s minNodeSize %g: %d records, %d drawn, %d samples, %d drawn below a non-large node" % ((name,) + r))


def drawn_digest(nodes_bytes, drawn):
    """sha256 of the drawn nodes' (level, X, Y, Z), sorted."""
    rec = np.frombuffer(np.ascontiguousarray(nodes_bytes).tobytes(), dtype=R.NODE_DTYPE)
    keys = np.stack([rec[f][drawn].astype(np.uint32) for f in ("level", "X", "Y", "Z")], axis=1)
    keys = keys[np.lexsort((keys[:, 3], keys[:, 2], keys[:, 1], keys[:, 0]))]
    return hashlib.sha256(np.ascontiguousarray(keys).tobytes()).hexdigest()


def sampled_digest(nodes):
    sampled = (nodes["flags"] & api.EXPORT_SAMPLED) != 0
    keys = np.stack([nodes[f][sampled].astype(np.uint32) for f in ("level", "X", "Y", "Z")], axis=1)
    keys = keys[np.lexsort((keys[:, 3], keys[:, 2], keys[:, 1], keys[:, 0]))]
    return hashlib.sha256(np.ascontiguousarray(keys).tobytes()).hexdigest()


def test_view_export_matches_the_reference_renderers_cut(sim):
    """The nodes the reference's kernel_render draws (its flags on our octree, same uniforms) are the export's SAMPLED set."""
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cams = view_cameras(box[1], True)

    def run():
        out = {}
        sim.use_module(1, oracle.REF_CUBINS[1])
        try:
            for cam, (view, proj) in cams:
                sim.set_camera(view, proj)
                for mns in MIN_NODE_SIZES:
                    sim.set_settings(minNodeSize=mns)
                    sim.render()
                    nb = nodes_image(sim)
                    out["%s/%g" % (cam, mns)] = drawn_digest(nb, V.drawn_from_flags(nb))
        finally:
            sim.use_module(1, None)
        return out
    ref = reference_result("view_drawn_terrain_ragged", run)
    ours = {}
    for cam, (view, proj) in cams:
        sim.set_camera(view, proj)
        for mns in MIN_NODE_SIZES:
            sim.set_settings(minNodeSize=mns)
            ours["%s/%g" % (cam, mns)] = sampled_digest(device_view(sim)[0])
    sim.set_settings(minNodeSize=64.0)
    assert len(ref) == len(ours)
    golden.assert_same(ours, ref, "view export's SAMPLED set vs the reference kernel_render's cut")


def test_view_export_of_the_reference_kernels_octree(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box, reference=True)
    heap = heap_image(sim)
    for cam, (view, proj) in view_cameras(box[1], True):
        sim.set_camera(view, proj)
        check_frame(sim, heap, "reference kernels' octree/%s" % cam)


def test_frozen_visibility(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    heap = heap_image(sim)
    cams = dict(cameras(box[1], W, H))
    sim.set_camera(*cams["far"])
    far = device_view(sim)
    sim.set_camera(*cams["close"], update_visibility=False)
    frozen = check_frame(sim, heap, "close camera, frozen at far")[2]
    same_export(frozen, far, "frozen visibility follows the far cut")
    sim.set_camera(*cams["close"])
    close = device_view(sim)
    assert close[0].tobytes() != far[0].tobytes()


def test_protocol(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cams = dict(cameras(box[1], W, H))
    sim.set_camera(*cams["close"])
    sim.render()                                 # flags of another camera in nodes[]
    sim.set_camera(*cams["autofocus"])
    info, _ = sim.export_view_into(0, 0, 0, 0)   # size query
    n, m = info.num_nodes, info.num_samples
    assert n > 1 and m > 0

    # nothing in nodes[], the heap, the momentary or render buffers, the ring or Stats changes
    b = sim.buffers()
    ring = lambda: hashlib.sha256(sim.memcpy_dtoh(b.ring, b.ring_bytes).tobytes()).hexdigest()   # noqa: E731
    before, ring_before = buffer_digests(sim), ring()
    a = device_view(sim)
    a2 = device_view(sim)
    assert buffer_digests(sim) == before and ring() == ring_before
    same_export(a, a2, "two view exports")
    assert bytes(a[2]) == bytes(info)

    # full and depth exports are the same before and after a view export
    fulls = [sim.export_octree(d, device="cpu") for d in (None, 3)]
    device_view(sim)
    for d, e in zip((None, 3), fulls):
        e2 = sim.export_octree(d, device="cpu")
        assert e2.nodes.tobytes() == e.nodes.tobytes() and e2.samples.tobytes() == e.samples.tobytes() and bytes(e2.info) == bytes(e.info)

    # the torch path
    torch = pytest.importorskip("torch")
    t = sim.export_view(device="cuda")
    assert isinstance(t.samples, torch.Tensor) and t.samples.is_cuda and tuple(t.samples.shape) == (m, 4)
    assert t.samples.cpu().numpy().tobytes() == a[1].tobytes() and t.nodes.tobytes() == a[0].tobytes()

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
                sim.export_view_into(dn + guard, caps[0], ds + guard, caps[1])
            assert err.value.code == -2
            assert (sim.memcpy_dtoh(dn, len(pattern_n)) == pattern_n).all() and (sim.memcpy_dtoh(ds, len(pattern_s)) == pattern_s).all()
        with pytest.raises(SimlodError) as err:
            sim.export_view_into(dn + guard + 8, n, ds + guard, m)          # misaligned
        assert err.value.code == -2
        info2, ms = sim.export_view_into(dn + guard, n, ds + guard, m)
        assert bytes(info2) == bytes(info) and ms > 0
        got_n, got_s = sim.memcpy_dtoh(dn, len(pattern_n)), sim.memcpy_dtoh(ds, len(pattern_s))
        assert (got_n[:guard] == 0xA5).all() and (got_n[guard + n * 64:] == 0xA5).all()
        assert (got_s[:guard] == 0x5A).all() and (got_s[guard + m * 16:] == 0x5A).all()
        assert got_n[guard:guard + n * 64].tobytes() == a[0].tobytes() and got_s[guard:guard + m * 16].tobytes() == a[1].tobytes()

        # an empty view (no node projects larger than minNodeSize, so none is drawn): the root alone, a null sample
        # destination accepted
        sim.set_settings(minNodeSize=1e9)
        e, _ = sim.export_view_into(0, 0, 0, 0)
        assert e.num_nodes == 1 and e.num_samples == 0 and e.max_level == info.max_level
        e2, _ = sim.export_view_into(dn + guard, 1, 0, 0)
        root = sim.memcpy_dtoh(dn + guard, 64).view(api.EXPORT_NODE_DTYPE)
        assert root["parent"][0] == -1 and root["first_child"][0] == -1 and root["flags"][0] == 0 and root["name"][0] == b"r"
        heap = heap_image(sim)
        check_frame(sim, heap, "empty view")
    finally:
        sim.set_settings(minNodeSize=64.0)
        sim.device_free(dn)
        sim.device_free(ds)
