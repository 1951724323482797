"""GPU tests of the LAS writer (run with -m gpu on an H100): every file SimLOD.write_las writes equals the restatement
(las_write_restatement over the same samples and parameters) byte for byte, for the caller's arrays (crafted tensors,
query and view results, every input path) and for the octree's samples (five octrees, four depths, one of five
windows); the round trip through insert_files and files_box; the reference's loader on a written file; and the
protocol (refusals before any launch with no file left, an invalid sample in the third window, launch counts, unchanged
buffers, batches pending in the ring, repeatability)."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import files_restatement as fr
import las_write_restatement as W
import oracle
import reference_golden as golden
from simlod_b200 import Region, SimLOD, SimlodError, api, camera, data, files_box
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream
from test_las_files_gpu import assert_files_build_restated_octree

pytestmark = pytest.mark.gpu

F = np.float32
WINDOW = 8 << 20


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def launches(sim):
    return sim.launch_info()["launches"]


def check(path, samples, scale=0.001, offset=None, translation=(0.0, 0.0, 0.0), info=None):
    """The file at `path` is the restatement's, byte for byte, and info describes it."""
    want, bad = W.file_bytes(samples, scale, offset, translation)
    assert bad is None
    got = open(path, "rb").read()
    assert len(got) == len(want) and got[:227] == want[:227], "header"
    assert got == want, "records"
    assert not os.path.exists(path + ".tmp")
    if info is not None:
        h, _ = W.decode(want)
        assert info.num_points == h["num_points"] and info.file_size == len(want) and info.first_invalid == api.NO_INVALID
        assert tuple(info.min) == h["min"] and tuple(info.max) == h["max"]
    return got


def crafted(n=256 * 5 + 77):
    """Half-way ties, the int32 edges under scale 1 / translation 2^31 - 1 - 8, negative coordinates, all colours, and a
    count that leaves a partial last tile."""
    rng = np.random.default_rng(5)
    pts = np.zeros(n, dtype=api.POINT_DTYPE)
    for ax in "xyz":
        pts[ax] = rng.uniform(-9.0, 9.0, n).astype(F)
    pts["x"][:16] = np.arange(-8, 8, dtype=F) + F(0.5)          # ties at scale 1
    pts["y"][:8] = np.array([0.0, -0.0, 8.0, -9.0, 7.5, -7.5, 6.5, -6.5], dtype=F)
    k = np.arange(n, dtype=np.uint32)
    pts["color"] = (k & 0xFF) | (((k * 7) & 0xFF) << 8) | (((k * 13 + 1) & 0xFF) << 16) | ((k & 0x3) << 30)
    return pts


def test_caller_source_crafted_arrays(sim, tmp_path):
    torch = pytest.importorskip("torch")
    pts = crafted()
    edge = (2.0 ** 31 - 1 - 9.0, -(2.0 ** 31) + 9.0, 0.0)           # x + 9 reaches int32 max, y - 9 int32 min
    arr = pts.view(F).reshape(-1, 4)
    t = torch.from_numpy(arr.copy()).cuda()
    wide = torch.zeros((len(pts), 8), dtype=torch.float32, device="cuda")
    wide[:, 2:6] = t
    for label, src in (("tensor", t), ("strided tensor", wide[:, 2:6]), ("numpy points", pts), ("numpy (N, 4)", arr)):
        for scale, offset, translation in ((1.0, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0)), (1.0, (0.0, 0.0, 0.0), edge),
                                           ((0.003, 0.25, 0.01), (1.5, -2.0, 0.0), (100.0, 200.0, -300.0))):
            path = str(tmp_path / "c.las")
            n0 = launches(sim)
            info = sim.write_las(path, src, scale=scale, offset=offset, translation=translation, writer_threads=3)
            assert launches(sim) - n0 == 1 and info.num_windows == 1, label
            check(path, pts, scale, offset, translation, info)
    # one step beyond the edge: the first sample with x >= 7.5 rounds beyond int32 max
    with pytest.raises(SimlodError) as e:
        sim.write_las(str(tmp_path / "beyond.las"), t, scale=1.0, offset=(0.0, 0.0, 0.0), translation=(2.0 ** 31 - 1 - 7.0, 0.0, 0.0))
    assert e.value.info.first_invalid == W.file_bytes(pts, 1.0, (0.0, 0.0, 0.0), (2.0 ** 31 - 1 - 7.0, 0.0, 0.0))[1]
    assert not os.path.exists(str(tmp_path / "beyond.las")) and not os.path.exists(str(tmp_path / "beyond.las.tmp"))
    # empty arrays
    for src in (t[:0], pts[:0]):
        path = str(tmp_path / "empty.las")
        n0 = launches(sim)
        info = sim.write_las(path, src, scale=0.01)
        assert launches(sim) == n0 and info.num_points == 0
        check(path, pts[:0], 0.01, None, (0.0, 0.0, 0.0), info)


def test_caller_source_query_and_view_results(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    found, _ = sim.query_region(Region.box((500.0, 400.0, 0.0), (2100.0, 1700.0, 300.0)), None)
    assert len(found) > 1000
    path = str(tmp_path / "region.las")
    tr = (601000.0, 5200000.0, 12.5)
    info = sim.write_las(path, found, scale=0.001, translation=tr)
    check(path, found.cpu().numpy(), 0.001, None, tr, info)
    view, proj = camera.autofocus(box[1], sim.width, sim.height)
    sim.set_camera(view, proj)
    sim.render()
    v = sim.export_view()
    path = str(tmp_path / "view.las")
    info = sim.write_las(path, v.samples, scale=(0.01, 0.01, 0.005), offset=(0.0, 0.0, 0.0))
    check(path, v.samples.cpu().numpy(), (0.01, 0.01, 0.005), (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), info)


def check_octree_depths(sim, tmp_path, depths=None, label=""):
    top = sim.export_octree(None, device="cpu").info.max_level
    for depth in ([None, 0, 3, top] if depths is None else depths):
        want = sim.export_octree(20 if depth is None else depth, device="cpu").samples
        path = str(tmp_path / "o.las")
        n0 = launches(sim)
        info = sim.write_las(path, depth=depth, scale=0.001, offset=(0.0, 0.0, 0.0), translation=(1000.0, -2000.0, 5.0))
        windows = (len(want) + WINDOW - 1) // WINDOW
        assert info.num_windows == windows and launches(sim) - n0 == 2 + 2 * windows, (label, depth)
        check(path, want, 0.001, (0.0, 0.0, 0.0), (1000.0, -2000.0, 5.0), info)


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged"])
def test_octree_source(sim, tmp_path, name):
    batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
    build(sim, batches, box)
    check_octree_depths(sim, tmp_path, label=name)
    # the inserted points, those on the cube's max face included: every point of the stream
    w = sim.export_octree(20, device="cpu").samples
    assert len(w) == sum(len(b) for b in batches) == sim.stats().numPointsProcessed


def test_octree_source_of_a_36m_device_generated_terrain(sim, tmp_path):
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
    check_octree_depths(sim, tmp_path, depths=[None, 4], label="36m")
    # five windows, and the writer thread count does not change the file
    path = str(tmp_path / "t.las")
    info = sim.write_las(path, writer_threads=1)
    assert info.num_windows == 5
    a = hashlib.sha256(open(path, "rb").read()).hexdigest()
    sim.write_las(path, writer_threads=64)
    assert hashlib.sha256(open(path, "rb").read()).hexdigest() == a


def test_octree_source_of_the_reference_kernels_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box, reference=True)
    check_octree_depths(sim, tmp_path, depths=[None, 2], label="reference kernels")
    build(sim, batches, box)
    saved = str(tmp_path / "t.octree")
    sim.save_octree(saved)
    other = SimLOD(320, 176, persistent_bytes=4 << 30)
    try:
        other.load_octree(saved)
        check_octree_depths(other, tmp_path, depths=[None, 3], label="loaded")
    finally:
        other.close()


def test_round_trip_through_insert_files(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    first = str(tmp_path / "first.las")
    sim.write_las(first, scale=0.001, offset=(0.0, 0.0, 0.0))
    _, want = W.decode(open(first, "rb").read())
    src = sim.export_octree(20, device="cpu").samples
    other = SimLOD(320, 176, persistent_bytes=6 << 30)
    try:
        # insert_files builds the octree the restated batches of the same file build
        assert_files_build_restated_octree(other, [first])
        other.insert_files([first])
        got = other.export_octree(20, device="cpu").samples
        # colours come back with alpha 0xff; positions within s/2 plus the float roundings (DESIGN.md §9.13)
        assert np.array_equal(np.sort(got["color"]), np.sort((src["color"] & np.uint32(0xFFFFFF)) | np.uint32(0xFF000000)))
        bmin, _ = files_box([first])
        back = np.sort(np.stack([got[a].astype(np.float64) + float(bmin[k]) for k, a in enumerate("xyz")], axis=1), axis=0)
        orig = np.sort(np.stack([src[a].astype(np.float64) for a in "xyz"], axis=1), axis=0)
        tol = 0.0005 + np.spacing(np.abs(orig).astype(F)).astype(np.float64) * 2
        assert (np.abs(back - orig) <= tol).all()
        # written again at the world position: the same records, as a sorted multiset
        second = str(tmp_path / "second.las")
        other.write_las(second, scale=0.001, offset=(0.0, 0.0, 0.0), translation=tuple(float(v) for v in bmin))
        _, again = W.decode(open(second, "rb").read())
        assert np.array_equal(np.sort(again.view("V26")), np.sort(want.view("V26")))
    finally:
        other.close()


def test_the_reference_loader_reads_a_written_file(sim, tmp_path):
    if oracle.ref_las() is None:
        pytest.skip("the reference's LAS loader has not been built (oracle/_ref/libref_las.so)")
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    path = str(tmp_path / "r.las")
    info = sim.write_las(path, scale=0.002, offset=(1.0, 2.0, 3.0), translation=(1000.0, 2000.0, 50.0))
    buf = open(path, "rb").read()
    tr = (-1000.0, -2000.0, -50.0)
    dec = oracle.decode_las(np.frombuffer(buf, np.uint8, offset=227), info.num_points, 26, 2, (0.002,) * 3, (1.0, 2.0, 3.0), tr)
    assert golden.points(oracle.ref_las_load(path, 0, info.num_points, tr)) == golden.points(dec)
    h = fr.ref_las_header(path)
    assert h["num_points"] == info.num_points and tuple(h["min"]) == tuple(info.min) and tuple(h["max"]) == tuple(info.max)


# ---- protocol --------------------------------------------------------------------------------------------------------

def digest(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def test_refusals_happen_before_any_launch_and_leave_no_file(sim, tmp_path):
    torch = pytest.importorskip("torch")
    batches, box, _ = uniform_stream()
    build(sim, batches, box)
    t = torch.zeros((100, 4), dtype=torch.float32, device="cuda")
    existing = str(tmp_path / "existing.las")
    open(existing, "wb").write(b"keep me")
    before = digest(existing)
    lib = api.load_library()
    p = api.las_write_params()

    def raw(path, params=p, samples=0, n=0, depth=-1, info=True):
        i = api.LasWriteInfo()
        return lib.simlod_write_las(sim._ctx, None if path is None else os.fsencode(path), None if params is None else C.byref(params),
                                    samples, n, depth, C.byref(i) if info else None, None)
    cases = [("null path", lambda path: raw(None)), ("null params", lambda path: raw(path, None)),
             ("null info", lambda path: raw(path, info=False)),
             ("misaligned", lambda path: raw(path, samples=t.data_ptr() + 4, n=10)),
             ("depth with samples", lambda path: raw(path, samples=t.data_ptr(), n=100, depth=0)),
             ("depth > 20", lambda path: raw(path, depth=21)),
             ("too many samples", lambda path: raw(path, samples=t.data_ptr(), n=2 ** 32)),
             ("no directory", lambda path: raw(str(tmp_path / "missing" / "x.las")))]
    for field, value in (("scale", (0.0, 1.0, 1.0)), ("scale", (1.0, -1.0, 1.0)), ("scale", (1.0, 1.0, float("inf"))),
                         ("scale", (float("nan"), 1.0, 1.0)), ("offset", (float("nan"), 0.0, 0.0)),
                         ("translation", (0.0, float("inf"), 0.0))):
        q = api.las_write_params()
        getattr(q, field)[:] = value
        cases.append(("%s %s" % (field, value), lambda path, q=q: raw(path, q)))
    for threads in (0, 65):
        cases.append(("writer_threads %d" % threads, lambda path, th=threads: raw(path, api.las_write_params(writer_threads=th))))
    for label, call in cases:
        for path in (existing, str(tmp_path / "new.las")):
            n0 = launches(sim)
            assert call(path) == -2, label
            assert launches(sim) == n0, label
            assert not os.path.exists(path + ".tmp") and not os.path.exists(str(tmp_path / "new.las")), label
            assert digest(existing) == before, label
    # a write over an existing file replaces it once complete
    sim.write_las(existing)
    check(existing, sim.export_octree(20, device="cpu").samples, 0.001)


def test_an_invalid_sample_in_the_third_window(sim, tmp_path):
    torch = pytest.importorskip("torch")
    n = 2 * WINDOW + 1000
    bad = 2 * WINDOW + 517
    t = torch.rand((n, 4), dtype=torch.float32, device="cuda") * 100.0
    t[bad, 1] = float("nan")
    t[bad + 3, 0] = 1e30                                   # also invalid, but later
    path = str(tmp_path / "bad.las")
    existing = str(tmp_path / "existing.las")
    open(existing, "wb").write(b"keep")
    for target in (path, existing):
        with pytest.raises(SimlodError) as e:
            sim.write_las(target, t, scale=0.001)
        assert e.value.code == -2 and e.value.info.first_invalid == bad and str(bad) in str(e.value)
        assert not os.path.exists(target + ".tmp")
    assert not os.path.exists(path) and open(existing, "rb").read() == b"keep"
    t[bad, 1] = 1.0
    t[bad + 3, 0] = 2.0
    n0 = launches(sim)
    info = sim.write_las(path, t, scale=0.001)
    assert launches(sim) - n0 == 3 and info.num_windows == 3
    check(path, t.cpu().numpy(), 0.001, None, (0.0, 0.0, 0.0), info)


def test_writes_change_nothing_and_repeat_byte_identically(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    view, proj = camera.autofocus(box[1], sim.width, sim.height)
    sim.set_camera(view, proj)
    sim.render()
    b = sim.buffers()
    ring = lambda: hashlib.sha256(sim.memcpy_dtoh(b.ring, b.ring_bytes).tobytes()).hexdigest()
    before, ring0 = buffer_digests(sim), ring()
    paths = [str(tmp_path / ("r%d.las" % k)) for k in range(3)]
    for k, path in enumerate(paths):
        sim.write_las(path, depth=None if k < 2 else 5, writer_threads=(1, 8, 16)[k])
    sim.write_las(paths[2], depth=None, writer_threads=16)
    assert buffer_digests(sim) == before and ring() == ring0
    assert digest(paths[0]) == digest(paths[1]) == digest(paths[2])


def test_a_write_while_batches_wait_writes_the_snapshot(sim, tmp_path):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for bt in batches:
        sim.upload_batch(bt)
    written = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        if sim.stats().batchletIndex < len(batches):
            path = str(tmp_path / "p.las")
            sim.write_las(path, scale=0.01)
            check(path, sim.export_octree(20, device="cpu").samples, 0.01)
            assert sim.stats().batchletIndex < len(batches)
            written += 1
    assert written >= 1
