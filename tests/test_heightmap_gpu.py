"""GPU tests of the height map (run with -m gpu on an H100): simlod_query_heightmap against its restatement
(heightmap_restatement over the export of the same device image, byte for byte) on several octrees, grids and depths,
against the inserted points and query_region, and its protocol (destination subsets, refused arguments with guard bytes,
launches, stage times, repeatability, the torch and numpy paths, no writes into the context's buffers, batches pending
in the ring, a query scratch shared with the other queries).

Not tested: the refusal of an export of 2^32 samples or more, which needs a heap of about 69 GB."""
import ctypes as C
import os

import numpy as np
import pytest

import export_restatement as R
import heightmap_restatement as H
import oracle
import query_restatement as Q
from simlod_b200 import Region, SimLOD, SimlodError, api, camera, data
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream

pytestmark = pytest.mark.gpu

F = np.float32
NAN = float("nan")
INF = float("inf")
NAMES = ("count", "z_min", "z_max", "z_mean", "top", "samples")
WIDTHS = (8, 4, 4, 4, 8, 16)


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def cube(sim, box):
    """(boxMin, boxMax, the device's reciprocal of the cube size) for the restatement."""
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    return box[0], box[1], sim.device_rcp(size)


def grids(box, fine=1000):
    """Named (origin, cell, shape): the whole box at coarse and fine cells, a sub-box tile, a grid straddling the
    cube's edge, and one cell."""
    mn, mx = np.asarray(box[0], np.float64), np.asarray(box[1], np.float64)
    ext = mx - mn
    size = float(ext.max())
    whole = lambda c: ((float(mn[0]), float(mn[1])), c, (int(np.ceil(ext[1] / c)) + 1, int(np.ceil(ext[0] / c)) + 1))
    return {"coarse": whole(size / 16), "fine": whole(size / fine),
            "tile": ((float(mn[0] + 0.3 * ext[0]), float(mn[1] + 0.4 * ext[1])), size / 2000, (300, 400)),
            "straddle": ((float(mn[0] - 0.25 * ext[0]), float(mx[1] - 0.5 * ext[1])), size / 64, (64, 40)),
            "one": ((float(mn[0]), float(mn[1])), size * 1.01, (1, 1))}


def same(got, want, label):
    for a, w, name in zip(got, want, NAMES):
        a, w = np.ascontiguousarray(a), np.ascontiguousarray(w)
        if a.tobytes() != w.tobytes():
            ab = np.frombuffer(a.tobytes(), np.uint8).reshape(w.size, -1)
            wb = np.frombuffer(w.tobytes(), np.uint8).reshape(w.size, -1)
            bad = np.nonzero((ab != wb).any(axis=1))[0]
            raise AssertionError("%s: %s differs in %d cells, first %s" % (label, name, len(bad), bad[:8]))


def check(sim, box, depths=None, names=None, fine=1000):
    """Every grid at every depth: all six results byte-identical to the restatement of the image, samples those of
    export_octree(depth)[top], the info's counts as expected."""
    image = sim.download_octree()
    cb = cube(sim, box)
    full = R.export_image(*image)
    top_level = full[2].max_level
    for depth in (sorted({0, 3, top_level}) + [None] if depths is None else depths):
        ex = full if depth is None else R.export_image(*image, depth)
        dev = sim.export_octree(depth, device="cpu")
        assert dev.samples.tobytes() == ex[1].tobytes()
        for name, (origin, cell, shape) in grids(box, fine).items():
            if names is not None and name not in names:
                continue
            label = "depth %s grid %s" % (depth, name)
            out = sim.query_heightmap(origin, cell, shape, depth, device="cpu", samples=True)
            info = out[-1]
            want = H.heightmap(ex, depth, *cb[:2], origin, cell, shape, cb[2])
            same(out[:-1], want, label)
            count, top, samples = out[0], out[4], out[5]
            expect = np.zeros(shape, dtype=api.POINT_DTYPE)
            expect[top >= 0] = dev.samples[top[top >= 0]]
            assert samples.tobytes() == expect.tobytes(), label
            assert info.num_binned == int(count.sum()) and info.nonempty_cells == int((count > 0).sum()), label
            assert (info.num_samples, info.max_level) == (ex[2].num_samples, top_level), label
            assert info.samples_tested >= info.records_visited and info.samples_tested >= info.num_binned, label
            if name == "one":                              # one cell over the whole cube: the region query's count
                region = Region.box(np.asarray(box[0], F) - 1, np.asarray(box[1], F) + float(cell))
                _, qinfo = sim.query_region(region, depth, device="cpu")
                assert count[0, 0] == qinfo.num_samples, label


def against_points(sim, box, points, grid):
    """depth None: count, z_min, z_max and z_mean equal a numpy binning of the inserted points in the cube."""
    origin, cell, shape = grid
    cb = cube(sim, box)
    inside = np.ascontiguousarray(points[Q.in_cube(points, *cb[:2], cb[2])]).view(R.POINT_DTYPE)
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["flags"], nodes["first_child"], nodes["num_points"] = R.LEAF, -1, len(inside)
    want = H.heightmap((nodes, inside, None), None, *cb[:2], origin, cell, shape, cb[2])
    out = sim.query_heightmap(origin, cell, shape, None, device="cpu")
    same(out[:4], want[:4], "the inserted points")


@pytest.mark.parametrize("stream", [uniform_stream, terrain_ragged_stream], ids=["uniform_1m", "terrain_ragged"])
def test_heightmap_equals_the_restatement(sim, stream):
    batches, box, _ = stream()
    build(sim, batches, box)
    check(sim, box)
    points = np.concatenate(batches)
    for name in ("coarse", "fine", "straddle"):
        against_points(sim, box, points, grids(box)[name])


def test_heightmap_of_a_36m_device_generated_terrain_stream(sim):
    n = 36_000_000
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        box = ((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.set_box(*box)
        sim.reset()
        sim.insert_device(dptr, n)
        points = sim.memcpy_dtoh(dptr, n * 16).view(api.POINT_DTYPE)
    finally:
        sim.device_free(dptr)
    assert sim.stats().dbg == 0 and sim.stats().numPointsProcessed == n
    check(sim, box, depths=(None, 3), names=("coarse", "tile", "straddle", "one"))
    against_points(sim, box, points, grids(box)["coarse"])


def test_heightmap_of_the_reference_kernels_octree_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    if all(os.path.exists(p) for p in oracle.REF_CUBINS.values()):
        build(sim, batches, box, reference=True)           # the query reads the ABI only
        check(sim, box, depths=(None, 2))
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    sim.save_octree(path)
    sim.reset()
    sim.load_octree(path)
    check(sim, box, depths=(None, 2))


def test_torch_and_numpy_paths_agree(sim):
    torch = pytest.importorskip("torch")
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    origin, cell, shape = grids(box)["tile"]
    for depth in (None, 3):
        n = sim.query_heightmap(origin, cell, shape, depth, device="cpu", samples=True)
        t = sim.query_heightmap(origin, cell, shape, depth, samples=True)
        dtypes = (torch.int64, torch.float32, torch.float32, torch.float32, torch.int64, torch.float32)
        for a, b, dt in zip(t[:-1], n[:-1], dtypes):
            assert isinstance(a, torch.Tensor) and a.is_cuda and a.dtype == dt and tuple(a.shape[:2]) == shape
            assert a.cpu().numpy().tobytes() == b.tobytes()
        assert tuple(t[5].shape) == shape + (4,) and n[5].dtype == api.POINT_DTYPE
        assert (t[-1].num_binned, t[-1].nonempty_cells) == (n[-1].num_binned, n[-1].nonempty_cells) and n[-1].num_binned > 0
        assert len(sim.query_heightmap(origin, cell, shape, depth, device="cpu")) == 6


def launches_of(sim, call):
    before = sim.launch_info()["launches"]
    out = call()
    return sim.launch_info()["launches"] - before, out


def stage_sum(*ms):
    total = np.float32(ms[0])
    for m in ms[1:]:
        total = np.float32(total + np.float32(m))
    return float(total)


def test_protocol(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    origin, cell, (ny, nx) = grids(box)["tile"]
    cells = nx * ny
    guard = 4096
    bufs = [sim.device_alloc(cells * w + 2 * guard) for w in WIDTHS]
    try:
        pats = [np.full(cells * w + 2 * guard, 0x5A, dtype=np.uint8) for w in WIDTHS]
        for p, pat in zip(bufs, pats):
            sim.memcpy_htod(p, pat)
        dst = [p + guard for p in bufs]

        def grid(o=origin, c=cell, x=nx, y=ny):
            g = api.SimlodHeightmap(cell=float(c), nx=int(x), ny=int(y))
            g.origin[:] = [float(v) for v in o]
            return g

        launches = sim.launch_info()["launches"]
        refused = {"origin_nan": (grid(o=(NAN, 0.0)), None, dst), "origin_inf": (grid(o=(0.0, -INF)), None, dst),
                   "cell_0": (grid(c=0.0), None, dst), "cell_negative": (grid(c=-1.0), None, dst),
                   "cell_nan": (grid(c=NAN), None, dst), "cell_inf": (grid(c=INF), None, dst),
                   "nx_0": (grid(x=0), None, dst), "ny_0": (grid(y=0), None, dst),
                   "cells_above_2^27": (grid(x=(1 << 27) + 1, y=1), None, dst), "cells_2^32": (grid(x=1 << 16, y=1 << 16), None, dst),
                   "depth_21": (grid(), 21, dst)}
        for k, w in enumerate(WIDTHS):
            d = list(dst)
            d[k] += w // 2 if w > 4 else 2
            refused["%s_misaligned" % NAMES[k]] = (grid(), None, d)
        for name, (g, depth, d) in refused.items():
            with pytest.raises(SimlodError) as err:
                sim.query_heightmap_into(g, depth, *d)
            assert err.value.code == -2, name
        info, ms = api.SimlodHeightmapInfo(), C.c_float(0)
        assert sim._lib.simlod_query_heightmap(sim._ctx, None, -1, *dst, C.byref(info), C.byref(ms)) == -2
        assert sim._lib.simlod_query_heightmap(sim._ctx, C.byref(grid()), -1, *dst, None, C.byref(ms)) == -2
        assert sim.launch_info()["launches"] == launches       # refused before any launch
        for p, pat in zip(bufs, pats):
            assert (sim.memcpy_dtoh(p, len(pat)) == pat).all()
        for depth in (None, 3):
            want = sim.query_heightmap(origin, cell, (ny, nx), depth, device="cpu", samples=True)
            n, (info0, ms0) = launches_of(sim, lambda: sim.query_heightmap_into(grid(), depth, 0, 0, 0, 0, 0, 0))
            assert n == 4 and ms0 == stage_sum(info0.plan_ms, info0.accumulate_ms, info0.finalize_ms) and ms0 > 0
            assert (info0.num_binned, info0.nonempty_cells) == (want[-1].num_binned, want[-1].nonempty_cells)
            for p, pat in zip(bufs, pats):                     # info only: nothing written
                assert (sim.memcpy_dtoh(p, len(pat)) == pat).all()
            # every subset of destinations: the same bytes for those it asks for, nothing outside them
            for mask in (1, 2, 4, 8, 16, 32, 6, 9, 48, 63):
                d = [dst[k] if mask >> k & 1 else 0 for k in range(6)]
                n, (info, ms) = launches_of(sim, lambda: sim.query_heightmap_into(grid(), depth, *d))
                assert n == 4 and ms == stage_sum(info.plan_ms, info.accumulate_ms, info.finalize_ms)
                assert (info.num_binned, info.samples_tested, info.records_visited, info.nonempty_cells) == \
                    (info0.num_binned, info0.samples_tested, info0.records_visited, info0.nonempty_cells)
                for k, (p, pat, w) in enumerate(zip(bufs, pats, want[:6])):
                    back = sim.memcpy_dtoh(p, len(pat))
                    assert (back[:guard] == 0x5A).all() and (back[len(pat) - guard:] == 0x5A).all()
                    if mask >> k & 1:
                        assert back[guard:len(pat) - guard].tobytes() == w.tobytes(), (mask, NAMES[k])
                for p, pat in zip(bufs, pats):
                    sim.memcpy_htod(p, pat)
            # repeat calls are byte-identical
            again = sim.query_heightmap(origin, cell, (ny, nx), depth, device="cpu", samples=True)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(again[:6], want[:6]))
            assert again[-1].plan_ms > 0 and again[-1].accumulate_ms > 0 and again[-1].finalize_ms > 0
    finally:
        for p in bufs:
            sim.device_free(p)


def test_heightmap_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], sim.width, sim.height))
    sim.render()
    before = buffer_digests(sim)
    ring = sim.ring_slot(0, 1000).tobytes()
    for depth in (None, 2):
        for origin, cell, shape in grids(box, 300).values():
            sim.query_heightmap(origin, cell, shape, depth, device="cpu", samples=True)
    assert buffer_digests(sim) == before and sim.ring_slot(0, 1000).tobytes() == ring


def test_heightmap_while_batches_are_pending_sees_the_last_completed_launch(sim):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for b in batches:
        sim.upload_batch(b)
    origin, cell, shape = grids((mn, mx), 100)["fine"]
    snapshots = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        done = sim.stats().batchletIndex
        if done < len(batches):
            image = sim.download_octree()
            out = sim.query_heightmap(origin, cell, shape, device="cpu", samples=True)
            want = H.heightmap_image(*image, None, mn, mx, origin, cell, shape)
            same(out[:-1], want, "pending")
            assert out[-1].num_binned == int(out[0].sum()) > 0
            snapshots += 1
    assert snapshots >= 1


def test_scratch_shared_with_the_other_queries_gives_a_fresh_contexts_bytes():
    """nearest, radius (large enough to outgrow the others' scratch), ray, pick and heightmap in turn on one context: each
    heightmap byte for byte the one the context made before any other query used its scratch, and its count, z_min,
    z_max and z_mean those of a fresh context built from the same points (its top indices may differ: two builds may
    store a leaf's points in different orders)."""
    pts, mn, mx = data.uniform_cube(1_000_000, size=64.0, seed=5)
    origin, cell, shape = grids((mn, mx), 200)["fine"]

    def make():
        s = SimLOD(320, 180, persistent_bytes=2 << 30)
        s.set_box(mn, mx)
        s.reset()
        s.insert(pts)
        s.set_camera(*camera.autofocus(mx, 320, 180))
        return s

    def heightmap(s):
        return [x.tobytes() for x in s.query_heightmap(origin, cell, shape, 3, device="cpu", samples=True)[:-1]]

    fresh = make()
    try:
        other = heightmap(fresh)
    finally:
        fresh.close()
    s = make()
    try:
        want = heightmap(s)
        assert want[:4] == other[:4]
        rng = np.random.default_rng(4)
        p = pts[rng.integers(0, len(pts), 60_000)]
        q = np.stack([p["x"], p["y"], p["z"]], axis=1).astype(F)
        s.query_nearest(q[:1000], 8, device="cpu")
        assert s.query_radius(q, 0.5, device="cpu")[-1].num_found > 0
        s.query_ray(q[:1000], np.tile([[0.0, 0.0, -1.0]], (1000, 1)), 0.5, device="cpu")
        s.render()
        s.pick([[160, 90]], device="cpu")
        for _ in range(2):
            assert heightmap(s) == want
            s.query_nearest(q[:1000], 8, device="cpu")
    finally:
        s.close()
