"""GPU tests of the k-nearest query (run with -m gpu on an H100): simlod_query_nearest against its restatement
(nearest_restatement over the export of the same device image, byte for byte) on several octrees and query sets, the
returned samples against export_octree(depth), and its protocol (refused arguments with guard bytes, repeatability, the
torch and numpy paths, no writes into the context's buffers, batches pending in the ring)."""
import os

import numpy as np
import pytest

import export_restatement as R
import nearest_restatement as N
import oracle
from simlod_b200 import Region, SimLOD, SimlodError, api, camera, data
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def cube(sim, box):
    """(boxMin, boxMax, the device's reciprocal of the cube size) for the restatement."""
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    return box[0], box[1], sim.device_rcp(size)


def query_sets(points, box, n=400, seed=1):
    """Named (n, 4) float32 query arrays: uniform in the cube, stored points, stored points jittered, points outside the
    cube, stored points moved onto the max face, and a mix of non-finite and finite queries."""
    rng = np.random.default_rng(seed)
    mn = np.asarray(box[0], dtype=np.float64)
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    xyz = np.stack([points["x"], points["y"], points["z"]], axis=1)
    stored = xyz[rng.choice(len(xyz), n)].astype(np.float64)
    outside = mn + rng.uniform(-0.5, 1.5, (n, 3)) * size
    outside[:, 0] = np.where(rng.random(n) < 0.5, mn[0] - rng.uniform(0, size, n), mn[0] + size * (1 + rng.uniform(0, 1, n)))
    face = stored.copy()
    face[:, 0] = mn[0] + size
    bad = mn + rng.uniform(0, 1, (n, 3)) * size
    bad[0::4, 0], bad[1::4, 1], bad[2::4, 2] = np.nan, np.inf, -np.inf
    sets = {"uniform": mn + rng.uniform(0, 1, (n, 3)) * size, "stored": stored,
            "jittered": stored + rng.normal(0, size * 1e-4, (n, 3)), "outside": outside, "max_face": face, "non_finite": bad}
    out = {}
    for name, v in sets.items():
        q = np.zeros((n, 4), dtype=F)
        q[:, :3] = v
        q[:, 3] = rng.uniform(-1, 1, n)                      # the ignored word
        out[name] = q
    return out


def check(sim, box, points, depths=None, ks=(1, 8, 32), radii=(None, "small"), sets=None, n=400):
    """Every query set at every k, depth and radius: index and dist2 byte-identical to the restatement of the image, the
    samples those of export_octree(depth), the counts as expected."""
    image = sim.download_octree()
    cb = cube(sim, box)
    full = R.export_image(*image)
    top = full[2].max_level
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    queries = query_sets(points, box, n)
    if sets is not None:
        queries = {k: v for k, v in queries.items() if k in sets}
    allq = np.concatenate(list(queries.values()))
    invalid = int((~np.isfinite(allq[:, :3]).all(axis=1)).sum())
    for depth in (sorted({0, 3, top}, key=int) + [None] if depths is None else depths):
        ex = full if depth is None else R.export_image(*image, depth)
        dev = sim.export_octree(depth, device="cpu")
        assert dev.samples.tobytes() == ex[1].tobytes()
        prep = N.Prepared(ex, depth, *cb)
        for k in ks:
            for radius in radii:
                r = size / 200.0 if radius == "small" else radius
                label = "depth %s k %d radius %s" % (depth, k, r)
                index, dist2, got, info = sim.query_nearest(allq, k, depth, r, device="cpu", samples=True)
                want_i, want_d = N.search(prep, allq, k, r)
                assert index.tobytes() == want_i.tobytes(), label
                assert dist2.tobytes() == want_d.tobytes(), label
                filled = index >= 0
                expect = np.zeros(index.shape, dtype=api.POINT_DTYPE)
                expect[filled] = dev.samples[index[filled]]
                assert got.tobytes() == expect.tobytes(), label
                assert (info.num_found, info.invalid_queries, info.max_level) == (int(filled.sum()), invalid, top), label
                assert (info.num_samples, info.num_queries, info.k) == (ex[2].num_samples, len(allq), k), label
                if radius is None and len(prep.cand) >= k:
                    assert info.num_found == (len(allq) - invalid) * k, label


@pytest.mark.parametrize("stream", [uniform_stream, terrain_ragged_stream], ids=["uniform_1m", "terrain_ragged"])
def test_nearest_equals_the_restatement(sim, stream):
    batches, box, _ = stream()
    build(sim, batches, box)
    check(sim, box, np.concatenate(batches))


def test_nearest_of_a_36m_device_generated_terrain_stream(sim):
    n = 36_000_000
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        box = ((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.set_box(*box)
        sim.reset()
        sim.insert_device(dptr, n)
        rng = np.random.default_rng(2)
        pick = np.sort(rng.choice(n, 200_000, replace=False))
        points = sim.memcpy_dtoh(dptr, n * 16).view(api.POINT_DTYPE)[pick]
    finally:
        sim.device_free(dptr)
    assert sim.stats().dbg == 0 and sim.stats().numPointsProcessed == n
    check(sim, box, points, depths=(None, 3), ks=(8, 32), n=200)


def test_nearest_of_the_reference_kernels_octree_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    points = np.concatenate(batches)
    if all(os.path.exists(p) for p in oracle.REF_CUBINS.values()):
        build(sim, batches, box, reference=True)           # the query reads the ABI only
        check(sim, box, points, depths=(None, 2), ks=(8,), n=200)
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    sim.save_octree(path)
    sim.reset()
    sim.load_octree(path)
    check(sim, box, points, depths=(None, 2), ks=(8,), n=200)


def test_queries_straight_from_a_region_query_and_the_torch_path(sim):
    torch = pytest.importorskip("torch")
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cb = cube(sim, box)
    region = Region.sphere((2400.0, 2100.0, 100.0), 150.0)
    found, _ = sim.query_region(region, None, device="cuda")  # (N, 4) float32 on the device, passed as it is
    assert found.shape[0] > 100
    index, dist2, samples, info = sim.query_nearest(found, 8, samples=True)
    assert isinstance(index, torch.Tensor) and index.is_cuda and index.dtype == torch.int64 and tuple(index.shape) == (found.shape[0], 8)
    assert dist2.dtype == torch.float32 and tuple(samples.shape) == (found.shape[0], 8, 4)
    host = found.cpu().numpy()
    want_i, want_d = N.nearest(R.export_image(*sim.download_octree()), host, 8, None, *cb)
    assert index.cpu().numpy().tobytes() == want_i.tobytes() and dist2.cpu().numpy().tobytes() == want_d.tobytes()
    assert (dist2[:, 0] == 0).all()                          # every stored point finds itself (or a duplicate) first
    # numpy in, numpy out: the same bytes; (N, 3) and POINT_DTYPE queries are the same queries
    ni, nd, ns, ninfo = sim.query_nearest(host, 8, device="cpu", samples=True)
    assert ni.tobytes() == want_i.tobytes() and nd.tobytes() == want_d.tobytes()
    assert ns.tobytes() == samples.cpu().numpy().tobytes() and ninfo.num_found == info.num_found
    i3, d3, _ = sim.query_nearest(host[:, :3].copy(), 8, device="cpu")
    ip, dp, _ = sim.query_nearest(host.view(api.POINT_DTYPE).reshape(-1), 8, device="cpu")
    i3t, _, _ = sim.query_nearest(found[:, :3], 8)
    assert i3.tobytes() == ip.tobytes() == ni.tobytes() == i3t.cpu().numpy().tobytes() and d3.tobytes() == dp.tobytes() == nd.tobytes()


def test_protocol(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    rng = np.random.default_rng(8)
    n, k = 1000, 16
    q = np.zeros((n, 4), dtype=F)
    q[:, :3] = np.asarray(box[0]) + rng.uniform(0, 1, (n, 3)) * np.subtract(box[1], box[0])
    guard = 4096
    dq = sim.device_alloc(n * 16 + 32)
    di, dd, ds = (sim.device_alloc(n * k * w + 2 * guard) for w in (8, 4, 16))
    try:
        sim.memcpy_htod(dq, q)
        pats = [np.full(n * k * w + 2 * guard, 0x5A, dtype=np.uint8) for w in (8, 4, 16)]
        for p, pat in zip((di, dd, ds), pats):
            sim.memcpy_htod(p, pat)
        dst = (di + guard, dd + guard, ds + guard)
        launches = sim.launch_info()["launches"]
        refused = {"k_0": (dq, n, 0, None, None, dst), "k_33": (dq, n, 33, None, None, dst),
                   "n_0": (dq, 0, k, None, None, dst), "n_above_2^24": (dq, (1 << 24) + 1, k, None, None, dst),
                   "depth_21": (dq, n, k, 21, None, dst), "radius_nan": (dq, n, k, None, float("nan"), dst),
                   "radius_negative": (dq, n, k, None, -1.0, dst), "queries_null": (0, n, k, None, None, dst),
                   "queries_misaligned": (dq + 4, n, k, None, None, dst),
                   "index_misaligned": (dq, n, k, None, None, (dst[0] + 4, dst[1], dst[2])),
                   "dist2_misaligned": (dq, n, k, None, None, (dst[0], dst[1] + 2, dst[2])),
                   "samples_misaligned": (dq, n, k, None, None, (dst[0], dst[1], dst[2] + 8))}
        for name, (qp, nq, kk, depth, radius, d) in refused.items():
            with pytest.raises(SimlodError) as err:
                sim.query_nearest_into(qp, nq, kk, depth, radius, *d)
            assert err.value.code == -2, name
        assert sim.launch_info()["launches"] == launches       # refused before any launch
        for p, pat in zip((di, dd, ds), pats):
            assert (sim.memcpy_dtoh(p, len(pat)) == pat).all()
        for depth in (None, 3):
            info0, _ = sim.query_nearest_into(dq, n, k, depth, None, 0, 0, 0)   # info only: nothing written
            info1, ms = sim.query_nearest_into(dq, n, k, depth, None, *dst)
            assert ms > 0 and info1.num_found == info0.num_found == n * k
            want = sim.query_nearest(q, k, depth, device="cpu", samples=True)
            backs = [sim.memcpy_dtoh(p, len(pat)) for p, pat in zip((di, dd, ds), pats)]
            for back, w, pat in zip(backs, want[:3], pats):
                assert (back[:guard] == 0x5A).all() and (back[len(pat) - guard:] == 0x5A).all()
                assert back[guard:len(pat) - guard].tobytes() == w.tobytes()
            # repeat calls are byte-identical
            again = sim.query_nearest(q, k, depth, device="cpu", samples=True)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(again[:3], want[:3]))
            a, b = want[3], again[3]
            assert (a.num_found, a.samples_tested, a.records_visited) == (b.num_found, b.samples_tested, b.records_visited)
            assert a.plan_ms > 0 and a.search_ms > 0
    finally:
        for p in (dq, di, dd, ds):
            sim.device_free(p)


def test_nearest_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], sim.width, sim.height))
    sim.render()
    before = buffer_digests(sim)
    ring = sim.ring_slot(0, 1000).tobytes()
    q = query_sets(np.concatenate(batches[:1]), box, 300)
    for depth in (None, 2):
        for queries in q.values():
            sim.query_nearest(queries, 8, depth, device="cpu", samples=True)
    assert buffer_digests(sim) == before and sim.ring_slot(0, 1000).tobytes() == ring


def test_nearest_while_batches_are_pending_sees_the_last_completed_launch(sim):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for b in batches:
        sim.upload_batch(b)
    queries = query_sets(pts, (mn, mx), 300)["jittered"]
    snapshots = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        done = sim.stats().batchletIndex
        if done < len(batches):
            image = sim.download_octree()
            index, dist2, info = sim.query_nearest(queries, 8, device="cpu")
            want_i, want_d = N.nearest_image(*image, queries, 8, None, mn, mx)
            assert index.tobytes() == want_i.tobytes() and dist2.tobytes() == want_d.tobytes()
            assert info.num_found == len(queries) * 8 and info.num_samples >= done * 40_000
            snapshots += 1
    assert snapshots >= 1
