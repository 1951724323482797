"""GPU tests of the radius query (run with -m gpu on an H100): simlod_query_radius against its restatement
(radius_restatement over the export of the same device image, byte for byte) on several octrees, query sets, radii and
depths; the returned samples against export_octree(depth); small neighbourhoods against query_nearest and a few against
query_region(Region.sphere); and its protocol (refused arguments with guard bytes, the capacity refusal, launch counts,
repeatability, the torch and numpy paths, no writes into the context's buffers, batches pending in the ring)."""
import os

import numpy as np
import pytest

import export_restatement as R
import radius_restatement as S
import oracle
from simlod_b200 import Region, SimLOD, SimlodError, api, camera, data
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream
from test_nearest_gpu import cube, query_sets

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def radii(sim, stored):
    """0, about the point spacing, and one that holds hundreds of neighbours: from the median distance d32 of the 32nd
    nearest stored point of stored points, d32 / 5 and 3 d32 (about 300 neighbours on a surface, 860 in a volume)."""
    _, d2, _ = sim.query_nearest(stored, 32, device="cpu")
    d32 = float(np.sqrt(np.median(d2[:, 31].astype(np.float64))))
    return (0.0, d32 / 5.0, 3.0 * d32)


def size_query_offsets(sim, queries, r, depth):
    """The offsets a size query writes, through query_radius_into on memory of the test's own."""
    n = len(queries)
    dq, do = sim.device_alloc(n * 16), sim.device_alloc((n + 1) * 8)
    try:
        sim.memcpy_htod(dq, np.ascontiguousarray(queries, dtype=F))
        info, _ = sim.query_radius_into(dq, n, r, depth, do, 0, 0, 0, 0)
        return sim.memcpy_dtoh(do, (n + 1) * 8).view(np.int64), info
    finally:
        sim.device_free(dq)
        sim.device_free(do)


def check(sim, box, points, depths=None, sets=None, n=300, nearest=True):
    """Every query set at every depth and radius: offsets, index and dist2 byte-identical to the restatement of the
    image, the samples those of export_octree(depth), the counts, the size query's offsets, and the neighbourhoods of
    at most 32 samples equal to query_nearest(k=32, max_radius=r)."""
    image = sim.download_octree()
    cb = cube(sim, box)
    full = R.export_image(*image)
    top = full[2].max_level
    queries = query_sets(points, box, n)
    if sets is not None:
        queries = {k: v for k, v in queries.items() if k in sets}
    allq = np.concatenate(list(queries.values()))
    invalid = int((~np.isfinite(allq[:, :3]).all(axis=1)).sum())
    rs = radii(sim, query_sets(points, box, n)["stored"])
    for depth in (sorted({0, 3, top}, key=int) + [None] if depths is None else depths):
        ex = full if depth is None else R.export_image(*image, depth)
        dev = sim.export_octree(depth, device="cpu")
        assert dev.samples.tobytes() == ex[1].tobytes()
        prep = S.Prepared(ex, depth, *cb)
        for r in rs:
            label = "depth %s radius %s" % (depth, r)
            offsets, index, dist2, got, info = sim.query_radius(allq, r, depth, device="cpu", samples=True)
            want_o, want_i, want_d = S.search(prep, allq, r)
            assert offsets.tobytes() == want_o.tobytes(), label
            assert index.tobytes() == want_i.tobytes(), label
            assert dist2.tobytes() == want_d.tobytes(), label
            assert got.tobytes() == dev.samples[index].tobytes(), label
            counts = np.diff(offsets)
            assert (info.num_found, info.max_found, info.invalid_queries, info.max_level) == \
                (int(offsets[-1]), int(counts.max()), invalid, top), label
            assert (info.num_samples, info.num_queries) == (ex[2].num_samples, len(allq)), label
            # the size query's offsets are the full call's
            size_offsets, sinfo = size_query_offsets(sim, allq, r, depth)
            assert size_offsets.tobytes() == offsets.tobytes() and sinfo.num_found == info.num_found, label
            if nearest:
                ni, nd, _ = sim.query_nearest(allq, 32, depth, r, device="cpu")
                for t in np.nonzero(counts <= 32)[0]:
                    a, b = offsets[t], offsets[t + 1]
                    o = np.lexsort((index[a:b], dist2[a:b]))
                    filled = ni[t] >= 0
                    assert index[a:b][o].tolist() == ni[t][filled].tolist() and dist2[a:b][o].tobytes() == nd[t][filled].tobytes(), label
    return allq


@pytest.mark.parametrize("stream", [uniform_stream, terrain_ragged_stream], ids=["uniform_1m", "terrain_ragged"])
def test_radius_equals_the_restatement(sim, stream):
    batches, box, _ = stream()
    build(sim, batches, box)
    check(sim, box, np.concatenate(batches))


def test_radius_of_a_36m_device_generated_terrain_stream(sim):
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
    check(sim, box, points, depths=(None, 3), sets=("stored", "jittered", "uniform", "non_finite"), n=200, nearest=False)


def test_radius_of_the_reference_kernels_octree_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    points = np.concatenate(batches)
    if all(os.path.exists(p) for p in oracle.REF_CUBINS.values()):
        build(sim, batches, box, reference=True)           # the query reads the ABI only
        check(sim, box, points, depths=(None, 2), n=150, nearest=False)
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    sim.save_octree(path)
    sim.reset()
    sim.load_octree(path)
    check(sim, box, points, depths=(None, 2), n=150, nearest=False)


def test_region_spheres_queries_from_a_region_query_and_the_torch_path(sim):
    torch = pytest.importorskip("torch")
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cb = cube(sim, box)
    found, _ = sim.query_region(Region.sphere((2400.0, 2100.0, 100.0), 150.0), None, device="cuda")
    assert found.shape[0] > 100                               # (N, 4) float32 on the device, passed as it is
    r = 4.0
    offsets, index, dist2, samples, info = sim.query_radius(found, r, samples=True)
    assert isinstance(offsets, torch.Tensor) and offsets.is_cuda and offsets.dtype == torch.int64
    assert tuple(offsets.shape) == (found.shape[0] + 1,) and index.dtype == torch.int64 and dist2.dtype == torch.float32
    assert tuple(samples.shape) == (info.num_found, 4) and tuple(index.shape) == (info.num_found,)
    host = found.cpu().numpy()
    want = S.radius(R.export_image(*sim.download_octree()), host, r, None, *cb)
    for g, w in zip((offsets, index, dist2), want):
        assert g.cpu().numpy().tobytes() == w.tobytes()
    assert (np.diff(want[0]) >= 1).all()                     # every stored point finds itself
    # a few neighbourhoods equal query_region(Region.sphere) as multisets of sample bytes
    off = want[0]
    samples_h = samples.cpu().numpy()
    for t in (0, 7, len(host) // 2):
        sphere, _ = sim.query_region(Region.sphere(host[t, :3], r), None, device="cpu")
        mine = samples_h[off[t]:off[t + 1]].view(api.POINT_DTYPE).reshape(-1)
        assert sorted(mine.tobytes()[i:i + 16] for i in range(0, len(mine) * 16, 16)) == \
            sorted(sphere.tobytes()[i:i + 16] for i in range(0, len(sphere) * 16, 16)), t
    # numpy in, numpy out: the same bytes; (N, 3), POINT_DTYPE and (N, 3) tensor queries are the same queries
    no, ni, nd, ns, ninfo = sim.query_radius(host, r, device="cpu", samples=True)
    assert no.tobytes() == want[0].tobytes() and ni.tobytes() == want[1].tobytes() and nd.tobytes() == want[2].tobytes()
    assert ns.tobytes() == samples_h.tobytes() and ninfo.num_found == info.num_found
    o3, i3, d3, _ = sim.query_radius(host[:, :3].copy(), r, device="cpu")
    op, ip, dp, _ = sim.query_radius(host.view(api.POINT_DTYPE).reshape(-1), r, device="cpu")
    ot, it, dt, _ = sim.query_radius(found[:, :3], r)
    for a, b, c, d in ((o3, op, no, ot), (i3, ip, ni, it), (d3, dp, nd, dt)):
        assert a.tobytes() == b.tobytes() == c.tobytes() == d.cpu().numpy().tobytes()


def test_protocol(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    points = np.concatenate(batches)
    rng = np.random.default_rng(8)
    n, r = 1000, 6.0
    q = np.zeros((n, 4), dtype=F)
    q[:, :3] = np.stack([points["x"], points["y"], points["z"]], axis=1)[rng.choice(len(points), n)]
    m = sim.query_radius(q, r, device="cpu")[3].num_found
    assert m > n
    guard = 4096
    dq = sim.device_alloc(n * 16 + 32)
    widths = (8, 8, 4, 16)                                    # offsets (n + 1), index, dist2, samples (m each)
    sizes = [(n + 1) * 8] + [m * w for w in widths[1:]]
    bufs = [sim.device_alloc(s + 2 * guard) for s in sizes]
    try:
        sim.memcpy_htod(dq, q)
        pats = [np.full(s + 2 * guard, 0x5A, dtype=np.uint8) for s in sizes]

        def reset_guards():
            for p, pat in zip(bufs, pats):
                sim.memcpy_htod(p, pat)

        def untouched():
            return all((sim.memcpy_dtoh(p, len(pat)) == pat).all() for p, pat in zip(bufs, pats))

        reset_guards()
        dst = tuple(p + guard for p in bufs)
        launches = sim.launch_info()["launches"]
        refused = {"radius_nan": (dq, n, float("nan"), None, dst), "radius_negative": (dq, n, -1.0, None, dst),
                   "radius_inf": (dq, n, float("inf"), None, dst), "n_0": (dq, 0, r, None, dst),
                   "n_above_2^24": (dq, (1 << 24) + 1, r, None, dst), "depth_21": (dq, n, r, 21, dst),
                   "queries_null": (0, n, r, None, dst), "queries_misaligned": (dq + 4, n, r, None, dst),
                   "offsets_misaligned": (dq, n, r, None, (dst[0] + 4,) + dst[1:]),
                   "index_misaligned": (dq, n, r, None, (dst[0], dst[1] + 4) + dst[2:]),
                   "dist2_misaligned": (dq, n, r, None, dst[:2] + (dst[2] + 2, dst[3])),
                   "samples_misaligned": (dq, n, r, None, dst[:3] + (dst[3] + 8,))}
        for name, (qp, nq, rad, depth, d) in refused.items():
            with pytest.raises(SimlodError) as err:
                sim.query_radius_into(qp, nq, rad, depth, *d, m)
            assert err.value.code == -2, name
        assert sim.launch_info()["launches"] == launches       # refused before any launch
        assert untouched()
        # a capacity one short: refused after the count, nothing written, info filled
        info = api.SimlodRadiusInfo()
        rc = sim._lib.simlod_query_radius(sim._ctx, dq, n, r, -1, *dst, m - 1, api.C.byref(info), None)
        assert rc == -2 and info.num_found == m and untouched()
        # launch counts: fixed for the size query and the full call
        before = sim.launch_info()["launches"]
        sim.query_radius_into(dq, n, r, None, 0, 0, 0, 0, 0)
        size_launches = sim.launch_info()["launches"] - before
        before = sim.launch_info()["launches"]
        info1, ms = sim.query_radius_into(dq, n, r, None, *dst, m)
        full_launches = sim.launch_info()["launches"] - before
        assert (size_launches, full_launches) == (2 + 3 + 3, 2 + 3 + 3 + 1) and ms > 0
        assert info1.num_found == m and info1.plan_ms > 0 and info1.count_ms > 0 and info1.write_ms > 0
        want = sim.query_radius(q, r, device="cpu", samples=True)
        backs = [sim.memcpy_dtoh(p, len(pat)) for p, pat in zip(bufs, pats)]
        for back, w, pat in zip(backs, want[:4], pats):
            assert (back[:guard] == 0x5A).all() and (back[len(pat) - guard:] == 0x5A).all()
            assert back[guard:len(pat) - guard].tobytes() == w.tobytes()
        # repeat calls are byte-identical
        for depth in (None, 3):
            a = sim.query_radius(q, r, depth, device="cpu", samples=True)
            b = sim.query_radius(q, r, depth, device="cpu", samples=True)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a[:4], b[:4]))
            assert (a[4].num_found, a[4].samples_tested, a[4].records_visited, a[4].max_found) == \
                (b[4].num_found, b[4].samples_tested, b[4].records_visited, b[4].max_found)
    finally:
        for p in [dq] + bufs:
            sim.device_free(p)


def test_radius_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], sim.width, sim.height))
    sim.render()
    before = buffer_digests(sim)
    ring = sim.ring_slot(0, 1000).tobytes()
    q = query_sets(np.concatenate(batches[:1]), box, 300)
    for depth in (None, 2):
        for queries in q.values():
            sim.query_radius(queries, 5.0, depth, device="cpu", samples=True)
    assert buffer_digests(sim) == before and sim.ring_slot(0, 1000).tobytes() == ring


def test_radius_while_batches_are_pending_sees_the_last_completed_launch(sim):
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
            got = sim.query_radius(queries, 6.0, device="cpu")
            want = S.radius_image(*image, queries, 6.0, None, mn, mx)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got[:3], want))
            assert got[3].num_samples >= done * 40_000
            snapshots += 1
    assert snapshots >= 1
