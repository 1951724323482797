"""GPU tests of the ray query (run with -m gpu on an H100): simlod_query_ray against its restatement (ray_restatement over
the export of the same device image, byte for byte) on several octrees and ray sets, the returned samples against
export_octree(depth), and its protocol (refused arguments with guard bytes, repeatability, the torch and numpy paths, no
writes into the context's buffers, batches pending in the ring)."""
import os

import numpy as np
import pytest

import export_restatement as R
import oracle
import ray_restatement as Y
from simlod_b200 import SimLOD, SimlodError, api, camera, data
from test_export_gpu import buffer_digests, build, terrain_ragged_stream, uniform_stream

pytestmark = pytest.mark.gpu

F = np.float32
INF = float("inf")
NAN = float("nan")


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30)
    yield s
    s.close()


def cube(sim, box):
    """(boxMin, boxMax, the device's reciprocal of the cube size) for the restatement."""
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    return box[0], box[1], sim.device_rcp(size)


def ray_sets(points, box, n=96, seed=1):
    """Named (n, 8) float32 ray arrays: camera rays through pixel centres, vertical rays from above, random rays through
    the cube, segments between two stored points, rays from 10^6 cube sizes away, axis-parallel rays (origins on node
    faces among them) and a mix of invalid and valid rays."""
    rng = np.random.default_rng(seed)
    mn = np.asarray(box[0], dtype=np.float64)
    mx = np.asarray(box[1], dtype=np.float64)
    size = float(np.max(mx - mn))
    xyz = np.stack([points["x"], points["y"], points["z"]], axis=1).astype(np.float64)
    a, b = xyz[rng.choice(len(xyz), n)], xyz[rng.choice(len(xyz), n)]
    view, proj = camera.autofocus(mx - mn, 64, 36)
    view = view @ camera.translate(-mn)
    pix = np.stack([rng.integers(0, 64, n), rng.integers(0, 36, n)], axis=1)
    co, cd = camera.pixel_rays(view, proj, 64, 36, pix)
    top = np.tile([[0.0, 0.0, mx[2] + 0.1 * size]], (n, 1))
    top[:, :2] = a[:, :2] + rng.normal(0, size * 1e-3, (n, 2))
    inside = mn + rng.uniform(0, 1, (n, 3)) * size
    start = mn + rng.uniform(-0.5, 1.5, (n, 3)) * size
    far_dir = rng.normal(0, 1, (n, 3))
    far_dir /= np.linalg.norm(far_dir, axis=1)[:, None]
    far = a - far_dir * size * 1e6
    axis = rng.integers(0, 3, n)
    ao = mn + rng.uniform(0, 1, (n, 3)) * size
    ad = np.zeros((n, 3))
    ad[np.arange(n), axis] = rng.choice([-1.0, 1.0], n)
    on_face = mn + rng.integers(0, 9, (n, 3)) * (size / 8)                 # origins on node faces of levels <= 3
    ao[::2] = np.where(ad[::2] != 0, ao[::2], on_face[::2])
    ao[np.arange(n), axis] = np.where(ad[np.arange(n), axis] > 0, mn[axis] - 0.01 * size, mn[axis] + 1.01 * size)
    ao[1::4] = np.where(ad[1::4] != 0, ao[1::4], a[1::4])                # axis-parallel through stored points
    bad_o, bad_d = inside.copy(), b - inside
    bad_t0, bad_t1 = np.zeros(n), np.full(n, np.inf)
    bad_o[0::8, 0] = np.nan
    bad_o[1::8, 1] = np.inf
    bad_d[2::8] = 0.0
    bad_d[3::8, 2] = -np.inf
    bad_t0[4::8] = -1.0
    bad_t0[5::8] = np.nan
    bad_t1[6::8] = -0.5
    sets = {"camera": Y.rays(co, cd), "vertical": Y.rays(top, np.tile([[0.0, 0.0, -1.0]], (n, 1))),
            "random": Y.rays(start, inside - start), "segments": Y.rays(a, b - a, 0.0, np.linalg.norm(b - a, axis=1)),
            "far": Y.rays(far, far_dir, size * 1e6 - 2 * size), "axis": Y.rays(ao, ad),
            "invalid": Y.rays(bad_o, bad_d, bad_t0, bad_t1)}
    return sets


def check(sim, box, points, depths=None, radii=("small", 0.0), sets=None, n=96):
    """Every ray set at every depth and radius: index, t and h2 byte-identical to the restatement of the image, the
    samples those of export_octree(depth), the counts as expected."""
    image = sim.download_octree()
    cb = cube(sim, box)
    full = R.export_image(*image)
    top = full[2].max_level
    size = float(np.max(np.subtract(box[1], box[0]).astype(F)))
    rays = ray_sets(points, box, n)
    if sets is not None:
        rays = {k: v for k, v in rays.items() if k in sets}
    allr = np.concatenate(list(rays.values()))
    invalid = int((~Y.valid(allr)).sum())
    assert invalid >= (n * 7 // 8 if "invalid" in rays else 0)
    for depth in (sorted({0, 3, top}, key=int) + [None] if depths is None else depths):
        ex = full if depth is None else R.export_image(*image, depth)
        dev = sim.export_octree(depth, device="cpu")
        assert dev.samples.tobytes() == ex[1].tobytes()
        prep = Y.Prepared(ex, depth, *cb)
        for radius in radii:
            r = size / 500.0 if radius == "small" else radius
            label = "depth %s radius %s" % (depth, r)
            index, t, h2, got, info = sim.query_ray(allr[:, 0:3], allr[:, 4:7], r, allr[:, 3], allr[:, 7], depth,
                                                    device="cpu", samples=True)
            want = Y.search(prep, allr, r)
            for a, w, what in zip((index, t, h2), want, ("index", "t", "h2")):
                diff = np.nonzero(a != w)[0]
                assert a.tobytes() == w.tobytes(), "%s: %s differs for rays %s: got %r want %r" % (label, what, diff[:8], a[diff[:8]], w[diff[:8]])
            hit = index >= 0
            expect = np.zeros(len(index), dtype=api.POINT_DTYPE)
            expect[hit] = dev.samples[index[hit]]
            assert got.tobytes() == expect.tobytes(), label
            assert (info.num_hits, info.invalid_rays, info.max_level) == (int(hit.sum()), invalid, top), label
            assert (info.num_samples, info.num_rays) == (ex[2].num_samples, len(allr)), label
            assert info.samples_tested >= info.records_visited
            if r > 0:
                names = list(rays)
                seg = slice(names.index("segments") * n, (names.index("segments") + 1) * n) if "segments" in rays else None
                if seg is not None and depth is None:
                    assert hit[seg].all(), label                # the segment's first stored point is on it


@pytest.mark.parametrize("stream", [uniform_stream, terrain_ragged_stream], ids=["uniform_1m", "terrain_ragged"])
def test_ray_equals_the_restatement(sim, stream):
    batches, box, _ = stream()
    build(sim, batches, box)
    check(sim, box, np.concatenate(batches))


def test_ray_of_a_36m_device_generated_terrain_stream(sim):
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
    check(sim, box, points, depths=(None, 3), n=48)


def test_ray_of_the_reference_kernels_octree_and_of_a_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    points = np.concatenate(batches)
    if all(os.path.exists(p) for p in oracle.REF_CUBINS.values()):
        build(sim, batches, box, reference=True)           # the query reads the ABI only
        check(sim, box, points, depths=(None, 2), n=48)
    build(sim, batches, box)
    path = str(tmp_path / "t.octree")
    sim.save_octree(path)
    sim.reset()
    sim.load_octree(path)
    check(sim, box, points, depths=(None, 2), n=48)


def test_torch_and_numpy_paths_agree(sim):
    torch = pytest.importorskip("torch")
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    r = np.concatenate([v for k, v in ray_sets(np.concatenate(batches), box, 64).items()])
    tmin, tmax = r[:, 3].copy(), r[:, 7].copy()
    ni, nt, nh, ns, ninfo = sim.query_ray(r[:, 0:3], r[:, 4:7], 1.0, tmin, tmax, device="cpu", samples=True)
    o, d = torch.from_numpy(r[:, 0:3].copy()).cuda(), torch.from_numpy(r[:, 4:7].copy()).cuda()
    ti, tt, th, ts, tinfo = sim.query_ray(o, d, 1.0, torch.from_numpy(tmin).cuda(), torch.from_numpy(tmax).cuda(), samples=True)
    assert isinstance(ti, torch.Tensor) and ti.is_cuda and ti.dtype == torch.int64 and tuple(ti.shape) == (len(r),)
    assert tt.dtype == torch.float32 and tuple(ts.shape) == (len(r), 4)
    assert ti.cpu().numpy().tobytes() == ni.tobytes() and tt.cpu().numpy().tobytes() == nt.tobytes()
    assert th.cpu().numpy().tobytes() == nh.tobytes() and ts.cpu().numpy().tobytes() == ns.tobytes()
    assert (tinfo.num_hits, tinfo.invalid_rays) == (ninfo.num_hits, ninfo.invalid_rays) and ninfo.num_hits > 0
    # scalar bounds are every ray's bounds
    si, st, _, _ = sim.query_ray(r[:, 0:3], r[:, 4:7], 1.0, 0.0, None, device="cpu")
    vi, vt, _, _ = sim.query_ray(r[:, 0:3], r[:, 4:7], 1.0, np.zeros(len(r)), np.full(len(r), np.inf), device="cpu")
    assert si.tobytes() == vi.tobytes() and st.tobytes() == vt.tobytes()


def test_protocol(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    rng = np.random.default_rng(8)
    n = 1000
    mx = np.asarray(box[1])
    points = np.concatenate(batches)
    top = np.zeros((n, 3))
    top[:, :2] = np.stack([points["x"], points["y"]], axis=1)[rng.choice(len(points), n)]   # above stored points
    top[:, 2] = mx[2] + 10.0
    r = Y.rays(top, np.tile([[0.0, 0.0, -1.0]], (n, 1)))
    guard = 4096
    dr = sim.device_alloc(n * 32 + 32)
    di, dt, dh, ds = (sim.device_alloc(n * w + 2 * guard) for w in (8, 4, 4, 16))
    try:
        sim.memcpy_htod(dr, r)
        pats = [np.full(n * w + 2 * guard, 0x5A, dtype=np.uint8) for w in (8, 4, 4, 16)]
        for p, pat in zip((di, dt, dh, ds), pats):
            sim.memcpy_htod(p, pat)
        dst = (di + guard, dt + guard, dh + guard, ds + guard)
        launches = sim.launch_info()["launches"]
        refused = {"radius_nan": (dr, n, NAN, None, dst), "radius_inf": (dr, n, INF, None, dst),
                   "radius_negative": (dr, n, -1.0, None, dst), "n_0": (dr, 0, 1.0, None, dst),
                   "n_above_2^24": (dr, (1 << 24) + 1, 1.0, None, dst), "depth_21": (dr, n, 1.0, 21, dst),
                   "rays_null": (0, n, 1.0, None, dst), "rays_misaligned": (dr + 8, n, 1.0, None, dst),
                   "index_misaligned": (dr, n, 1.0, None, (dst[0] + 4, dst[1], dst[2], dst[3])),
                   "t_misaligned": (dr, n, 1.0, None, (dst[0], dst[1] + 2, dst[2], dst[3])),
                   "h2_misaligned": (dr, n, 1.0, None, (dst[0], dst[1], dst[2] + 1, dst[3])),
                   "samples_misaligned": (dr, n, 1.0, None, (dst[0], dst[1], dst[2], dst[3] + 8))}
        for name, (rp, nr, radius, depth, d) in refused.items():
            with pytest.raises(SimlodError) as err:
                sim.query_ray_into(rp, nr, radius, depth, *d)
            assert err.value.code == -2, name
        assert sim.launch_info()["launches"] == launches       # refused before any launch
        for p, pat in zip((di, dt, dh, ds), pats):
            assert (sim.memcpy_dtoh(p, len(pat)) == pat).all()
        for depth in (None, 3):
            info0, _ = sim.query_ray_into(dr, n, 10.0, depth, 0, 0, 0, 0)   # info only: nothing written
            info1, ms = sim.query_ray_into(dr, n, 10.0, depth, *dst)
            assert ms > 0 and info1.num_hits == info0.num_hits == n
            want = sim.query_ray(r[:, 0:3], r[:, 4:7], 10.0, depth=depth, device="cpu", samples=True)
            backs = [sim.memcpy_dtoh(p, len(pat)) for p, pat in zip((di, dt, dh, ds), pats)]
            for back, w, pat in zip(backs, want[:4], pats):
                assert (back[:guard] == 0x5A).all() and (back[len(pat) - guard:] == 0x5A).all()
                assert back[guard:len(pat) - guard].tobytes() == w.tobytes()
            # repeat calls are byte-identical
            again = sim.query_ray(r[:, 0:3], r[:, 4:7], 10.0, depth=depth, device="cpu", samples=True)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(again[:4], want[:4]))
            a, b = want[4], again[4]
            assert (a.num_hits, a.samples_tested, a.records_visited) == (b.num_hits, b.samples_tested, b.records_visited)
            assert a.plan_ms > 0 and a.trace_ms > 0
    finally:
        for p in (dr, di, dt, dh, ds):
            sim.device_free(p)


def test_ray_writes_nothing_into_the_context(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], sim.width, sim.height))
    sim.render()
    before = buffer_digests(sim)
    ring = sim.ring_slot(0, 1000).tobytes()
    for depth in (None, 2):
        for r in ray_sets(np.concatenate(batches[:1]), box, 64).values():
            sim.query_ray(r[:, 0:3], r[:, 4:7], 1.0, r[:, 3], r[:, 7], depth, device="cpu", samples=True)
    assert buffer_digests(sim) == before and sim.ring_slot(0, 1000).tobytes() == ring


def test_ray_while_batches_are_pending_sees_the_last_completed_launch(sim):
    pts, mn, mx = data.uniform_cube(1_000_000, size=512.0, seed=31)
    batches = np.split(pts, 25)               # 25 batches of 40 000: one launch consumes at most 20
    sim.set_box(mn, mx)
    sim.reset()
    for b in batches:
        sim.upload_batch(b)
    r = ray_sets(pts, (mn, mx), 64)["random"]
    snapshots = 0
    while sim.stats().batchletIndex < len(batches):
        sim.update_octree()
        done = sim.stats().batchletIndex
        if done < len(batches):
            image = sim.download_octree()
            index, t, h2, info = sim.query_ray(r[:, 0:3], r[:, 4:7], 2.0, device="cpu")
            want = Y.trace_image(*image, r, 2.0, None, mn, mx)
            assert index.tobytes() == want[0].tobytes() and t.tobytes() == want[1].tobytes() and h2.tobytes() == want[2].tobytes()
            assert info.num_hits == int((index >= 0).sum()) > 0 and info.num_samples >= done * 40_000
            snapshots += 1
    assert snapshots >= 1
