"""GPU tests of what the export's plan consumers share (run with -m gpu on an H100): the launches of pick, k nearest and
rays, the kernel time each of pick, nearest, radius and rays returns as the sum of its info's stage times, the empty
results of a region query and a radius query, and one context's scratch reused by all four in turn."""
import numpy as np
import pytest

from simlod_b200 import Region, SimLOD, api, camera, data

pytestmark = pytest.mark.gpu

W, H = 320, 180


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(W, H, persistent_bytes=2 << 30)
    pts, mn, mx = data.uniform_cube(1_000_000, size=64.0, seed=5)
    s.set_box(mn, mx)
    s.reset()
    s.insert(pts)
    s.set_camera(*camera.autofocus(mx, W, H))
    st = s.stats()
    assert st.dbg == 0 and st.numNodes > 8 and st.numVoxels > 0
    s.pts, s.mn, s.mx = pts, np.asarray(mn, np.float32), np.asarray(mx, np.float32)
    yield s
    s.close()


@pytest.fixture()
def device(sim):
    """device_alloc whose allocations are freed after the test."""
    ptrs = []

    def alloc(nbytes):
        ptrs.append(sim.device_alloc(max(int(nbytes), 16)))
        return ptrs[-1]
    yield alloc
    for p in ptrs:
        sim.device_free(p)


def launches_of(sim, call):
    before = sim.launch_info()["launches"]
    out = call()
    return sim.launch_info()["launches"] - before, out


def stage_sum(*ms):
    """The float32 sum of the stage times, left to right, as the library adds them."""
    total = np.float32(ms[0])
    for m in ms[1:]:
        total = np.float32(total + np.float32(m))
    return float(total)


def jittered(sim, n, seed):
    rng = np.random.default_rng(seed)
    p = sim.pts[rng.integers(0, len(sim.pts), n)]
    return np.stack([p["x"], p["y"], p["z"]], axis=1).astype(np.float32) + rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)


def staged(sim, device, a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    ptr = device(a.nbytes)
    sim.memcpy_htod(ptr, a)
    return ptr


def queries4(q):
    out = np.zeros((len(q), 4), dtype=np.float32)
    out[:, :3] = q
    return out


def rays8(sim, n, seed):
    rng = np.random.default_rng(seed)
    p = sim.pts[rng.integers(0, len(sim.pts), n)]
    r = np.zeros((n, 8), dtype=np.float32)
    r[:, 0], r[:, 1], r[:, 2] = p["x"], p["y"], np.float32(100.0)
    r[:, 6], r[:, 7] = -1.0, np.inf
    return r


@pytest.mark.parametrize("pixels", [None, [[0, 0], [W // 2, H // 2], [W - 1, H - 1]]])
def test_pick_launches_and_stage_times(sim, device, pixels):
    n = W * H if pixels is None else len(pixels)
    launches, (info, ms) = launches_of(sim, lambda: sim.pick_into(pixels, 0, 0))
    assert launches == 3 + 4
    assert ms == stage_sum(info.plan_ms, info.key_ms, info.index_ms, info.write_ms) and ms > 0
    di, ds = device(n * 8), device(n * 16)
    launches, (info, ms) = launches_of(sim, lambda: sim.pick_into(pixels, di, ds))
    assert launches == 3 + 4 and info.num_pixels == n
    assert ms == stage_sum(info.plan_ms, info.key_ms, info.index_ms, info.write_ms)


@pytest.mark.parametrize("depth", [None, 3])
def test_nearest_launches_and_stage_times(sim, device, depth):
    n, k = 1000, 4
    qptr = staged(sim, device, queries4(jittered(sim, n, 1)))
    launches, (info, ms) = launches_of(sim, lambda: sim.query_nearest_into(qptr, n, k, depth, None, 0, 0, 0))
    assert launches == 2 + 3 + 1
    assert ms == stage_sum(info.plan_ms, info.bucket_ms, info.search_ms) and ms > 0
    di, dd, ds = device(n * k * 8), device(n * k * 4), device(n * k * 16)
    launches, (info, ms) = launches_of(sim, lambda: sim.query_nearest_into(qptr, n, k, depth, None, di, dd, ds))
    assert launches == 2 + 3 + 1 and info.num_found == n * k
    assert ms == stage_sum(info.plan_ms, info.bucket_ms, info.search_ms)


@pytest.mark.parametrize("depth", [None, 3])
def test_ray_launches_and_stage_times(sim, device, depth):
    n = 1000
    rptr = staged(sim, device, rays8(sim, n, 2))
    launches, (info, ms) = launches_of(sim, lambda: sim.query_ray_into(rptr, n, 0.5, depth, 0, 0, 0, 0))
    assert launches == 2 + 2
    assert ms == stage_sum(info.plan_ms, info.trace_ms) and ms > 0
    di, dt, dh, ds = device(n * 8), device(n * 4), device(n * 4), device(n * 16)
    launches, (info, ms) = launches_of(sim, lambda: sim.query_ray_into(rptr, n, 0.5, depth, di, dt, dh, ds))
    assert launches == 2 + 2 and info.num_rays == n
    assert ms == stage_sum(info.plan_ms, info.trace_ms)


def test_radius_stage_times(sim, device):
    n = 1000
    qptr = staged(sim, device, queries4(jittered(sim, n, 3)))
    info, ms = sim.query_radius_into(qptr, n, 0.5, None, 0, 0, 0, 0, 0)
    assert info.write_ms == 0.0 and ms == stage_sum(info.plan_ms, info.bucket_ms, info.count_ms) and ms > 0
    m = info.num_found
    assert m > 0
    do, di, dd, ds = device((n + 1) * 8), device(m * 8), device(m * 4), device(m * 16)
    info, ms = sim.query_radius_into(qptr, n, 0.5, None, do, di, dd, ds, m)
    assert info.num_found == m and ms == stage_sum(info.plan_ms, info.bucket_ms, info.count_ms, info.write_ms)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
def test_empty_region(sim, device):
    import torch
    far = sim.mx + 100.0
    samples, info = sim.query_region(Region.box(far, far + 1.0), None, device=device)
    assert info.num_samples == 0
    if device == "cpu":
        assert isinstance(samples, np.ndarray) and samples.dtype == api.POINT_DTYPE and samples.shape == (0,)
    else:
        assert samples.is_cuda and samples.dtype == torch.float32 and tuple(samples.shape) == (0, 4)


@pytest.mark.parametrize("device", ["cpu", "cuda"])
@pytest.mark.parametrize("samples", [False, True])
def test_radius_without_neighbours_runs_its_write_pass(sim, device, samples):
    import torch
    n = 5
    q = np.tile(sim.mx + 100.0, (n, 1)).astype(np.float32)
    before = sim.launch_info()["launches"]
    out = sim.query_radius(q, 1.0, device=device, samples=samples)
    assert sim.launch_info()["launches"] - before == (2 + 3 + 3) + (2 + 3 + 3 + 1)
    info = out[-1]
    assert info.num_found == 0 and info.num_queries == n
    offsets, index, dist2 = out[0], out[1], out[2]
    if device == "cpu":
        assert offsets.dtype == np.int64 and offsets.shape == (n + 1,) and not offsets.any()
        assert index.dtype == np.int64 and index.shape == (0,)
        assert dist2.dtype == np.float32 and dist2.shape == (0,)
        if samples:
            assert out[3].dtype == api.POINT_DTYPE and out[3].shape == (0,)
    else:
        assert offsets.dtype == torch.int64 and tuple(offsets.shape) == (n + 1,) and not offsets.any()
        assert index.dtype == torch.int64 and tuple(index.shape) == (0,)
        assert dist2.dtype == torch.float32 and tuple(dist2.shape) == (0,)
        if samples:
            assert out[3].dtype == torch.float32 and tuple(out[3].shape) == (0, 4)


def test_scratch_reused_by_every_consumer(sim):
    """A radius query large enough that its scratch outgrows the others', then a one-pixel pick, 1 k nearest queries,
    rays and the same radius query: each result byte for byte the same call's made before the radius query ran."""
    big = jittered(sim, 60_000, 4)
    near = jittered(sim, 1000, 5)
    r = rays8(sim, 1000, 6)
    origins, directions = r[:, 0:3], r[:, 4:7]

    def as_bytes(out):
        return [x.tobytes() for x in out[:-1]]

    def pick():
        return as_bytes(sim.pick([[W // 2, H // 2]], device="cpu", samples=True))

    def nearest():
        return as_bytes(sim.query_nearest(near, 8, device="cpu", samples=True))

    def ray():
        return as_bytes(sim.query_ray(origins, directions, 0.5, device="cpu", samples=True))

    def radius():
        return as_bytes(sim.query_radius(big, 0.5, device="cpu", samples=True))

    alone = {"pick": pick(), "nearest": nearest(), "ray": ray()}
    first = radius()
    assert sum(len(b) for b in first) > 0
    assert pick() == alone["pick"]
    assert nearest() == alone["nearest"]
    assert ray() == alone["ray"]
    assert radius() == first
