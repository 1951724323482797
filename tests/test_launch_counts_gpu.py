"""GPU tests of the launch counter (run with -m gpu on an H100): how much launch_info()["launches"] grows across one C call,
for every call whose number of launches does not depend on timing. bench.py derives its launch counts from this counter,
so a launch that is not counted, counted twice, dropped or run twice shows up here."""
import numpy as np
import pytest

from simlod_b200 import Region, SimLOD, SimlodError, camera, data

pytestmark = pytest.mark.gpu

WINDOW_SAMPLES = 16_000_000          # samples an octree file stages per window: half the 512 MB page-locked pool


@pytest.fixture(scope="module")
def sim():
    s = SimLOD(320, 180, persistent_bytes=2 << 30)
    pts, mn, mx = data.uniform_cube(1_000_000, size=64.0, seed=5)
    s.set_box(mn, mx)
    s.reset()
    s.insert(pts)
    s.set_camera(*camera.autofocus(mx, 320, 180))
    st = s.stats()
    assert st.dbg == 0 and st.numNodes > 8 and st.numVoxels > 0
    s.box = (np.asarray(mn, np.float64), np.asarray(mx, np.float64))
    yield s
    s.close()


def launches_of(sim, call):
    before = sim.launch_info()["launches"]
    call()
    return sim.launch_info()["launches"] - before


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


def test_render_flush_rcp_and_generate(sim, device):
    assert launches_of(sim, sim.render) == 1
    assert launches_of(sim, sim.flush_l2) == 1
    assert launches_of(sim, lambda: sim.device_rcp(3.0)) == 1
    dst = device(1000 * 16)
    for kind in (sim.GEN_UNIFORM, sim.GEN_TERRAIN, sim.GEN_SHELL):
        assert launches_of(sim, lambda: sim.generate(kind, dst, 1000, 0, 1000, 3, 64.0)) == 1, kind


@pytest.mark.parametrize("depth", [None, 2])
def test_export_octree(sim, device, depth):
    info, _ = sim.export_octree_into(depth, 0, 0, 0, 0)
    assert launches_of(sim, lambda: sim.export_octree_into(depth, 0, 0, 0, 0)) == 2
    dn, ds = device(info.num_nodes * 64), device(info.num_samples * 16)
    assert launches_of(sim, lambda: sim.export_octree_into(depth, dn, info.num_nodes, ds, info.num_samples)) == 3


def test_export_view(sim, device):
    info, _ = sim.export_view_into(0, 0, 0, 0)
    assert launches_of(sim, lambda: sim.export_view_into(0, 0, 0, 0)) == 3
    dn, ds = device(info.num_nodes * 64), device(info.num_samples * 16)
    assert launches_of(sim, lambda: sim.export_view_into(dn, info.num_nodes, ds, info.num_samples)) == 4


def test_query_region(sim, device):
    mn, mx = sim.box
    region = Region.box(mn - 1.0, mx + 1.0)
    info, _ = sim.query_region_into(region, None, 0, 0)
    assert info.num_samples > 0
    assert launches_of(sim, lambda: sim.query_region_into(region, None, 0, 0)) == 4
    ds = device(info.num_samples * 16)
    assert launches_of(sim, lambda: sim.query_region_into(region, None, ds, info.num_samples)) == 5

    def malformed():
        with pytest.raises(SimlodError):
            sim.query_region_into(Region.box(mx, mn), None, 0, 0)
    assert launches_of(sim, malformed) == 0


def test_partition_count_and_scatter(sim, device):
    n = 100_000
    pts, _, _ = data.uniform_cube(n, size=64.0, seed=9)
    src, dst = device(n * 16), device(n * 16)
    sim.memcpy_htod(src, pts.view(np.uint8))
    plan = sim.partition_plan(1, np.zeros(8, dtype=np.uint8), 1)
    assert launches_of(sim, lambda: sim.partition_count(src, n, plan)) == 2
    assert launches_of(sim, lambda: sim.partition_scatter(src, n, plan, [dst], [0])) == 1
    sim.synchronize()


def test_save_load_and_reset(sim, tmp_path):
    path = str(tmp_path / "tree.simlodoctree")
    samples = sim.export_octree_into(None, 0, 0, 0, 0)[0].num_samples
    windows = (samples + WINDOW_SAMPLES - 1) // WINDOW_SAMPLES
    assert windows >= 1
    assert launches_of(sim, lambda: sim.save_octree(path)) == 3 + windows
    assert launches_of(sim, lambda: sim.load_octree(path)) == 7 + windows
    assert launches_of(sim, sim.reset) == 1
