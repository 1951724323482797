"""BASELINE.json's full-size configurations on the GPU (streams generated on the device, csrc/gen.cu), ours against the
reference's own kernels (oracle/_ref/*.cubin, stored as digests in tests/golden/reference.json by
tests/reference_golden.py) through the same C ABI, same buffers, same input:
  config 2   36 M-point terrain stream: canonical octree (every node's counters, sorted point / voxel multisets) + Stats
  config 3   350 M-point terrain stream: the deterministic Stats fields, then
  config 5   kernel_render on that octree, 6 cameras x {atomicMin, HQS}: depth of every pixel identical, and
             the raw u64 framebuffer and surface for frames that draw no voxel
  config 4   one GPU's share of the shell stream (250 M points, cube 4096^3): the deterministic Stats fields
"""
import numpy as np
import pytest

import oracle
import reference_golden as golden
from simlod_b200 import SimLOD, camera, data

pytestmark = pytest.mark.gpu
BATCH = 1_000_000


def build(sim, dptr, n, box, reference):
    for p in (0, 2):
        sim.use_module(p, oracle.REF_CUBINS[p] if reference else None)
    sim.set_box(*box)
    sim.reset()
    sim.insert_device(dptr, n)
    st = sim.stats()
    for p in (0, 2):
        sim.use_module(p, None)
    assert st.numPointsProcessed == n and st.numPoints == n, (st.numPoints, st.numPointsProcessed, st.dbg)
    return st


def test_config2_36m_stream_canonical_octree_vs_reference_kernels():
    n = 36 * BATCH
    sim = SimLOD(1920, 1080, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=6 << 30, render_blocks_per_sm=3)
    try:
        dptr = sim.device_alloc(n * 16)
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        box = ((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        st = build(sim, dptr, n, box, False)
        assert st.dbg == 0
        cn = oracle.canon_from_image(*sim.download_octree())

        def run():
            st_r = build(sim, dptr, n, box, True)
            return golden.octree(st_r, oracle.canon_from_image(*sim.download_octree()))
        golden.assert_same(golden.octree(st, cn), golden.reference("config2_36m", run), "36M: ours vs reference kernels")
    finally:
        sim.close()


def cameras(box_max, w, h):
    cams = [camera.autofocus(box_max, w, h, yaw_offset=k * np.pi / 2) for k in range(4)]
    cams += [camera.orbit_camera(width=w, height=h, **camera.MORRO_BIRD), camera.orbit_camera(width=w, height=h, **camera.MORRO_CLOSE)]
    return cams


def test_config3_350m_stats_and_config5_twelve_frames_vs_reference_kernels():
    n = 350 * BATCH
    # 3 render blocks per SM = the grid the reference's render kernel gets from the occupancy query (EDL tile coverage depends on it)
    sim = SimLOD(1920, 1080, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=24 << 30, render_blocks_per_sm=3)
    try:
        dptr = sim.device_alloc(n * 16)
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
        box = ((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        ref = golden.reference("config3_350m", lambda: golden.stats(build(sim, dptr, n, box, True)))
        st = build(sim, dptr, n, box, False)
        assert st.dbg == 0
        golden.assert_same(golden.stats(st), ref, "350M: ours vs reference kernels")
        # config 5: both rasterisers on the octree OUR builder just made
        for hqs in (0, 1):
            sim.set_settings(useHighQualityShading=hqs, pointSize=1)
            for k, (view, proj) in enumerate(cameras(data.TERRAIN_EXTENT, sim.width, sim.height)):
                sim.set_camera(view, proj)

                def frame():
                    sim.render()
                    s = sim.stats()
                    return golden.frame(sim.framebuffer(), sim.surface(), (s.numVisibleNodes, s.numVisiblePoints, s.numVisibleVoxels),
                                        s.numVisibleVoxels)

                def run():
                    sim.use_module(1, oracle.REF_CUBINS[1])
                    try:
                        return frame()
                    finally:
                        sim.use_module(1, None)
                ours = frame()
                assert ours["visible"][0] > 0
                golden.assert_same(ours, golden.reference("config5_350m/camera%d/hqs%d" % (k, hqs), run), "camera %d hqs %d" % (k, hqs))
        sim.set_settings(useHighQualityShading=0)
    finally:
        sim.close()


def test_config4_one_gpu_share_of_the_shell_stream_vs_reference_kernels():
    n = 250 * BATCH
    sim = SimLOD(640, 360, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=24 << 30)
    try:
        dptr = sim.device_alloc(n * 16)
        sim.generate(sim.GEN_SHELL, dptr, n, 0, n, 1234)
        box = ((0.0, 0.0, 0.0), (data.SHELL_CUBE,) * 3)
        ref = golden.reference("config4_250m_shell", lambda: golden.stats(build(sim, dptr, n, box, True)))
        st = build(sim, dptr, n, box, False)
        assert st.dbg == 0
        golden.assert_same(golden.stats(st), ref, "shell 250M: ours vs reference kernels")
    finally:
        sim.close()
