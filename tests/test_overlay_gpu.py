"""GPU tests of the bounding-box overlay (Uniforms::showBoundingBox; run with -m gpu on an H100): our kernel_render
against the reference's kernel_render on the same octree and uniforms. With showPoints=1 the comparison is the
reference_golden.frame digest (depth of every pixel, visible counts, flags, colours when no voxel is drawn); with
showPoints=0 no sample is drawn, so the raw u64 framebuffer and the RGBA8 surface are compared bit for bit on every case.
Reference digests are in tests/golden/overlay_reference.json, recorded again live with SIMLOD_RECORD_GOLDEN set. Above the
reference's line capacity (|D| > 10 416 drawn nodes) its frame is undefined; there the overlay is checked against the CPU
restatement (overlay_restatement.py) by coverage."""
import json
import os

import numpy as np
import pytest

import export_restatement as R
import export_view_restatement as V
import oracle
import overlay_restatement as O
import reference_golden as golden
from simlod_b200 import SimLOD, camera, data
from test_export_view_gpu import build_stream, nodes_image, view_cameras
from test_parity_gpu import VISIBLE, cameras

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
MIN_NODE_SIZES = (16.0, 64.0, 256.0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "overlay_reference.json")
# line pixels (symmetric difference) on which the device and the CPU restatement may disagree: a fraction of the union
# plus a fixed allowance. MUFU rcp / sqrt / rsqrt against correctly rounded ones move `steps` and the clipped endpoints in
# the last bits; the view's own frustum edges lie on the screen border, where such a bit decides whether a step is
# inside [-1, 1] (measured on an H100: at most 24 pixels, on the far camera, whose frames have few line pixels)
COVERAGE_TOLERANCE = 0.02
COVERAGE_ALLOWANCE = 64


@pytest.fixture(scope="module")
def sim():
    # 3 render blocks per SM: the grid the reference's own kernel_render gets from the occupancy query on sm_90
    s = SimLOD(W, H, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30, render_blocks_per_sm=3)
    yield s
    s.set_settings(showBoundingBox=0)
    s.close()


def reference_result(key, run):
    """The reference kernel's result for `key`: run() live (and recorded) with SIMLOD_RECORD_GOLDEN set, else the stored one."""
    if golden.RECORD:
        return golden.reference(key, run)
    with open(GOLDEN) as f:
        stored = json.load(f)
    assert key in stored, "no stored reference result for %r in %s" % (key, GOLDEN)
    return stored[key]


def frame_digest(sim):
    """The frame just rendered: golden.frame, with the raw framebuffer and surface whenever no sample is drawn."""
    st = sim.stats()
    fb = sim.framebuffer()
    nodes = sim.memcpy_dtoh(sim.buffers().nodes, st.numNodes * 152)
    voxels = st.numVisibleVoxels if sim.uniforms.showPoints else 0
    return golden.frame(fb, sim.surface(), [getattr(st, f) for f in VISIBLE], voxels, nodes)


def frames(sim, cases, reference=False):
    """{label: frame digest} of (label, settings, camera) cases; the reference's kernel_render when `reference`."""
    out = {}
    if reference:
        sim.use_module(1, oracle.REF_CUBINS[1])
    try:
        for label, settings, cam in cases:
            if cam is not None:
                sim.set_camera(*cam)
            sim.set_settings(**settings)
            sim.render()
            out[label] = frame_digest(sim)
    finally:
        if reference:
            sim.use_module(1, None)
    return out


def vs_reference(sim, key, cases, label):
    ours = frames(sim, cases)
    ref = reference_result(key, lambda: frames(sim, cases, reference=True))
    assert set(ours) == set(ref), label
    golden.assert_same(ours, ref, label)
    return ours


DEFAULTS = dict(showBoundingBox=1, showPoints=1, useHighQualityShading=0, pointSize=1, colorByNode=0, colorByLOD=0, minNodeSize=64.0)


def settings(**kw):
    return dict(DEFAULTS, **kw)


def drawn_lxyz(sim):
    """(level, X, Y, Z) of the nodes the last frame drew (its visible / isLarge flags)."""
    nb = nodes_image(sim)
    rec = np.frombuffer(np.ascontiguousarray(nb).tobytes(), dtype=R.NODE_DTYPE)
    d = V.drawn_from_flags(nb)
    return np.stack([rec[f][d].astype(np.int64) for f in ("level", "X", "Y", "Z")], axis=1)


def coverage_vs_restatement(sim, label):
    """The frame just rendered with showPoints=0 against the CPU restatement, by the pixels that carry a line."""
    got = O.coverage(sim.framebuffer())
    want = O.coverage(O.overlay_frame(O.uniforms_from_bytes(sim.uniforms_bytes()), drawn_lxyz(sim), W, H))
    union = int((got | want).sum())
    diff = int((got ^ want).sum())
    assert union > 0, label
    assert diff <= COVERAGE_TOLERANCE * union + COVERAGE_ALLOWANCE, "%s: %d of %d line pixels differ" % (label, diff, union)
    return diff, union


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged", "terrain_36m"])
def test_overlay_matches_the_reference(sim, name):
    box_max, terrain = build_stream(sim, name)
    cases = []
    for cam, view in view_cameras(box_max, terrain):
        for mns in MIN_NODE_SIZES:
            for hqs in (0, 1):
                for points in (1, 0):
                    cases.append(("%s/%g/hqs%d/points%d" % (cam, mns, hqs, points),
                                  settings(minNodeSize=mns, useHighQualityShading=hqs, showPoints=points), view))
    ours = vs_reference(sim, "overlay/" + name, cases, "overlay " + name)
    for label, d in ours.items():
        print("overlay %s %s: %d drawn nodes" % (name, label, d["visible"][0]))
    sim.set_settings(**settings(showBoundingBox=0))


def test_overlay_without_samples_covers_the_restatement(sim):
    box_max, terrain = build_stream(sim, "terrain_ragged")
    for cam, view in view_cameras(box_max, terrain):
        sim.set_camera(*view)
        for mns in MIN_NODE_SIZES:
            sim.set_settings(**settings(minNodeSize=mns, showPoints=0))
            sim.render()
            diff, union = coverage_vs_restatement(sim, "%s/%g" % (cam, mns))
            print("overlay coverage %s/%g: %d of %d line pixels differ from the CPU restatement" % (cam, mns, diff, union))
    sim.set_settings(**settings(showBoundingBox=0))


def test_frozen_visibility_draws_the_bound_frustum(sim):
    box_max, _ = build_stream(sim, "terrain_ragged")
    cams = dict(cameras(box_max, W, H))
    cases = []
    for hqs in (0, 1):
        for points in (1, 0):
            cases.append(("bind far/hqs%d/points%d" % (hqs, points), settings(useHighQualityShading=hqs, showPoints=points), cams["far"]))
            cases.append(("close, frozen at far/hqs%d/points%d" % (hqs, points), settings(useHighQualityShading=hqs, showPoints=points), None))
    ours = {}
    for label, s, cam in cases:          # the frozen frames depend on the camera bound before them: render in order
        ours.update(frames(sim, [(label, s, cam)]))
        if cam is not None:
            sim.set_camera(*cams["close"], update_visibility=False)
    order = list(cases)

    def run():
        out = {}
        for label, s, cam in order:
            out.update(frames(sim, [(label, s, cam)], reference=True))
            if cam is not None:
                sim.set_camera(*cams["close"], update_visibility=False)
        return out
    ref = reference_result("overlay/frozen", run)
    golden.assert_same(ours, ref, "frozen visibility")
    # the frustum of the far view is in the close frame: its lines differ from the close view's own
    sim.set_camera(*cams["close"], update_visibility=False)
    sim.set_settings(**settings(showPoints=0))
    sim.render()
    frozen = sim.framebuffer()
    coverage_vs_restatement(sim, "frozen")
    sim.set_camera(*cams["close"])
    sim.render()
    assert (sim.framebuffer() != frozen).any()
    sim.set_settings(**settings(showBoundingBox=0))


def test_nothing_drawn_gives_the_frustum_alone(sim):
    box_max, _ = build_stream(sim, "uniform_1m")
    cams = dict(cameras(box_max, W, H))
    cases = [("non-large root/points%d" % p, settings(minNodeSize=1e9, showPoints=p), cams["autofocus"]) for p in (1, 0)]
    ours = frames(sim, cases)
    assert all(d["visible"][0] == 0 for d in ours.values())
    coverage_vs_restatement(sim, "non-large root")
    sim.reset()
    cases_reset = [("after reset/points%d" % p, settings(showPoints=p), cams["close"]) for p in (1, 0)]
    ours_reset = frames(sim, cases_reset)
    assert all(d["visible"][0] == 0 for d in ours_reset.values())
    coverage_vs_restatement(sim, "after reset")
    ours.update(ours_reset)

    def run():
        build_stream(sim, "uniform_1m")
        out = frames(sim, cases, reference=True)
        sim.reset()
        out.update(frames(sim, cases_reset, reference=True))
        return out
    golden.assert_same(ours, reference_result("overlay/nothing_drawn", run), "nothing drawn")
    sim.set_settings(**settings(showBoundingBox=0))


def test_overlay_with_other_settings(sim):
    box_max, terrain = build_stream(sim, "terrain_ragged")
    view = camera.autofocus(box_max, W, H)
    cases = [("pointSize=2", settings(pointSize=2), view), ("colorByNode", settings(colorByNode=1), view),
             ("pointSize=2,hqs", settings(pointSize=2, useHighQualityShading=1), view),
             ("colorByNode,hqs", settings(colorByNode=1, useHighQualityShading=1), view)]
    vs_reference(sim, "overlay/settings", cases, "other settings")
    sim.set_settings(**settings(showBoundingBox=0))


CONFIG3_BATCHES = 350
CONFIG5_MIN_NODE_SIZES = (1.0, 2.0, 4.0, 8.0, 16.0, 32.0, 64.0)


def config5_cameras():
    """bench.py's config-5 cameras: autofocus at four yaws, Morro bird and close."""
    cams = [("autofocus+%d" % k, camera.autofocus(data.TERRAIN_EXTENT, W, H, yaw_offset=k * np.pi / 2)) for k in range(4)]
    return cams + [("morro_bird", camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD)),
                   ("morro_close", camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE))]


def test_largest_cut_and_above_the_reference_capacity():
    """The full-size config-3 octree (350 M terrain points generated on the device): the largest |D| <= 10 416 over the
    config-5 cameras and minNodeSize 1-64 against the reference; the largest |D| above it (where the reference overruns its
    line list and its frame is undefined) rendered twice, identical, and covered like the CPU restatement."""
    n = CONFIG3_BATCHES * 1_000_000
    big = SimLOD(W, H, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=24 << 30, render_blocks_per_sm=3)
    try:
        dptr = big.device_alloc(n * 16)
        try:
            big.generate(big.GEN_TERRAIN, dptr, n, 0, n, 7)
            big.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
            big.reset()
            big.insert_device(dptr, n)
        finally:
            big.device_free(dptr)
        st = big.stats()
        assert st.dbg == 0 and st.numPointsProcessed == n
        cams = dict(config5_cameras())
        sizes = []
        for cam, view in cams.items():
            big.set_camera(*view)
            for mns in CONFIG5_MIN_NODE_SIZES:
                big.set_settings(**settings(minNodeSize=mns, showBoundingBox=0))
                big.render()
                sizes.append((big.stats().numVisibleNodes, cam, mns))
        for d, cam, mns in sorted(sizes):
            print("overlay cut, config 3 (%d nodes): camera %s minNodeSize %g: %d drawn nodes" % (st.numNodes, cam, mns, d))
        below = max(s for s in sizes if s[0] <= O.REFERENCE_CAPACITY_NODES)
        above = max(sizes)
        print("largest |D| <= %d: %d (%s, minNodeSize %g); largest |D|: %d (%s, minNodeSize %g)"
              % ((O.REFERENCE_CAPACITY_NODES,) + below + above))
        d, cam, mns = below
        cases = [("largest/points%d/hqs%d" % (p, h), settings(minNodeSize=mns, showPoints=p, useHighQualityShading=h), cams[cam])
                 for p in (1, 0) for h in (0, 1)]
        ours = vs_reference(big, "overlay/config3_largest/%s/%g" % (cam, mns), cases, "largest |D| within the reference's capacity")
        assert all(v["visible"][0] == d for v in ours.values())
        if above[0] <= O.REFERENCE_CAPACITY_NODES:
            pytest.skip("no case of the config-3 octree reached above %d drawn nodes (largest %d)" % (O.REFERENCE_CAPACITY_NODES, above[0]))
        d, cam, mns = above
        big.set_camera(*cams[cam])
        for points in (0, 1):
            big.set_settings(**settings(minNodeSize=mns, showPoints=points))
            big.render()
            a, a_surface = big.framebuffer(), big.surface()
            big.render()
            assert (big.framebuffer() == a).all() and (big.surface() == a_surface).all()
            assert big.stats().numVisibleNodes == d
            if points == 0:
                diff, union = coverage_vs_restatement(big, "above capacity")
                print("above capacity: %d drawn nodes (%s, minNodeSize %g), %d of %d line pixels differ from the CPU restatement"
                      % (d, cam, mns, diff, union))
    finally:
        big.close()


def cache_counters(sim):
    c = sim.memcpy_dtoh(sim.buffers().renderbuffer + 40, 8).view(np.uint32)
    return int(c[0]), int(c[1])


def test_overlay_leaves_nothing_behind(sim):
    box_max, _ = build_stream(sim, "terrain_ragged")
    before = oracle.canon_from_image(*sim.download_octree())
    sim.set_camera(*camera.autofocus(box_max, W, H))
    after_overlay = {}
    # minNodeSize 0.5: every visible node is large, so the cut is the visible leaves and no voxel is drawn. A voxel's colour
    # is a race in the builders, so only frames without voxels are the same in a context that built the octree again.
    for hqs in (0, 1):
        sim.set_settings(**settings(showBoundingBox=0, useHighQualityShading=hqs, minNodeSize=0.5))
        sim.render()
        plain, plain_surface, plain_st = sim.framebuffer(), sim.surface(), sim.stats()
        assert plain_st.numVisibleVoxels == 0 and plain_st.numVisiblePoints > 0
        sim.set_settings(showBoundingBox=1)
        sim.render()
        on, on_st = sim.framebuffer(), sim.stats()
        assert (on != plain).any()
        assert [getattr(on_st, f) for f in VISIBLE] == [getattr(plain_st, f) for f in VISIBLE]
        sim.set_settings(showBoundingBox=0)
        sim.render()
        hits, walks = cache_counters(sim)
        assert hits > 0 and walks == 0, (hits, walks)
        assert (sim.framebuffer() == plain).all() and (sim.surface() == plain_surface).all()
        assert [getattr(sim.stats(), f) for f in VISIBLE] == [getattr(plain_st, f) for f in VISIBLE]
        after_overlay[hqs] = sim.framebuffer(), sim.surface()
    after = oracle.canon_from_image(*sim.download_octree())
    assert not oracle.compare_canon(before, after)
    sim.set_settings(**settings(showBoundingBox=0))
    # the same octree and camera in a context that never had the overlay on: the same frames
    fresh = SimLOD(W, H, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=2 << 30, render_blocks_per_sm=3)
    try:
        build_stream(fresh, "terrain_ragged")
        fresh.set_camera(*camera.autofocus(box_max, W, H))
        for hqs in (0, 1):
            fresh.set_settings(**settings(showBoundingBox=0, useHighQualityShading=hqs, minNodeSize=0.5))
            fresh.render()
            fb, surface = after_overlay[hqs]
            assert (fresh.framebuffer() == fb).all() and (fresh.surface() == surface).all(), hqs
    finally:
        fresh.close()
