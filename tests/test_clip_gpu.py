"""GPU tests of the clip volumes (run with -m gpu on an H100): simlod_render_clip's frame and the clipped pick against the
restatement (clip_restatement) and against the unclipped frame. For every clip, octree, camera and setting the frame is
test_pick_gpu.check_frame's: the framebuffer holds frame_key of the pick (all 64 bits outside the EDL-covered tiles, the
depth word everywhere), and every picked sample is one the clip keeps. On orthographic cameras, where the restatement
projects exactly, the pick equals the restated clipped pick in every pixel, out-of-cube points included. Also: the
partition identity min(INSIDE, OUTSIDE) == unclipped, no-op clips, an unchanged cut, refusals, launch counts,
repeatability and untouched buffers."""
import hashlib

import numpy as np
import pytest

import clip_restatement as K
import oracle
import pick_restatement as P
from frame_restatement import covered
from simlod_b200 import SimlodError, api
from test_export_gpu import build, buffer_digests, terrain_ragged_stream, uniform_stream
from test_export_view_gpu import build_generated_terrain, view_cameras
from test_pick_gpu import PLAIN, SETTINGS, W, H, check_frame, make_sim

pytestmark = pytest.mark.gpu

CLIP_SETTINGS = ["default", "pointSize3", "pointSize5", "colorByNode", "hqs", "hqs_pointSize3"]
ATOMIC_MIN = ["default", "pointSize3", "pointSize5", "colorByNode"]
HI = np.uint64(32)


@pytest.fixture(scope="module")
def sim():
    s = make_sim()
    yield s
    s.close()


def clip_struct(regions, mode):
    c = api.SimlodClip(mode={"inside": K.INSIDE, "outside": K.OUTSIDE}[mode], num_regions=len(regions))
    for k, r in enumerate(regions):
        c.regions[k] = r
    return c


def clips(box_min, box_max):
    """A sub-box, a sphere, a 6-plane box turned 30 degrees about z, and a union of two boxes, all in the cube's middle."""
    mn, mx = np.asarray(box_min, np.float64), np.asarray(box_max, np.float64)
    c, e = (mn + mx) / 2, (mx - mn)
    sub = api.Region.box(c - e * [0.2, 0.15, 0.5], c + e * [0.1, 0.2, 0.5])
    sphere = api.Region.sphere(c, 0.2 * e[:2].max())
    t = np.radians(30.0)
    axes = [(np.cos(t), np.sin(t), 0.0), (-np.sin(t), np.cos(t), 0.0), (0.0, 0.0, 1.0)]
    half = [0.2 * e[0], 0.1 * e[1], 0.3 * e[2]]
    planes = []
    for a, h in zip(axes, half):
        a = np.asarray(a)
        planes += [list(a) + [h - a @ c], list(-a) + [h + a @ c]]           # -h <= a.(p - c) <= h
    two = [api.Region.box(c - e * [0.4, 0.4, 0.5], c - e * [0.1, 0.2, -0.5]), api.Region.box(c - e * [0.2, 0.0, 0.5], c + e * [0.3, 0.3, 0.5])]
    return {"subbox": [sub], "sphere": [sphere], "planes6": [api.Region.planes(planes)], "two_boxes": two}


def clipped_frame(sim, label, regions, mode):
    """check_frame under the clip; the picked samples are ones the clip keeps. Returns (framebuffer, index, export, u)."""
    sim.set_clip(regions, mode)
    try:
        index, e, u = check_frame(sim, label)
        fb = sim.framebuffer()
    finally:
        sim.set_clip(None)
    keep = K.keep_mask(clip_struct(regions, mode), e.samples)
    assert keep[index[index >= 0]].all(), "%s: a picked sample lies where the clip drops it" % label
    return fb, index, e, u


def check_partition(sim, label, full, inside, outside):
    """Per pixel min(INSIDE, OUTSIDE) == unclipped: in the depth word everywhere, in all 64 bits outside EDL's tiles."""
    both = np.minimum(inside, outside)
    bad = (both >> HI) != (full >> HI)
    bad |= (both != full) & ~covered(sim.width, sim.height, sim.launch_info()["render_blocks"])
    assert not bad.any(), "%s: partition identity fails in %d pixels, first at %s" % (label, int(bad.sum()), np.argwhere(bad)[:3].tolist())


def run_clips(sim, label, box, cams, settings, clip_names=None):
    regions = clips(*box)
    for cam, (view, proj) in cams:
        sim.set_camera(view, proj)
        for name in settings:
            sim.set_settings(**dict(PLAIN, **SETTINGS[name]))
            sim.render()
            full = sim.framebuffer()
            for cname in clip_names or regions:
                fbs = {mode: clipped_frame(sim, "%s/%s/%s/%s/%s" % (label, cam, name, cname, mode), regions[cname], mode)[0]
                       for mode in ("inside", "outside")}
                if name in ATOMIC_MIN:
                    check_partition(sim, "%s/%s/%s/%s" % (label, cam, name, cname), full, fbs["inside"], fbs["outside"])
    sim.set_settings(**PLAIN)


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged"])
def test_clipped_frames(sim, name):
    batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
    build(sim, batches, box)
    run_clips(sim, name, box, view_cameras(box[1], name.startswith("terrain"))[:2], CLIP_SETTINGS)


def test_clipped_frames_of_a_36m_terrain(sim):
    box_max = build_generated_terrain(sim)
    run_clips(sim, "terrain_36m", ((0.0, 0.0, 0.0), box_max), view_cameras(box_max, True)[:1], ["default", "pointSize3", "hqs"])


def test_reference_kernels_and_loaded_octrees(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box, reference=True)
    cams = view_cameras(box[1], True)[:1]
    run_clips(sim, "reference kernels' octree", box, cams, ["default", "colorByNode"], ["sphere", "two_boxes"])
    build(sim, batches, box)
    path = str(tmp_path / "tree.octree")
    sim.save_octree(path)
    other = make_sim()
    try:
        other.load_octree(path)
        run_clips(other, "loaded octree", box, cams, ["default", "hqs_pointSize3"], ["subbox", "planes6"])
    finally:
        other.close()


def ortho_grid(sim, extra=()):
    """Integer-grid points in [0, 256)^3 under an orthographic camera that shows [-64, 320)^2: w = 1 for every sample,
    so the restatement projects as the device does. `extra` points are inserted with them."""
    rng = np.random.default_rng(17)
    n = 1_000_000
    xyz = rng.integers(0, 256, size=(n, 3)).astype(np.float32)
    color = rng.integers(0, 4, size=n).astype(np.uint32) * 0x00010101
    if len(extra):
        xyz = np.concatenate([xyz, np.asarray(extra, np.float32)])
        color = np.concatenate([color, np.full(len(extra), 0x00FF00FF, np.uint32)])
    pts = api.make_points(xyz, color)
    build(sim, [pts[:n], pts[n:]], ((0.0, 0.0, 0.0), (256.0, 256.0, 256.0)))
    ortho = np.array([[1 / 192, 0, 0, -1 / 3], [0, 1 / 192, 0, -1 / 3], [0, 0, 1 / 256, -1], [0, 0, 0, 1]], dtype=np.float64)
    sim.set_camera(np.eye(4), ortho)


def test_orthographic_pick_is_the_restated_clipped_pick(sim):
    """Points below boxMin, on the max face and beyond it are drawn, or clipped, exactly as the restatement says."""
    extra = [(x, y, z) for x in (-1.0, -0.5, 256.0, 260.0, 300.0) for y in np.arange(10.0, 250.0, 20.0) for z in (0.0, 128.0, 256.0, 280.0)]
    ortho_grid(sim, extra)
    regions = {"slab": [api.Region.box((-40.0, -1.0, -1.0), (100.0, 300.0, 300.0))], "sphere": [api.Region.sphere((256.0, 128.0, 128.0), 90.0)],
               "face": [api.Region.planes([[1.0, 0.0, 0.0, -256.0]])]}
    special = 0
    for name in ("default", "pointSize3", "colorByNode"):
        sim.set_settings(**dict(PLAIN, **SETTINGS[name]))
        for cname, rs in regions.items():
            for mode in ("inside", "outside"):
                _, index, e, u = clipped_frame(sim, "orthographic/%s/%s/%s" % (name, cname, mode), rs, mode)
                want = K.clipped_pick(clip_struct(rs, mode), e.nodes, e.samples, u, W, H)
                assert np.array_equal(index, want), "%s/%s/%s: %d pixels differ" % (name, cname, mode, int((index != want).sum()))
                x = e.samples["x"][index[index >= 0]]
                special += int(((x < 0) | (x >= 256)).sum())
    sim.set_settings(**PLAIN)
    assert special > 0, "no out-of-cube point was drawn"


def test_no_op_clips_and_clearing(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    mn, mx = np.asarray(box[0], np.float64), np.asarray(box[1], np.float64)
    e = (mx - mn).max()
    enclosing = api.Region.box(mn - e, mx + e)
    far = api.Region.sphere(mx + 10 * e, 0.5 * e)
    for cam, (view, proj) in view_cameras(box[1], True)[:2]:
        sim.set_camera(view, proj)
        for name in ("default", "pointSize3", "hqs"):
            sim.set_settings(**dict(PLAIN, **SETTINGS[name]))
            sim.render()
            fb, surf = sim.framebuffer(), sim.surface()
            for regions, mode in (([enclosing], "inside"), ([far], "outside"), ([far, enclosing], "inside")):
                sim.set_clip(regions, mode)
                sim.render()
                assert (sim.framebuffer() == fb).all() and (sim.surface() == surf).all(), (cam, name, mode)
            sim.set_clip([enclosing], "outside")
            sim.render()
            got = sim.framebuffer()
            assert (got >> HI == np.uint64(0x7F800000)).all(), (cam, name)
            assert (got[~covered(W, H, sim.launch_info()["render_blocks"])] == np.uint64(P.CLEAR)).all(), (cam, name)
            index, info = sim.pick(device="cpu")
            assert (index == -1).all() and info.num_hits == 0
            sim.set_clip(None)
            sim.render()
            assert (sim.framebuffer() == fb).all() and (sim.surface() == surf).all(), (cam, name)
    sim.set_settings(**PLAIN)


def test_the_cut_and_the_buffers_do_not_change(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*view_cameras(box[1], True)[0][1])
    regions = clips(*box)["two_boxes"]
    sim.render()
    base = buffer_digests(sim)
    stats = bytes(sim.stats())[4:]                                        # all but frameID
    view = sim.export_view(device="cpu")
    for mode in ("inside", "outside"):
        sim.set_clip(regions, mode)
        try:
            before = sim.launch_info()["launches"]
            sim.render()
            assert sim.launch_info()["launches"] == before + 1
            fb, surf = sim.framebuffer(), sim.surface()
            digests = buffer_digests(sim)
            assert bytes(sim.stats())[4:] == stats, mode                  # numVisible* still count the cut
            for k in ("nodes", "heap", "momentary"):                     # nodes: the same visible / isLarge flags
                assert digests[k] == base[k], (mode, k)
            v = sim.export_view(device="cpu")
            assert v.nodes.tobytes() == view.nodes.tobytes() and v.samples.tobytes() == view.samples.tobytes(), mode
            for _ in range(2):
                sim.render()
                assert (sim.framebuffer() == fb).all() and (sim.surface() == surf).all(), mode
        finally:
            sim.set_clip(None)


def test_refusals_keep_the_previous_clip(sim):
    batches, box, _ = uniform_stream()
    build(sim, batches, box)
    sim.set_camera(*view_cameras(box[1], False)[0][1])
    regions = clips(*box)["sphere"]
    sim.set_clip(regions, "inside")
    sim.render()
    want = sim.framebuffer()
    bad_regions = [api.Region.sphere((0.0, 0.0, 0.0), -1.0), api.Region.box((1.0, 0.0, 0.0), (0.0, 1.0, 1.0)),
                   api.Region.box((float("nan"), 0.0, 0.0), (1.0, 1.0, 1.0)), api.SimlodRegion(kind=7)]
    p = api.Region.planes([[1.0, 0.0, 0.0, 0.0]])
    p.num_planes = 17
    bad_regions.append(p)
    calls = [lambda r=r: sim.set_clip([regions[0], r], "outside") for r in bad_regions]
    calls += [lambda: sim.set_clip([], "inside"), lambda: sim.set_clip(regions * 5, "inside")]
    for mode in (3, 0xFFFFFFFF):
        c = clip_struct(regions, "inside")
        c.mode = mode
        calls.append(lambda c=c: sim._check(sim._lib.simlod_set_clip(sim._ctx, api.C.byref(c))))
    for call in calls:
        before = sim.launch_info()["launches"]
        with pytest.raises(SimlodError) as err:
            call()
        assert err.value.code == -2 and sim.launch_info()["launches"] == before
        sim.render()
        assert (sim.framebuffer() == want).all()
    # the reference's render cubin has no simlod_render_clip: refused with the clip set, nothing launched
    sim.use_module(api.PROGRAM_RENDER, oracle.REF_CUBINS[1])
    try:
        before = sim.launch_info()["launches"]
        with pytest.raises(SimlodError) as err:
            sim.render()
        assert err.value.code == -4 and sim.launch_info()["launches"] == before
        sim.set_clip(None)
        sim.render()                                   # without a clip it renders as before
        assert sim.launch_info()["launches"] == before + 1
    finally:
        sim.use_module(api.PROGRAM_RENDER, None)
    sim.set_clip(regions, "inside")
    sim.render()
    assert (sim.framebuffer() == want).all()
    sim.set_clip(None)


def test_clipped_pick_protocol_and_repeatability(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    sim.set_camera(*view_cameras(box[1], True)[0][1])
    regions = clips(*box)["planes6"]
    sim.set_clip(regions, "outside")
    try:
        full, info = sim.pick(device="cpu")
        again, _ = sim.pick(device="cpu")
        assert full.tobytes() == again.tobytes()
        hit = np.argwhere(full >= 0)
        px = hit[:: max(1, len(hit) // 500)][:, ::-1]
        index, picked, _ = sim.pick(px, device="cpu", samples=True)
        assert (index == full[px[:, 1], px[:, 0]]).all()
        e = sim.export_view(device="cpu")
        assert picked.tobytes() == e.samples[index].tobytes()
        assert info.num_samples == e.info.num_samples
        digest = hashlib.sha256(sim.memcpy_dtoh(sim.buffers().nodes, sim.stats().numNodes * api.NODE_BYTES).tobytes()).hexdigest()
        sim.pick(device="cpu")
        assert hashlib.sha256(sim.memcpy_dtoh(sim.buffers().nodes, sim.stats().numNodes * api.NODE_BYTES).tobytes()).hexdigest() == digest
    finally:
        sim.set_clip(None)
