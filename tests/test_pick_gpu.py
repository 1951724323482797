"""GPU tests of the pick (run with -m gpu on an H100): simlod_pick against the frame kernel_render draws for the same
uniforms. Where the pick names sample i of the view export, the framebuffer holds that sample's key depth << 32 | colour
(pick_restatement.frame_key, exact on any camera since the depth is w itself), and the clear value where the pick is -1.
Eye-dome lighting rewrites the colour word of the pixels in the 16x16 tiles it covers, so there only the depth word is
compared; every other pixel is compared in all 64 bits (with HQS, the depth word everywhere). The tie rule is pinned to
the restatement on an orthographic camera, where w = 1 and MUFU.RCP is exact; perspective cameras are compared within
a pixel. Also: pixel lists, samples, the torch path, repeatability, no writes into the context, the overlay and
showPoints, the protocol with guard bytes, a frozen visibility transform, a second resolution, the reference kernels'
octree and a loaded octree."""
import hashlib

import numpy as np
import pytest

import oracle
import pick_restatement as P
from frame_restatement import covered
from simlod_b200 import SimLOD, SimlodError, api, camera
from test_export_gpu import build, buffer_digests, terrain_ragged_stream, uniform_stream
from test_export_view_gpu import build_generated_terrain, view_cameras

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
SETTINGS = {
    "default": {},
    "pointSize2": {"pointSize": 2}, "pointSize3": {"pointSize": 3}, "pointSize5": {"pointSize": 5},
    "colorByLOD": {"colorByLOD": 1}, "colorByNode": {"colorByNode": 1},
    "hqs": {"useHighQualityShading": 1}, "hqs_pointSize3": {"useHighQualityShading": 1, "pointSize": 3},
}
PLAIN = {"pointSize": 1, "colorByLOD": 0, "colorByNode": 0, "useHighQualityShading": 0, "showBoundingBox": 0, "showPoints": 1}


def make_sim(w=W, h=H):
    # 3 render blocks per SM, as in the view export's tests
    return SimLOD(w, h, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=12 << 30, render_blocks_per_sm=3)


@pytest.fixture(scope="module")
def sim():
    s = make_sim()
    yield s
    s.close()


def check_frame(sim, label):
    """render(), then the whole-frame pick against the framebuffer. Returns (index, view export, uniforms)."""
    sim.render()
    fb = sim.framebuffer()
    index, info = sim.pick(device="cpu")
    e = sim.export_view(device="cpu")
    u = P.uniforms_from_bytes(sim.uniforms_bytes())
    assert index.shape == (sim.height, sim.width) and index.dtype == np.int64, label
    assert info.num_samples == e.info.num_samples and info.num_nodes == e.info.num_nodes, label
    assert info.num_pixels == sim.width * sim.height and info.num_hits == int((index >= 0).sum()), label
    assert index.max() < e.info.num_samples, label
    want = P.frame_key(e.nodes, e.samples, u, index)
    hi = np.uint64(32)
    bad = (fb >> hi) != (want >> hi)
    if not u["useHighQualityShading"]:
        bad |= (fb != want) & ~covered(sim.width, sim.height, sim.launch_info()["render_blocks"])
    assert not bad.any(), "%s: %d pixels differ from the frame, first at %s" % (label, int(bad.sum()), np.argwhere(bad)[:3].tolist())
    return index, e, u


def run_settings(sim, label, settings):
    hits = []
    for name in settings:
        sim.set_settings(**dict(PLAIN, **SETTINGS[name]))
        index, _, _ = check_frame(sim, "%s/%s" % (label, name))
        hits.append(int((index >= 0).sum()))
    sim.set_settings(**PLAIN)
    return hits


@pytest.mark.parametrize("name", ["uniform_1m", "terrain_ragged", "terrain_36m"])
def test_pick_is_the_frames_sample(sim, name):
    if name == "terrain_36m":
        box_max, terrain = build_generated_terrain(sim), True
        settings = ["default", "pointSize3", "colorByNode", "hqs"]
    else:
        batches, box, _ = {"uniform_1m": uniform_stream, "terrain_ragged": terrain_ragged_stream}[name]()
        build(sim, batches, box)
        box_max, terrain = box[1], name.startswith("terrain")
        settings = list(SETTINGS)
    for cam, (view, proj) in view_cameras(box_max, terrain):
        sim.set_camera(view, proj)
        hits = run_settings(sim, "%s/%s" % (name, cam), settings)
        print("pick %s/%s: hits %s" % (name, cam, hits))


def test_reference_kernels_octree(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box, reference=True)
    for cam, (view, proj) in view_cameras(box[1], True):
        sim.set_camera(view, proj)
        run_settings(sim, "reference kernels' octree/%s" % cam, ["default", "pointSize3", "colorByNode"])


def test_loaded_octree(sim, tmp_path):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    path = str(tmp_path / "tree.octree")
    sim.save_octree(path)
    other = make_sim()
    try:
        other.load_octree(path)
        for cam, (view, proj) in view_cameras(box[1], True):
            other.set_camera(view, proj)
            run_settings(other, "loaded octree/%s" % cam, ["default", "colorByLOD"])
    finally:
        other.close()


def test_frozen_visibility_and_a_second_resolution(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cams = dict(view_cameras(box[1], True))
    sim.set_camera(*cams["far"])
    sim.set_camera(*cams["close"], update_visibility=False)
    run_settings(sim, "close camera, frozen at far", ["default", "pointSize3"])
    sim.set_camera(*cams["close"])
    small = make_sim(1001, 563)                   # not a multiple of 16: EDL covers whole tiles only
    try:
        small.set_box(*box)
        small.reset()
        small.insert_batches(batches)
        for cam, (view, proj) in view_cameras(box[1], True):
            small.set_camera(view, proj)
            run_settings(small, "1001x563/%s" % cam, ["default", "pointSize5", "hqs"])
    finally:
        small.close()


def test_pixel_lists_samples_and_repeatability(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cams = dict(view_cameras(box[1], True))
    sim.set_camera(*cams["autofocus"])
    full, info = sim.pick(device="cpu")
    again, info2 = sim.pick(device="cpu")
    assert full.tobytes() == again.tobytes() and bytes(info)[:24] == bytes(info2)[:24]
    e = sim.export_view(device="cpu")
    rng = np.random.default_rng(5)
    hit = np.argwhere(full >= 0)
    px = np.concatenate([hit[rng.integers(0, len(hit), 3000)][:, ::-1], np.stack([rng.integers(0, W, 1000), rng.integers(0, H, 1000)], 1),
                         [[0, 0], [W - 1, H - 1]]])
    index, picked, pinfo = sim.pick(px, device="cpu", samples=True)
    assert index.shape == (len(px),) and (index == full[px[:, 1], px[:, 0]]).all()
    assert pinfo.num_hits == int((index >= 0).sum()) and pinfo.num_pixels == len(px)
    assert picked[index >= 0].tobytes() == e.samples[index[index >= 0]].tobytes()
    assert (picked[index < 0].view(np.uint32) == 0).all()
    one, _ = sim.pick([[int(hit[0][1]), int(hit[0][0])]], device="cpu")
    assert one[0] == full[hit[0][0], hit[0][1]]
    # the whole frame with samples, and the torch path
    _, whole, _ = sim.pick(device="cpu", samples=True)
    assert whole.shape == (H, W) and whole[full >= 0].tobytes() == e.samples[full[full >= 0]].tobytes()
    torch = pytest.importorskip("torch")
    ti, ts, _ = sim.pick(torch.from_numpy(px), samples=True)
    assert ti.is_cuda and ti.dtype == torch.int64 and (ti.cpu().numpy() == index).all()
    assert ts.shape == (len(px), 4) and ts.cpu().numpy().tobytes() == picked.tobytes()
    tf, _ = sim.pick()
    assert tuple(tf.shape) == (H, W) and (tf.cpu().numpy() == full).all()


def test_writes_nothing_and_ignores_the_overlay(sim):
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    cams = dict(view_cameras(box[1], True))
    sim.set_camera(*cams["close"])
    sim.render()
    b = sim.buffers()
    ring = lambda: hashlib.sha256(sim.memcpy_dtoh(b.ring, b.ring_bytes).tobytes()).hexdigest()   # noqa: E731
    sim.set_camera(*cams["autofocus"])
    before, ring_before = buffer_digests(sim), ring()
    plain, _ = sim.pick(device="cpu")
    assert buffer_digests(sim) == before and ring() == ring_before
    # the next frame is the frame without the pick
    sim.render(); fb_a, surf_a = sim.framebuffer(), sim.surface()
    sim.pick(device="cpu")
    sim.render(); fb_b, surf_b = sim.framebuffer(), sim.surface()
    assert (fb_a == fb_b).all() and (surf_a == surf_b).all()
    sim.set_settings(showBoundingBox=1)
    try:
        boxed, _ = sim.pick(device="cpu")
        assert boxed.tobytes() == plain.tobytes()
    finally:
        sim.set_settings(showBoundingBox=0)
    sim.set_settings(showPoints=0)
    try:
        off, info = sim.pick(device="cpu")
        assert (off == -1).all() and info.num_hits == 0
        sim.render()
        assert (sim.framebuffer() >> np.uint64(32) == np.uint64(0x7F800000)).all()
    finally:
        sim.set_settings(showPoints=1)


def test_protocol(sim):
    batches, box, _ = uniform_stream()
    build(sim, batches, box)
    sim.set_camera(*camera.autofocus(box[1], W, H))
    full, info = sim.pick(device="cpu")
    n = 4
    guard = 4096
    di, ds = sim.device_alloc(n * 8 + 2 * guard), sim.device_alloc(n * 16 + 2 * guard)
    try:
        pat_i, pat_s = np.full(n * 8 + 2 * guard, 0xA5, np.uint8), np.full(n * 16 + 2 * guard, 0x5A, np.uint8)
        sim.memcpy_htod(di, pat_i)
        sim.memcpy_htod(ds, pat_s)
        good = [[10, 10], [W // 2, H // 2], [W - 1, 0], [0, H - 1]]
        for pixels, dsts in (([[W, 0]], (di + guard, ds + guard)), ([[0, H]], (di + guard, ds + guard)),
                             ([[-1, 0]], (di + guard, ds + guard)), (np.zeros((0, 2), np.int64), (di + guard, ds + guard)),
                             (np.zeros((W * H + 1, 2), np.int64), (di + guard, ds + guard)),
                             (good, (di + guard + 4, ds + guard)), (good, (di + guard, ds + guard + 8))):
            with pytest.raises(SimlodError) as err:
                sim.pick_into(pixels, *dsts)
            assert err.value.code == -2
            assert (sim.memcpy_dtoh(di, len(pat_i)) == pat_i).all() and (sim.memcpy_dtoh(ds, len(pat_s)) == pat_s).all()
        with pytest.raises(SimlodError):
            sim._check(sim._lib.simlod_pick(sim._ctx, None, 3, 0, 0, api.C.byref(api.SimlodPickInfo()), None))
        only, _ = sim.pick_into(good, 0, 0)                 # info only
        assert only.num_samples == info.num_samples and only.num_pixels == n
        got, _ = sim.pick_into(good, di + guard, ds + guard)
        gi, gs = sim.memcpy_dtoh(di, len(pat_i)), sim.memcpy_dtoh(ds, len(pat_s))
        assert (gi[:guard] == 0xA5).all() and (gi[guard + n * 8:] == 0xA5).all()
        assert (gs[:guard] == 0x5A).all() and (gs[guard + n * 16:] == 0x5A).all()
        want = np.array([full[y, x] for x, y in good])
        assert (gi[guard:guard + n * 8].view(np.int64) == want).all() and got.num_hits == int((want >= 0).sum())
    finally:
        sim.device_free(di)
        sim.device_free(ds)


def test_orthographic_grid_pins_the_tie_rule(sim):
    """Integer-grid points under an orthographic camera: w = 1 for every sample, so every depth ties and MUFU.RCP(1) is
    exact; the restatement must equal the device pick in every pixel, ties on the colour and the index included."""
    rng = np.random.default_rng(11)
    n = 1_000_000
    xyz = rng.integers(0, 256, size=(n, 3)).astype(np.float32)
    color = rng.integers(0, 4, size=n).astype(np.uint32) * 0x00010101         # four colours: many ties on the key
    pts = api.make_points(xyz, color)
    build(sim, [pts], ((0.0, 0.0, 0.0), (256.0, 256.0, 256.0)))
    ortho = np.array([[1 / 128, 0, 0, -1], [0, 1 / 128, 0, -1], [0, 0, 1 / 128, -1], [0, 0, 0, 1]], dtype=np.float64)
    sim.set_camera(np.eye(4), ortho)
    for name in ("default", "pointSize3", "colorByNode", "colorByLOD"):
        sim.set_settings(**dict(PLAIN, **SETTINGS[name]))
        index, e, u = check_frame(sim, "orthographic/%s" % name)
        want = P.pick_frame(e.nodes, e.samples, u, W, H)
        assert np.array_equal(index, want), "orthographic/%s: %d pixels differ" % (name, int((index != want).sum()))
        assert (index >= 0).sum() >= 255 * 255             # every grid column and row but 0 lands inside
    sim.set_settings(**PLAIN)


def test_perspective_within_a_pixel(sim):
    """Under perspective the restatement's 1 / w is not the device's MUFU.RCP: each picked sample lies within a pixel of
    the pixel that picked it, and exactly on it for all but 0.1 % of the hits."""
    batches, box, _ = terrain_ragged_stream()
    build(sim, batches, box)
    for cam, (view, proj) in view_cameras(box[1], True):
        sim.set_camera(view, proj)
        index, e, u = check_frame(sim, "perspective/%s" % cam)
        y, x = np.nonzero(index >= 0)
        sx, sy, _, _, _ = P.sample_keys(e.nodes, e.samples, u, W, H)
        dx, dy = sx[index[y, x]] - x, sy[index[y, x]] - y
        assert (np.abs(dx) <= 1).all() and (np.abs(dy) <= 1).all(), cam
        off = float(((dx != 0) | (dy != 0)).mean()) if len(x) else 0.0
        print("perspective %s: %d hits, %.2e off by one pixel" % (cam, len(x), off))
        assert off <= 1e-3, cam
