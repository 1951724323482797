"""CPU tests of the bounding-box overlay: kernel_render's resources with the overlay compiled in, and the CPU restatement
of the reference's line list and line rasteriser (overlay_restatement.py) on hand-made uniforms, including degenerate
lines."""
import os
import re
import subprocess

import numpy as np
import pytest

import overlay_restatement as O
from simlod_b200 import build as B

# kernel_render without the overlay: 64 registers (4 blocks of 256 threads per SM), 88 B stack frame, 100 B of
# spill stores, 212 B of spill loads
MAX_REGISTERS, MAX_STACK, MAX_SPILL_STORES, MAX_SPILL_LOADS = 64, 88, 100, 212


def test_kernel_render_resources(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "render.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("render", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "render.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    m = re.search(r"Function properties for kernel_render\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                  r".*Used (\d+) registers", res.stdout)
    assert m, res.stdout
    stack, stores, loads, regs = (int(v) for v in m.groups())
    assert regs <= MAX_REGISTERS and stack <= MAX_STACK and stores <= MAX_SPILL_STORES and loads <= MAX_SPILL_LOADS, res.stdout
    assert "overlayFrame" in res.stdout, "the frame with the overlay ends in a function of its own, outside kernel_render's register allocation"


# ---- the restatement -------------------------------------------------------------------------------------------------

def uniforms(transform=None, inverse=None, box=(0.0, 8.0), width=64, height=64):
    eye = np.eye(4, dtype=np.float32)
    return {"width": float(width), "height": float(height),
            "transform": np.asarray(eye if transform is None else transform, np.float32),
            "transformInv_updateBound": np.asarray(eye if inverse is None else inverse, np.float32),
            "boxMin": np.full(3, box[0], np.float32), "boxMax": np.full(3, box[1], np.float32), "showBoundingBox": 1}


def test_capacity_of_the_reference_list():
    assert O.REFERENCE_CAPACITY_NODES == 10416
    assert 2 * O.reference_line_count(10416) <= O.REFERENCE_VERTEX_CAPACITY < 2 * O.reference_line_count(10417)
    assert O.overlay_line_count(10417) == 8 + 12 * 10417


def test_line_list_counts_and_colours():
    u = uniforms()
    lxyz = [(0, 0, 0, 0), (1, 1, 0, 1), (3, 7, 2, 5)]
    s, e, c = O.line_list(u, lxyz)
    assert len(s) == len(e) == len(c) == O.overlay_line_count(3)
    assert (c[:8] == O.FRUSTUM_COLOR).all() and (c[8:] == O.BOX_COLOR).all()
    s0, e0, c0 = O.line_list(u, np.zeros((0, 4)))
    assert len(s0) == 8 and (c0 == O.FRUSTUM_COLOR).all()


def test_frustum_lines_are_the_ndc_corners_through_the_bound_inverse():
    # identity inverse: the corners themselves, near plane z = -1, far plane z = 0.99995
    s, e = O.frustum_lines(uniforms())
    f = np.float32(0.99995)
    want_s = [(1, 1, -1), (1, -1, -1), (-1, 1, -1), (-1, -1, -1), (-1, -1, f), (-1, 1, f), (-1, -1, f), (1, -1, f)]
    want_e = [(1, 1, f), (1, -1, f), (-1, 1, f), (-1, -1, f), (1, -1, f), (1, 1, f), (-1, 1, f), (1, 1, f)]
    assert (s == np.array(want_s, np.float32)).all() and (e == np.array(want_e, np.float32)).all()
    # a scaled and translated inverse: x, y, z map through the rows, divided by w
    inv = np.array([[2, 0, 0, 1], [0, 3, 0, 0], [0, 0, 1, 5], [0, 0, 0, 2]], np.float32)
    s, _ = O.frustum_lines(uniforms(inverse=inv))
    assert tuple(s[0]) == (1.5, 1.5, 2.0)


def test_box_edges_of_a_node():
    u = uniforms(box=(0.0, 8.0))
    s, e = O.box_lines(u, [(1, 1, 0, 1)])           # level 1: edge 4, cell (1, 0, 1) = [4, 8] x [0, 4] x [4, 8]
    mn, mx = np.array([4, 0, 4], np.float32), np.array([8, 4, 8], np.float32)

    def corner(c):
        return tuple(np.where([c & 4, c & 2, c & 1], mx, mn))
    for k in range(12):
        assert tuple(s[k]) == corner(O.EDGE_FROM[k]) and tuple(e[k]) == corner(O.EDGE_TO[k]), k
    # the 12 edges of a cube, each once
    edges = {frozenset((a, b)) for a, b in zip(O.EDGE_FROM, O.EDGE_TO)}
    assert len(edges) == 12 and all(bin(a ^ b).count("1") == 1 for a, b in (tuple(x) for x in edges))


def covered(u, starts, ends, width=64, height=64):
    pixel, value = O.rasterize(u, np.array(starts, np.float32), np.array(ends, np.float32), np.full(len(starts), O.BOX_COLOR, np.uint64), width, height)
    fb = np.full(width * height, (O.INF_DEPTH << np.uint64(32)) | np.uint64(0x00332211), np.uint64)
    np.minimum.at(fb, pixel, value)
    return O.coverage(fb).reshape(height, width), fb


def test_a_horizontal_line_in_ndc():
    # identity transform: NDC = world, w = 1. x from -0.5 to 0.5 is 32 pixels: 33 steps u = 0, 1/32, ..., 1
    cov, fb = covered(uniforms(), [(-0.5, -0.5, 0.0)], [(0.5, -0.5, 0.0)])
    assert cov.sum() == 33 and cov[16, 16:49].all()
    assert ((fb.reshape(64, 64)[16, 16:49] >> np.uint64(32)) == np.uint64(0x3F800000)).all()      # depth w = 1.0


def test_zero_length_projected_line_draws_its_first_step():
    # along the view axis: both ends project to the same pixel, steps = 0, stepSize = inf: the u = 0 step only
    pixel, _ = O.rasterize(uniforms(), np.array([(0.25, 0.25, -0.5)], np.float32), np.array([(0.25, 0.25, 0.5)], np.float32),
                           np.array([O.BOX_COLOR], np.uint64), 64, 64)
    assert len(pixel) == 1 and pixel[0] == 40 + 64 * 40


def test_endpoint_on_a_plane_is_not_clipped():
    # x = 1 lies on the right plane (distance 0, not < 0): kept, the pixel clamps to the last column
    cov, _ = covered(uniforms(), [(1.0, -0.5, 0.0)], [(1.0, 0.5, 0.0)])
    assert cov[:, 63].sum() == 33 and cov.sum() == 33


def test_clipped_endpoint_moves_onto_the_frustum():
    # from inside to x = 3: the end moves back along the line to x = 1 (the right plane)
    cov, _ = covered(uniforms(), [(0.0, 0.0, 0.0)], [(3.0, 0.0, 0.0)])
    assert cov[32, 32:64].all() and cov.sum() == cov[32].sum()


def test_fully_clipped_line_draws_nothing():
    # both ends outside and no plane ahead of them: farthest = -Infinity, the endpoints and depths are NaN; the steps
    # land on pixel 0 with NaN depth bits, which never win against the cleared +Infinity
    cov, fb = covered(uniforms(), [(2.0, 2.0, 0.0)], [(3.0, 3.0, 0.0)])
    assert cov.sum() == 0


def test_nothing_drawn_is_the_frustum_alone():
    t = np.array([[1.5, 0, 0, 0], [0, 1.5, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
    u = uniforms(transform=t, inverse=np.linalg.inv(t.astype(np.float64)).astype(np.float32))
    frame = O.overlay_frame(u, np.zeros((0, 4)), 64, 64)
    s, e = O.frustum_lines(u)
    pixel, _ = O.rasterize(u, s, e, np.full(8, O.FRUSTUM_COLOR, np.uint64), 64, 64)
    cov = O.coverage(frame)
    assert cov.sum() > 0 and set(np.nonzero(cov)[0]) == set(pixel.tolist())
    assert set((frame[cov] & np.uint64(0xFFFFFFFF)).tolist()) == {O.FRUSTUM_COLOR}


def test_nearer_line_wins():
    # two lines over the same pixels: the smaller depth word takes them, whatever the order
    u = uniforms()
    t = np.diag(np.array([1, 1, 1, 1], np.float32))
    t[3] = (0, 0, 1, 2)                                  # w = z + 2
    u["transform"] = t
    a = [(-0.5, 0.0, 0.0)], [(0.5, 0.0, 0.0)]           # w = 2
    b = [(-1.0, 0.0, 2.0)], [(1.0, 0.0, 2.0)]           # w = 4: the same NDC row, farther
    for order in ((a, b), (b, a)):
        s = np.concatenate([np.array(order[0][0], np.float32), np.array(order[1][0], np.float32)])
        e = np.concatenate([np.array(order[0][1], np.float32), np.array(order[1][1], np.float32)])
        pixel, value = O.rasterize(u, s, e, np.array([O.BOX_COLOR, O.FRUSTUM_COLOR], np.uint64), 64, 64)
        fb = np.full(64 * 64, np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
        np.minimum.at(fb, pixel, value)
        row = (fb.reshape(64, 64)[32, 24:41] >> np.uint64(32)).view(np.uint64).astype(np.uint32).view(np.float32)
        assert (row <= 2.0).all()


# ---- the CPU model of a whole frame: oracle.Canon.render with the overlay over it ------------------------------------

def canon_uniforms(mn, mx, width, height, overlay):
    from simlod_b200 import api, camera
    u = api.Uniforms()
    u.width, u.height = float(width), float(height)
    view, proj = camera.autofocus(mx, width, height)
    wvp = (np.asarray(proj, np.float32) @ np.asarray(view, np.float32)).astype(np.float32)
    for name in ("world", "view", "proj"):
        setattr(u, name, api.mat4_to_struct(np.eye(4, dtype=np.float32)))
    u.transform = u.transform_updateBound = api.mat4_to_struct(wvp)
    u.transformInv_updateBound = api.mat4_to_struct(np.linalg.inv(wvp.astype(np.float64)).astype(np.float32))
    for i in range(3):
        u.boxMin[i], u.boxMax[i] = float(mn[i]), float(mx[i])
    u.showPoints, u.minNodeSize, u.pointSize, u.LOD, u.doUpdateVisibility = 1, 64.0, 1, 0.2, 1
    u.showBoundingBox = 1 if overlay else 0
    return bytes(bytearray(u))


def test_canon_render_draws_the_overlay_over_the_oracle_frame():
    import oracle
    from simlod_b200 import data
    pts, mn, mx = data.uniform_cube(200_000, size=256.0, seed=5)
    o = oracle.Oracle(mn, mx)
    o.add_batch(pts)
    canon = o.canon()
    w, h = 320, 176
    plain, rs, flags = canon.render(canon_uniforms(mn, mx, w, h, False), w, h)
    off, rs_off, _ = O.canon_render(canon, canon_uniforms(mn, mx, w, h, False), w, h)
    assert (off == plain).all()                                      # the flag off: Canon.render's frame itself
    on, rs_on, flags_on = O.canon_render(canon, canon_uniforms(mn, mx, w, h, True), w, h)
    assert rs_on.numVisibleNodes == rs.numVisibleNodes and (flags_on == flags).all()
    drawn = O.drawn_from_canon_flags(canon.records, flags)
    assert len(drawn) == rs.numVisibleNodes > 0
    # every pixel either keeps the sample frame's word or carries a line colour, in front of what was there
    changed = (on != plain)
    assert changed.any()
    colors = set((on[changed] & np.uint64(0xFFFFFFFF)).tolist())
    assert colors <= {O.FRUSTUM_COLOR, O.BOX_COLOR} and (on <= plain).all()
    u = O.uniforms_from_bytes(canon_uniforms(mn, mx, w, h, True))
    assert (on.reshape(-1) == O.overlay_frame(u, drawn, w, h, plain)).all()
