"""CPU-only: the clip's layout and constants, its restatement (clip_restatement) against a plain per-sample, per-pixel
loop on hand-made sets (samples exactly on box faces, on a sphere's surface and at plane value 0, -0.0, overlapping
regions), and the resource use of simlod_render_clip and of the clipped pick kernels. The GPU frames are pinned to this
restatement in test_clip_gpu.py."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import clip_restatement as K
import pick_restatement as P
from conftest import ROOT
from simlod_b200 import api
from simlod_b200 import build as B

F = np.float32
W, H = 40, 24


def test_clip_layout_matches_the_c_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include "simlod_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %zu\\n", sizeof(SimlodClip), offsetof(SimlodClip, mode), offsetof(SimlodClip, num_regions), '
                   'offsetof(SimlodClip, regions));\n'
                   'printf("%d %d %d %d\\n", SIMLOD_CLIP_NONE, SIMLOD_CLIP_INSIDE, SIMLOD_CLIP_OUTSIDE, SIMLOD_CLIP_MAX_REGIONS);\n'
                   'return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    s = api.SimlodClip
    assert out[:4] == [C.sizeof(s), s.mode.offset, s.num_regions.offset, s.regions.offset] == [1224, 0, 4, 8]
    assert out[4:] == [api.CLIP_NONE, api.CLIP_INSIDE, api.CLIP_OUTSIDE, api.CLIP_MAX_REGIONS] == [0, 1, 2, 4]
    assert (K.NONE, K.INSIDE, K.OUTSIDE) == (0, 1, 2)
    assert "simlod_set_clip" in api.EXPORTS and hasattr(api.load_library(), "simlod_set_clip")


def clip(mode, *regions):
    c = api.SimlodClip(mode=mode, num_regions=len(regions))
    for k, r in enumerate(regions):
        c.regions[k] = r
    return c


# ---- a plain loop, stated without the restatement's helpers -------------------------------------------------------------

def plain_in(region, x, y, z):
    """The region query's predicate on one sample, float32 scalar by scalar."""
    x, y, z = F(x), F(y), F(z)
    if region.kind == api.REGION_BOX:
        return all(F(region.box_min[a]) <= p <= F(region.box_max[a]) for a, p in enumerate((x, y, z)))
    if region.kind == api.REGION_SPHERE:
        d = [p - F(region.center[a]) for a, p in enumerate((x, y, z))]
        return F(F(d[0] * d[0]) + F(d[1] * d[1])) + F(d[2] * d[2]) <= F(region.radius) * F(region.radius)
    return all(F(F(F(F(region.planes[k][0]) * x) + F(F(region.planes[k][1]) * y)) + F(F(region.planes[k][2]) * z)) +
               F(region.planes[k][3]) >= F(0) for k in range(region.num_planes))


def plain_frame(c, rec, pts, u):
    """Per sample: drawn or not by the clip; per covered pixel: the smallest (key, index) among the drawn candidates."""
    x, y, _, cand, key = P.sample_keys(rec, pts, u, W, H)
    best = {}
    for i in range(len(pts)):
        inside = any(plain_in(c.regions[k], pts["x"][i], pts["y"][i], pts["z"][i]) for k in range(c.num_regions))
        drawn = c.mode == K.NONE or (inside if c.mode == K.INSIDE else not inside)
        if not drawn or not cand[i]:
            continue
        for ox in range(u["pointSize"]):
            for oy in range(u["pointSize"]):
                p = min(max(int(x[i]) + ox, 0), W) + W * min(max(int(y[i]) + oy, 0), H)
                if p < W * H and (p not in best or (int(key[i]), i) < best[p]):
                    best[p] = (int(key[i]), i)
    out = np.full(W * H, -1, dtype=np.int64)
    for p, (_, i) in best.items():
        out[p] = i
    return out.reshape(H, W)


# w = z: a sample at (x, y, z) lands at pixel ((x/z + 1) W / 2, (y/z + 1) H / 2) with depth z
PERSPECTIVE = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 1, 0]]


def uniforms(**kw):
    u = api.Uniforms()
    u.width, u.height, u.showPoints, u.pointSize = float(W), float(H), 1, 1
    u.transform = api.mat4_to_struct(np.asarray(PERSPECTIVE, dtype=np.float32))
    for k, v in kw.items():
        setattr(u, k, v)
    return P.uniforms_from_bytes(bytes(bytearray(u)))


def view(xyz, color):
    pts = api.make_points(np.asarray(xyz, dtype=np.float32), np.asarray(color, dtype=np.uint32))
    rec = np.zeros(1, dtype=api.EXPORT_NODE_DTYPE)
    rec["name"], rec["num_points"] = [b"r"], [len(pts)]
    return rec, pts


# Samples on a 5 x 5 grid of x, y in [-0.4, 0.4] at three depths each (nearer ones win a pixel unless clipped), plus the
# edge cases: the faces of the box [-0.0, 0.2] x [-0.2, 0.2] x [1, 2], the sphere |p - (0, 0, 2)| <= 0.5 (0.3, 0.4, 2 lies on
# it exactly: 0.09 + 0.16 rounds to 0.25 in float32), and the plane z - 1.5 >= 0 at exactly 0
def edge_view():
    xyz, color = [], []
    for gx in np.linspace(-0.4, 0.4, 5):
        for gy in np.linspace(-0.4, 0.4, 5):
            for z, c in ((1.0, 0x10), (1.5, 0x20), (2.0, 0x30)):
                xyz.append((gx * z, gy * z, z)); color.append(c)
    xyz += [(0.0, 0.0, 1.0), (-0.0, 0.1, 1.0), (0.2, 0.2, 2.0), (0.2, -0.2, 1.0), (0.3, 0.4, 2.0), (0.1, 0.1, 1.5),
            (-0.3, 0.1, 1.5), (0.3, 0.4000001, 2.0)]
    color += [0x01, 0x02, 0x03, 0x04, 0x05, 0x06, 0x07, 0x08]
    return view(xyz, color)


BOX = api.Region.box((-0.0, -0.2, 1.0), (0.2, 0.2, 2.0))
SPHERE = api.Region.sphere((0.0, 0.0, 2.0), 0.5)
PLANE = api.Region.planes([[0.0, 0.0, 1.0, -1.5]])
OVERLAP = api.Region.box((0.0, -0.4, 0.9), (0.6, 0.4, 3.5))
CLIPS = [(K.NONE,)] + [(mode,) + regions for mode in (K.INSIDE, K.OUTSIDE)
                       for regions in ((BOX,), (SPHERE,), (PLANE,), (BOX, OVERLAP), (SPHERE, OVERLAP, PLANE), (BOX, SPHERE, PLANE, OVERLAP))]


def test_edge_cases_of_the_predicate():
    _, pts = edge_view()
    tail = pts[-8:]
    assert K.keep_mask(clip(K.INSIDE, BOX), tail).tolist() == [True, True, True, True, False, True, False, False]
    assert K.keep_mask(clip(K.INSIDE, SPHERE), tail).tolist() == [False, False, True, False, True, False, False, False]
    assert K.keep_mask(clip(K.INSIDE, PLANE), tail).tolist() == [False, False, True, False, True, True, True, True]
    # -0.0 >= -0.0 and 0.0 >= -0.0: both zeros lie on the box's min face
    assert np.signbit(tail["x"][1]) and not np.signbit(tail["x"][0])
    for c in CLIPS:
        keep = K.keep_mask(clip(*c), pts)
        plain = [c[0] == K.NONE or (any(plain_in(r, *p) for r in c[1:]) == (c[0] == K.INSIDE)) for p in zip(pts["x"], pts["y"], pts["z"])]
        assert keep.tolist() == plain, c


def test_the_two_modes_partition_the_samples():
    _, pts = edge_view()
    for regions in ((BOX,), (SPHERE, OVERLAP), (BOX, SPHERE, PLANE, OVERLAP)):
        a, b = K.keep_mask(clip(K.INSIDE, *regions), pts), K.keep_mask(clip(K.OUTSIDE, *regions), pts)
        assert (a ^ b).all()


@pytest.mark.parametrize("settings", [{}, {"pointSize": 3}, {"pointSize": 5}, {"colorByNode": 1},
                                      {"useHighQualityShading": 1}, {"useHighQualityShading": 1, "pointSize": 3}])
def test_restatement_equals_the_plain_loop(settings):
    rec, pts = edge_view()
    u = uniforms(**settings)
    frames = []
    for c in CLIPS:
        got = K.clipped_pick(clip(*c), rec, pts, u, W, H)
        assert np.array_equal(got, plain_frame(clip(*c), rec, pts, u)), (c, settings)
        frames.append(got)
        keep = K.keep_mask(clip(*c), pts)
        assert keep[got[got >= 0]].all()
    assert np.array_equal(frames[0], P.pick_frame(rec, pts, u, W, H))
    # with one pixel per sample the frame of each clip differs from the unclipped one somewhere: the cases are not vacuous
    if not settings:
        assert all((f != frames[0]).any() for f in frames[1:])


def test_partition_identity_of_the_frame_keys():
    """Per pixel the smaller of the INSIDE and OUTSIDE keys is the unclipped frame's key (the atomicMin paths)."""
    rec, pts = edge_view()
    for settings in ({}, {"pointSize": 3}, {"colorByNode": 1}):
        u = uniforms(**settings)
        full = P.frame_key(rec, pts, u, P.pick_frame(rec, pts, u, W, H))
        for regions in ((BOX,), (SPHERE, OVERLAP), (PLANE,)):
            a = P.frame_key(rec, pts, u, K.clipped_pick(clip(K.INSIDE, *regions), rec, pts, u, W, H))
            b = P.frame_key(rec, pts, u, K.clipped_pick(clip(K.OUTSIDE, *regions), rec, pts, u, W, H))
            assert np.array_equal(np.minimum(a, b), full), (settings, regions)


def ptxas(name, tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / (name + ".cubin"))
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get(name, []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, name + ".cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                       r"[^\n]*Used (\d+) registers", res.stdout)
    return {k: tuple(int(v) for v in rest) for k, *rest in found}, res.stdout


# simlod_render_clip is kernel_render's text with the clip test in its draw paths: 64 registers at 4 blocks of 256 threads
# per SM, as kernel_render, and 8 bytes more stack frame (88 against 80 B, spill stores 96 against 92 B on nvcc 12.9)
CLIP_EXTRA_LOCAL = 8


def test_render_clip_resources(tmp_path):
    props, out = ptxas("render", tmp_path)
    assert "kernel_render" in props and "simlod_render_clip" in props, out
    k_stack, k_stores, _, k_regs = props["kernel_render"]
    c_stack, c_stores, _, c_regs = props["simlod_render_clip"]
    assert c_regs <= 64 and k_regs <= 64, out
    assert c_stack <= k_stack + CLIP_EXTRA_LOCAL and c_stores <= k_stores + CLIP_EXTRA_LOCAL, out


def test_clipped_pick_kernels_use_no_local_memory(tmp_path):
    props, out = ptxas("pick", tmp_path)
    for k in ("simlod_pick_key", "simlod_pick_index"):
        assert props[k][:3] == (0, 0, 0), out
