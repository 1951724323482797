"""Camera math of the reference host, restated (inputs to the kernels, passed as bytes in Uniforms).

  OrbitControls::update   include/OrbitControls.h:140-159   world = T(target) Rz(yaw) Rx(pitch) flip T(0,0,radius)
  Camera::update          include/GLRenderer.h:156-161      view = inverse(world); proj = perspective(fovy, aspect, 0.1, 2e6)
  auto-focus on load      main_progressive_octree.cpp:1077-1084
  presets                 main_progressive_octree.cpp:1314-1329

Matrices here are row-major math matrices (M @ column vector); the reference keeps column-major
glm matrices and uploads their transpose, which is the same bytes as our rows (main.cpp:290-298).
"""
import math

import numpy as np


def translate(v):
    m = np.eye(4)
    m[:3, 3] = v
    return m


def rotate(angle, axis):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    c, s = math.cos(angle), math.sin(angle)
    x, y, z = axis
    r = np.array([
        [c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s, 0],
        [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s, 0],
        [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c), 0],
        [0, 0, 0, 1]], dtype=np.float64)
    return r


FLIP = np.array([[1, 0, 0, 0], [0, 0, -1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], dtype=np.float64)


def orbit_world(yaw, pitch, radius, target):
    return translate(target) @ rotate(yaw, (0, 0, 1)) @ rotate(pitch, (1, 0, 0)) @ FLIP @ translate((0.0, 0.0, radius))


def perspective(fovy_rad, aspect, near, far):
    """glm::perspective, right-handed, clip z in [-1, 1] (GLM 0.9.9 defaults)."""
    t = math.tan(fovy_rad / 2.0)
    p = np.zeros((4, 4))
    p[0, 0] = 1.0 / (aspect * t)
    p[1, 1] = 1.0 / t
    p[2, 2] = -(far + near) / (far - near)
    p[3, 2] = -1.0
    p[2, 3] = -(2.0 * far * near) / (far - near)
    return p


def orbit_camera(yaw, pitch, radius, target, width, height, fovy_deg=60.0, near=0.1, far=2_000_000.0):
    """Returns (view, proj) as float64 row-major matrices."""
    world = orbit_world(yaw, pitch, radius, np.asarray(target, dtype=np.float64))
    view = np.linalg.inv(world)
    proj = perspective(math.pi * fovy_deg / 180.0, float(width) / float(height), near, far)
    return view, proj


def autofocus(box_size, width, height, yaw_offset=0.0):
    """The view the reference selects after loading a file (main.cpp:1077-1084)."""
    bs = np.asarray(box_size, dtype=np.float64)
    radius = math.sqrt(float((bs * bs).sum()))
    target = (bs[0] * 0.5, bs[1] * 0.5, bs[2] * 0.1)
    return orbit_camera(-1.15 + yaw_offset, -0.57, radius, target, width, height)


MORRO_BIRD = dict(yaw=-0.207, pitch=-0.797, radius=3866.886, target=(2398.747, 2167.120, -394.165))
MORRO_CLOSE = dict(yaw=-11.270, pitch=-0.225, radius=93.982, target=(2750.218, 974.775, 76.230))


def pixel_rays(view, proj, width, height, pixels=None):
    """World-space rays through the centres of pixels of a width x height frame: (origins, directions), (N, 3) float64,
    the origin the camera's position, the direction from the near to the far plane through (x + 0.5, y + 0.5), with
    NDC y = 2 (y + 0.5) / height - 1. pixels: an (N, 2) array of (x, y), or None for every pixel, row by row. For
    SimLOD.query_ray."""
    if pixels is None:
        ys, xs = np.mgrid[0:height, 0:width]
        pixels = np.stack([xs.ravel(), ys.ravel()], axis=1)
    p = np.asarray(pixels, dtype=np.float64).reshape(-1, 2)
    ndc = np.stack([2.0 * (p[:, 0] + 0.5) / width - 1.0, 2.0 * (p[:, 1] + 0.5) / height - 1.0], axis=1)
    inv = np.linalg.inv(np.asarray(proj, dtype=np.float64) @ np.asarray(view, dtype=np.float64))
    ends = []
    for z in (-1.0, 1.0):
        h = np.concatenate([ndc, np.full((len(p), 1), z), np.ones((len(p), 1))], axis=1) @ inv.T
        ends.append(h[:, :3] / h[:, 3:4])
    origin = np.linalg.inv(np.asarray(view, dtype=np.float64))[:3, 3]
    return np.tile(origin, (len(p), 1)), ends[1] - ends[0]
