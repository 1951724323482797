"""Inputs of the golden fixtures (shared by the generator, which runs the reference's kernels on an
H100, and by the CPU-only test that checks the oracle against what they produced)."""
import numpy as np

from simlod_b200 import camera, data

GOLDEN_W, GOLDEN_H = 320, 176      # fewer 16x16 tiles than render blocks: the EDL pass covers no tile (render.cu:1273)


def _split(points, sizes):
    out, s = [], 0
    for n in sizes:
        out.append(points[s:s + n])
        s += n
    assert s == len(points)
    return out


def cases():
    """(name, batches, (box_min, box_max), (view, proj))"""
    pts, mn, mx = data.uniform_cube(300_000, size=256.0, seed=21)
    yield "uniform_300k", _split(pts, [200_000, 100_000]), (mn, mx), camera.autofocus(mx, GOLDEN_W, GOLDEN_H)
    pts, mn, mx = data.uniform_cube(120_000, size=64.0, seed=5)
    yield "root_split_120k", _split(pts, [20_000, 20_000, 10_000, 1, 30_000, 39_999]), (mn, mx), camera.autofocus(mx, GOLDEN_W, GOLDEN_H, yaw_offset=1.0)
    pts, mn, mx = data.terrain(1_000_000)
    yield "terrain_1m_ragged", _split(pts, [400_000, 0, 7, 599_993]), (mn, mx), camera.autofocus(mx, GOLDEN_W, GOLDEN_H)
