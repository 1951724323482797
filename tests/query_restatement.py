"""TEST INFRASTRUCTURE — CPU restatement of simlod_query_region (DESIGN.md §9.8), independent of simlod_b200 (which it
checks): the two per-sample predicates in numpy float32, one operation at a time (numpy contracts nothing), and the
query as a plain filter over the export's samples, with no hierarchy shortcut.

  contains(region, xyz)                    the point predicate; region: anything with the fields of SimlodRegion
  in_cube(xyz, box_min, box_max, rcp)      the eligibility predicate (the builder's quantisation below 2^20)
  brute_force(points, region, box, rcp)    the eligible points of a source stream inside the region
  query_export(export, region, depth, box, rcp)   the filter over (nodes, samples, info) of export_restatement
  query_image(nodes, heap, nodes_addr, heap_addr, region, depth, box, rcp)   the same for a raw device image: the
      byte-exact expectation for the same buffers

`rcp` is MUFU.RCP(cube size): exact for a power-of-two cube (the default); otherwise pass SimLOD.device_rcp's float."""
import numpy as np

import export_restatement as R

BOX, SPHERE, PLANES = 1, 2, 3
F = np.float32


def _xyz(samples):
    s = np.ascontiguousarray(samples)
    return s["x"].astype(F), s["y"].astype(F), s["z"].astype(F)


def contains(region, samples):
    x, y, z = _xyz(samples)
    if region.kind == BOX:
        mn, mx = [F(v) for v in region.box_min], [F(v) for v in region.box_max]
        return (x >= mn[0]) & (x <= mx[0]) & (y >= mn[1]) & (y <= mx[1]) & (z >= mn[2]) & (z <= mx[2])
    if region.kind == SPHERE:
        c, r = [F(v) for v in region.center], F(region.radius)
        dx, dy, dz = x - c[0], y - c[1], z - c[2]
        with np.errstate(over="ignore"):
            return ((dx * dx + dy * dy) + dz * dz) <= r * r
    if region.kind == PLANES:
        ok = np.ones(len(x), dtype=bool)
        for k in range(region.num_planes):
            nx, ny, nz, d = (F(v) for v in region.planes[k])
            with np.errstate(over="ignore", invalid="ignore"):
                ok &= (((nx * x + ny * y) + nz * z) + d) >= F(0)
        return ok
    raise ValueError("unknown region kind %r" % region.kind)


def cube_of(box_min, box_max, rcp=None):
    mn, mx = np.asarray(box_min, dtype=F), np.asarray(box_max, dtype=F)
    size = (mx - mn).max()
    if rcp is None:
        m, _ = np.frexp(size)
        assert m == 0.5, "cube size %r is not a power of two: pass the device's MUFU.RCP of it" % size
        rcp = F(1.0) / size
    return mn, F(rcp)


def in_cube(samples, box_min, box_max, rcp=None):
    """Not below boxMin, and u32(2^20 * (p - boxMin) * rcp) < 2^20, on every axis (construct.cu quantize)."""
    mn, rcp = cube_of(box_min, box_max, rcp)
    ok = np.ones(len(samples), dtype=bool)
    for p, m in zip(_xyz(samples), mn):
        with np.errstate(over="ignore", invalid="ignore"):
            u = ((p + (-m)) * F(1048576.0)) * rcp
        ok &= (p >= m) & ~(u >= F(1048576.0))            # the conversion truncates; NaN converts to 0
    return ok


def brute_force(points, region, box_min, box_max, rcp=None):
    p = np.ascontiguousarray(points)
    return p[contains(region, p) & in_cube(p, box_min, box_max, rcp)]


def query_export(export, region, depth, box_min, box_max, rcp=None):
    """export: (nodes, samples, info) of export_restatement for the same `depth` (None: the full export, of which the
    query takes the leaves' points). Returns (samples, num_points, num_voxels)."""
    nodes, samples, _ = export
    is_voxel = np.zeros(len(samples), dtype=bool)
    taken = np.ones(len(samples), dtype=bool)
    full = depth is None or depth < 0
    for r in range(len(nodes)):
        a, n_p, n_v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
        is_voxel[a + n_p:a + n_p + n_v] = True
        if full:
            taken[a + n_p:a + n_p + n_v] = False
            if not nodes["flags"][r] & R.LEAF:
                taken[a:a + n_p] = False
    keep = taken & contains(region, samples) & (is_voxel | in_cube(samples, box_min, box_max, rcp))
    return samples[keep], int((keep & ~is_voxel).sum()), int((keep & is_voxel).sum())


def query_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, region, depth, box_min, box_max, rcp=None):
    return query_export(R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth), region, depth, box_min, box_max, rcp)
