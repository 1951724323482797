"""TEST INFRASTRUCTURE — CPU restatement of simlod_query_heightmap (DESIGN.md §9.14), independent of simlod_b200 (which it
checks): every sample of the sample set is binned, with no culling, in numpy float32 / float64 one operation at a time
in the device's order. Equality with the device therefore also shows that the device's culling never drops a sample.

  cell_of(samples, origin, cell, nx, ny)      the cell id j * nx + i of each sample, -1 for none
  binned(export, depth, box_min, box_max, origin, cell, shape, rcp)    the non-empty cells only (sparse)
  heightmap(export, depth, box_min, box_max, origin, cell, shape, rcp)  the dense (ny, nx) results
  heightmap_image(nodes, heap, nodes_addr, heap_addr, depth, box_min, box_max, origin, cell, shape, rcp)   the same for
      a raw device image: the byte-exact expectation for the same buffers

heightmap returns (count int64, z_min, z_max, z_mean float32, top int64, samples POINT_DTYPE), each (ny, nx): 0, NaN
(0x7fc00000), -1 and zeros for an empty cell."""
import numpy as np

import export_restatement as R
import nearest_restatement as N

F = np.float32
NAN_BITS = 0x7FC00000


def ordered(z):
    """The sign-aware bit order of float32 z as uint32: -0 below +0."""
    b = np.ascontiguousarray(z, dtype=F).view(np.uint32)
    return np.where(b >> 31 == 1, ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def unordered(o):
    o = np.asarray(o, dtype=np.uint32)
    return np.where(o >> 31 == 1, o & np.uint32(0x7FFFFFFF), ~o).astype(np.uint32).view(F)


def cell_of(samples, origin, cell, nx, ny):
    """u = fl(fl(x - ox) / cell), v likewise; cell (trunc u, trunc v) when u >= 0, v >= 0 (a NaN fails, -0 passes),
    trunc u < nx and trunc v < ny."""
    s = np.ascontiguousarray(samples)
    with np.errstate(all="ignore"):
        u = (s["x"].astype(F) - F(origin[0])) / F(cell)
        v = (s["y"].astype(F) - F(origin[1])) / F(cell)
        tu, tv = np.trunc(u), np.trunc(v)
        ok = (u >= 0) & (v >= 0) & (tu < nx) & (tv < ny)
        i = np.where(ok, tu, 0).astype(np.int64)
        j = np.where(ok, tv, 0).astype(np.int64)
    return np.where(ok, j * nx + i, -1)


def mean_constants(box_min, box_max):
    """(minz, K) in float64: minz = boxMin[2]; K = 2^30 / size, size the cube edge in float32."""
    mn, mx = np.asarray(box_min, dtype=F), np.asarray(box_max, dtype=F)
    size = (mx - mn).max()
    return float(mn[2]), 2.0 ** 30 / float(size)


def quantised(z, box_min, box_max):
    """q = rint_even(((double)z - minz) * K) as int64."""
    minz, K = mean_constants(box_min, box_max)
    return np.rint((np.asarray(z, dtype=F).astype(np.float64) - minz) * K).astype(np.int64)


def mean_of(S, n, box_min, box_max):
    """z_mean = float32(minz + ((double)S / (double)n) / K)."""
    minz, K = mean_constants(box_min, box_max)
    return (minz + (np.asarray(S, dtype=np.int64).astype(np.float64) / np.asarray(n, dtype=np.float64)) / K).astype(F)


def binned(export, depth, box_min, box_max, origin, cell, shape, rcp=None):
    """The non-empty cells in ascending id: (ids, count, z_min, z_max, z_mean, top)."""
    _, samples, _ = export
    ny, nx = shape
    cand = np.nonzero(N.candidates(export, depth, box_min, box_max, rcp))[0]
    cid = cell_of(samples[cand], origin, cell, nx, ny)
    keep = cid >= 0
    idx, cid = cand[keep], cid[keep]
    z = np.ascontiguousarray(samples["z"][idx]).astype(F)
    if not len(idx):
        e = np.zeros(0, dtype=np.int64)
        return e, e, np.zeros(0, F), np.zeros(0, F), np.zeros(0, F), e
    oz = ordered(z)
    order = np.lexsort((idx, ~oz, cid))              # per cell: the highest z first, equal z by index
    cid, idx, oz, q = cid[order], idx[order], oz[order], quantised(z[order], box_min, box_max)
    starts = np.concatenate([[0], np.nonzero(np.diff(cid))[0] + 1])
    count = np.diff(np.concatenate([starts, [len(cid)]])).astype(np.int64)
    z_min = unordered(np.minimum.reduceat(oz, starts))
    z_max = unordered(oz[starts])
    z_mean = mean_of(np.add.reduceat(q, starts), count, box_min, box_max)
    return cid[starts], count, z_min, z_max, z_mean, idx[starts].astype(np.int64)


def heightmap(export, depth, box_min, box_max, origin, cell, shape, rcp=None):
    ny, nx = shape
    ids, count, z_min, z_max, z_mean, top = binned(export, depth, box_min, box_max, origin, cell, shape, rcp)
    out_count = np.zeros(nx * ny, dtype=np.int64)
    out_top = np.full(nx * ny, -1, dtype=np.int64)
    zs = [np.full(nx * ny, NAN_BITS, dtype=np.uint32).view(F) for _ in range(3)]
    out_count[ids], out_top[ids] = count, top
    for dst, src in zip(zs, (z_min, z_max, z_mean)):
        dst[ids] = src
    out_samples = np.zeros(nx * ny, dtype=R.POINT_DTYPE)
    out_samples[ids] = export[1][top]
    return tuple(a.reshape(ny, nx) for a in (out_count, *zs, out_top, out_samples))


def heightmap_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth, box_min, box_max, origin, cell, shape, rcp=None):
    export = R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth)
    return heightmap(export, depth, box_min, box_max, origin, cell, shape, rcp)
