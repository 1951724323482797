"""TEST INFRASTRUCTURE — CPU restatement of simlod_query_nearest (DESIGN.md §9.10), independent of simlod_b200 (which it
checks): the k samples of the sample set with the smallest (d2, index) key, d2 in numpy float32 one operation at a time
(the device's order: ((dx*dx + dy*dy) + dz*dz), d = p - q), over the export's samples.

  candidates(export, depth, box_min, box_max, rcp)   boolean mask over the export's samples: the sample set (the leaves'
      eligible points for depth None, the cut's eligible points and all its voxels otherwise)
  key(samples, q)                                    the float32 d2 of every sample for one query
  brute_force(export, queries, k, depth, box, rcp, max_radius)   every key of every candidate, sorted: the plain statement
  nearest(export, queries, k, depth, box, rcp, max_radius)       the same result through a float64 k-d tree superset
  Prepared(export, depth, box, rcp) / search(prepared, queries, k, max_radius)   the same, one tree for several calls
  nearest_image(nodes, heap, nodes_addr, heap_addr, queries, k, depth, box_min, box_max, rcp, max_radius)   the same for
      a raw device image: the byte-exact expectation for the same buffers

Both return (index int64 (N, k), d2 float32 (N, k)), -1 / +inf in an empty slot and for a query with a non-finite
coordinate. The superset: every candidate within the float64 k-th distance D of the query, scaled by (1 + 1e-5) plus
1e-22. The float32 key's relative error is about 2^-21, far inside that margin, and 1e-22 covers distances whose squares
underflow; a query whose keys reach +inf (coordinates near the float range) is answered by brute force, since then ties
by index decide."""
import numpy as np

import export_restatement as R
import query_restatement as Q

F = np.float32


def candidates(export, depth, box_min, box_max, rcp=None):
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
    return taken & (is_voxel | Q.in_cube(samples, box_min, box_max, rcp))


def _xyz(samples):
    s = np.ascontiguousarray(samples)
    return s["x"].astype(F), s["y"].astype(F), s["z"].astype(F)


def key(xyz, q):
    """xyz: (x, y, z) float32 arrays; q: 3 floats. d = p - q, ((dx*dx + dy*dy) + dz*dz), all float32."""
    x, y, z = xyz
    with np.errstate(over="ignore", under="ignore"):
        dx, dy, dz = x - F(q[0]), y - F(q[1]), z - F(q[2])
        return (dx * dx + dy * dy) + dz * dz


def _queries(queries):
    a = np.asarray(queries)
    if a.dtype.names:
        a = np.stack([a["x"], a["y"], a["z"]], axis=1)
    return np.ascontiguousarray(a[:, :3], dtype=F)


def _radius2(max_radius):
    r = F(np.inf if max_radius is None else max_radius)
    with np.errstate(over="ignore"):
        return r * r


def _take(idx, d2, k, rr):
    """The k smallest (d2, index) keys among idx / d2 with d2 <= rr."""
    ok = d2 <= rr
    idx, d2 = idx[ok], d2[ok]
    order = np.lexsort((idx, d2))[:k]
    out_i = np.full(k, -1, dtype=np.int64)
    out_d = np.full(k, np.inf, dtype=F)
    out_i[:len(order)], out_d[:len(order)] = idx[order], d2[order]
    return out_i, out_d


def brute_force(export, queries, k, depth, box_min, box_max, rcp=None, max_radius=None):
    q = _queries(queries)
    cand = np.nonzero(candidates(export, depth, box_min, box_max, rcp))[0]
    xyz = tuple(v[cand] for v in _xyz(export[1]))
    rr = _radius2(max_radius)
    index = np.full((len(q), k), -1, dtype=np.int64)
    dist2 = np.full((len(q), k), np.inf, dtype=F)
    for t in range(len(q)):
        if np.isfinite(q[t]).all():
            index[t], dist2[t] = _take(cand, key(xyz, q[t]), k, rr)
    return index, dist2


class Prepared:
    """The sample set of one export with its float64 k-d tree, for several calls of search()."""

    def __init__(self, export, depth, box_min, box_max, rcp=None):
        from scipy.spatial import cKDTree
        self.cand = np.nonzero(candidates(export, depth, box_min, box_max, rcp))[0]
        self.xyz = tuple(v[self.cand] for v in _xyz(export[1]))
        self.tree = cKDTree(np.stack(self.xyz, axis=1).astype(np.float64)) if len(self.cand) else None


def search(prep, queries, k, max_radius=None):
    q = _queries(queries)
    cand, xyz = prep.cand, prep.xyz
    rr = _radius2(max_radius)
    index = np.full((len(q), k), -1, dtype=np.int64)
    dist2 = np.full((len(q), k), np.inf, dtype=F)
    valid = np.nonzero(np.isfinite(q).all(axis=1))[0]
    if len(cand) == 0 or len(valid) == 0:
        return index, dist2
    kk = min(k, len(cand))
    qv = q[valid].astype(np.float64)
    dist, _ = prep.tree.query(qv, k=kk)
    dk = dist.reshape(len(valid), kk)[:, kk - 1]
    reach = dk * (1.0 + 1e-5) + 1e-22
    if max_radius is not None:                               # nothing beyond the radius is a candidate
        reach = np.minimum(reach, float(max_radius) * (1.0 + 1e-5) + 1e-22)
    balls = prep.tree.query_ball_point(qv, reach)
    for t, members in zip(valid, balls):
        members = np.asarray(members, dtype=np.int64)
        d2 = key(tuple(v[members] for v in xyz), q[t])
        if rr == np.inf and np.isinf(d2).any():               # overflowed keys tie, and the index decides among all
            index[t], dist2[t] = _take(cand, key(xyz, q[t]), k, rr)
        else:
            index[t], dist2[t] = _take(cand[members], d2, k, rr)
    return index, dist2


def nearest(export, queries, k, depth, box_min, box_max, rcp=None, max_radius=None):
    return search(Prepared(export, depth, box_min, box_max, rcp), queries, k, max_radius)


def nearest_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, queries, k, depth, box_min, box_max, rcp=None, max_radius=None):
    export = R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth)
    return nearest(export, queries, k, depth, box_min, box_max, rcp, max_radius)
