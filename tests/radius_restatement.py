"""TEST INFRASTRUCTURE — CPU restatement of simlod_query_radius (DESIGN.md §9.12), independent of simlod_b200 (which it
checks): for each query every sample of the sample set whose float32 key d2 (nearest_restatement.key, the device's
((dx*dx + dy*dy) + dz*dz), d = p - q) is <= fl(radius * radius), ordered by (Z-key of the sample's terminal record,
index), in CSR form.

  zkeys(nodes)                                    per record: morton(X, Y, Z at its level) << 3 * (20 - level)
  brute_force(export, queries, radius, depth, box_min, box_max, rcp)   every key of every candidate: the plain statement
  radius(export, queries, radius, depth, box_min, box_max, rcp)        the same through a float64 k-d tree superset
  Prepared(export, depth, box, rcp) / search(prepared, queries, radius)   the same, one tree for several calls
  radius_image(nodes, heap, nodes_addr, heap_addr, queries, radius, depth, box_min, box_max, rcp)   the same for a raw
      device image: the byte-exact expectation for the same buffers

All return (offsets int64 (N + 1,), index int64 (M,), dist2 float32 (M,)); a query with a non-finite coordinate has no
neighbours. The superset: query_ball_point at radius * (1 + 1e-5) + 1e-22 in float64, then the exact float32 keys. The
key's relative error is about 2^-21, far inside that margin, and 1e-22 covers distances whose squares underflow. When
fl(radius * radius) is +inf every candidate is a neighbour (keys that overflowed included), answered by brute force."""
import numpy as np

import export_restatement as R
import nearest_restatement as N

F = np.float32


def _spread(v):
    x = np.asarray(v, dtype=np.uint64) & np.uint64(0x1FFFFF)
    for shift, mask in ((32, 0x1F00000000FFFF), (16, 0x1F0000FF0000FF), (8, 0x100F00F00F00F00F), (4, 0x10C30C30C30C30C3),
                        (2, 0x1249249249249249)):
        x = (x | (x << np.uint64(shift))) & np.uint64(mask)
    return x


def zkeys(nodes):
    level = nodes["level"].astype(np.uint64)
    key = (_spread(nodes["X"]) << np.uint64(2)) | (_spread(nodes["Y"]) << np.uint64(1)) | _spread(nodes["Z"])
    return key << (np.uint64(3) * (np.uint64(R.MAX_DEPTH) - level))


def rank(export):
    """Per sample: its position in the order (Z-key of its terminal record, index). Samples of inner records (never
    candidates) follow."""
    nodes, samples, _ = export
    z = np.full(len(samples), np.iinfo(np.uint64).max, dtype=np.uint64)
    zk = zkeys(nodes)
    for r in np.nonzero(nodes["first_child"] < 0)[0]:
        a = int(nodes["sample_offset"][r])
        z[a:a + int(nodes["num_points"][r]) + int(nodes["num_voxels"][r])] = zk[r]
    out = np.empty(len(samples), dtype=np.int64)
    out[np.lexsort((np.arange(len(samples)), z))] = np.arange(len(samples))
    return out


def _rr(radius):
    r = F(radius)
    with np.errstate(over="ignore"):
        return r * r


def _csr(parts):
    counts = np.array([len(p[0]) for p in parts], dtype=np.int64)
    offsets = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum(counts, out=offsets[1:])
    index = np.concatenate([p[0] for p in parts] + [np.zeros(0, dtype=np.int64)]).astype(np.int64)
    dist2 = np.concatenate([p[1] for p in parts] + [np.zeros(0, dtype=F)]).astype(F)
    return offsets, index, dist2


_EMPTY = (np.zeros(0, dtype=np.int64), np.zeros(0, dtype=F))


def _select(idx, d2, rr, order_rank):
    ok = d2 <= rr
    idx, d2 = idx[ok], d2[ok]
    o = np.argsort(order_rank[idx], kind="stable")
    return idx[o], d2[o]


def brute_force(export, queries, radius, depth, box_min, box_max, rcp=None):
    q = N._queries(queries)
    cand = np.nonzero(N.candidates(export, depth, box_min, box_max, rcp))[0]
    xyz = tuple(v[cand] for v in N._xyz(export[1]))
    rr, rk = _rr(radius), rank(export)
    return _csr([_select(cand, N.key(xyz, q[t]), rr, rk) if np.isfinite(q[t]).all() else _EMPTY for t in range(len(q))])


class Prepared(N.Prepared):
    """The sample set of one export with its float64 k-d tree and its output order, for several calls of search()."""

    def __init__(self, export, depth, box_min, box_max, rcp=None):
        super().__init__(export, depth, box_min, box_max, rcp)
        self.rank = rank(export)


def search(prep, queries, radius):
    q = N._queries(queries)
    cand, xyz, rr = prep.cand, prep.xyz, _rr(radius)
    parts = [_EMPTY] * len(q)
    valid = np.nonzero(np.isfinite(q).all(axis=1))[0]
    if len(cand) == 0 or len(valid) == 0:
        return _csr(parts)
    if rr == np.inf:                                          # every candidate, overflowed keys included
        for t in valid:
            parts[t] = _select(cand, N.key(xyz, q[t]), rr, prep.rank)
        return _csr(parts)
    balls = prep.tree.query_ball_point(q[valid].astype(np.float64), float(radius) * (1.0 + 1e-5) + 1e-22)
    for t, members in zip(valid, balls):
        members = np.asarray(members, dtype=np.int64)
        parts[t] = _select(cand[members], N.key(tuple(v[members] for v in xyz), q[t]), rr, prep.rank)
    return _csr(parts)


def radius(export, queries, radius_, depth, box_min, box_max, rcp=None):
    return search(Prepared(export, depth, box_min, box_max, rcp), queries, radius_)


def radius_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, queries, radius_, depth, box_min, box_max, rcp=None):
    export = R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth)
    return radius(export, queries, radius_, depth, box_min, box_max, rcp)
