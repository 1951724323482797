"""TEST INFRASTRUCTURE — CPU restatement of simlod_query_ray (DESIGN.md §9.11), independent of simlod_b200 (which it
checks): per ray, the sample of the sample set with the smallest (t bits, index) key among the hits. The direction is
normalised in float64 and t, h2 computed in numpy float32 one operation at a time, in the device's order.

  rays(origins, directions, tmin, tmax)              (N, 8) float32 ray records ox, oy, oz, tmin, dx, dy, dz, tmax
  normalise(rays) / valid(rays)                      the direction u (float32) and which rays are valid
  key(xyz, o, u)                                     float32 t and h2 of every sample for one ray
  brute_force(export, rays, radius, depth, box_min, box_max, rcp)   every candidate of every ray: the plain statement
  Prepared(export, depth, box, rcp) / search(prepared, rays, radius)  the same result through a coarse grid superset
  trace(export, rays, radius, depth, box, rcp)       Prepared + search in one call
  trace_image(nodes, heap, nodes_addr, heap_addr, rays, radius, depth, box_min, box_max, rcp)   the same for a raw
      device image: the byte-exact expectation for the same buffers

All return (index int64 (N,), t float32 (N,), h2 float32 (N,)): -1 / +inf / +inf for a ray without a hit. The superset:
the candidates are binned into a uniform grid; a ray keeps the cells whose sample bounds, inflated by
radius (1 + 1e-5) + 1e-5 D (D the largest distance from the origin to the cell), its segment [tmin, tmax], widened by
1e-5 D, crosses, all in float64, and takes exact keys over their samples in order of the cells' least possible t,
GROUP samples at a time, until no later cell can hold a better hit. The float32 t and h2 are within about 2^-21 D of their exact values, far inside that
margin. A ray whose float32 products could overflow (a distance of 1e37 or more) or whose radius squares to +inf is
answered by brute force."""
import numpy as np

import export_restatement as R
import nearest_restatement as N

F = np.float32
GRID = 24                                                    # cells per axis of the superset's grid
GROUP = 1 << 15                                              # samples evaluated at a time, front to back


def rays(origins, directions, tmin=0.0, tmax=np.inf):
    o, d = np.asarray(origins, dtype=F).reshape(-1, 3), np.asarray(directions, dtype=F).reshape(-1, 3)
    r = np.empty((len(o), 8), dtype=F)
    r[:, 0:3], r[:, 4:7] = o, d
    r[:, 3] = np.broadcast_to(np.asarray(tmin, dtype=F), (len(o),))
    r[:, 7] = np.broadcast_to(np.asarray(tmax, dtype=F), (len(o),))
    return r


def normalise(r):
    """u = float32(d / len), len = sqrt((dx*dx + dy*dy) + dz*dz), every operation float64 round to nearest."""
    d = np.asarray(r, dtype=F)[:, 4:7].astype(np.float64)
    with np.errstate(all="ignore"):
        length = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        return (d / length[:, None]).astype(F)


def valid(r):
    r = np.asarray(r, dtype=F)
    o, d, tmin, tmax = r[:, 0:3], r[:, 4:7], r[:, 3], r[:, 7]
    with np.errstate(invalid="ignore"):
        return (np.isfinite(o).all(axis=1) & np.isfinite(d).all(axis=1) & (d != 0).any(axis=1) & np.isfinite(tmin) &
                (tmin >= 0) & (tmax >= tmin))


def key(xyz, o, u):
    """xyz: (x, y, z) float32 arrays; o, u: 3 float32 each. w = p - o; t = ((wx*ux + wy*uy) + wz*uz) + 0;
    c = w x u; h2 = (cx*cx + cy*cy) + cz*cz; all float32."""
    x, y, z = xyz
    ox, oy, oz = (F(v) for v in o)
    ux, uy, uz = (F(v) for v in u)
    with np.errstate(all="ignore"):
        wx, wy, wz = x - ox, y - oy, z - oz
        t = ((wx * ux + wy * uy) + wz * uz) + F(0.0)
        cx = wy * uz - wz * uy
        cy = wz * ux - wx * uz
        cz = wx * uy - wy * ux
        h2 = (cx * cx + cy * cy) + cz * cz
    return t, h2


def _radius2(radius):
    with np.errstate(over="ignore"):
        return F(radius) * F(radius)


def _first(idx, t, h2, tmin, tmax, rr):
    """The hit with the least (t bits, index) among idx / t / h2, or (-1, +inf, +inf)."""
    with np.errstate(invalid="ignore"):
        hit = (t >= tmin) & (t <= tmax) & (h2 <= rr)
    if not hit.any():
        return -1, F(np.inf), F(np.inf)
    idx, t, h2 = idx[hit], t[hit], h2[hit]
    j = np.lexsort((idx, t.view(np.uint32)))[0]
    return int(idx[j]), t[j], h2[j]


def _empty(n):
    return np.full(n, -1, dtype=np.int64), np.full(n, np.inf, dtype=F), np.full(n, np.inf, dtype=F)


class Prepared:
    """The sample set of one export, binned into a GRID^3 grid, for several calls of search()."""

    def __init__(self, export, depth, box_min, box_max, rcp=None):
        self.cand = np.nonzero(N.candidates(export, depth, box_min, box_max, rcp))[0]
        self.xyz = tuple(v[self.cand] for v in N._xyz(export[1]))
        if not len(self.cand):
            return
        p = np.stack(self.xyz, axis=1).astype(np.float64)
        lo, hi = p.min(axis=0), p.max(axis=0)
        span = np.where(hi > lo, hi - lo, 1.0)
        cell = np.minimum(((p - lo) / span * GRID).astype(np.int64), GRID - 1)
        cid = (cell[:, 0] * GRID + cell[:, 1]) * GRID + cell[:, 2]
        self.order = np.argsort(cid, kind="stable")
        cid = cid[self.order]
        self.starts = np.concatenate([[0], np.nonzero(np.diff(cid))[0] + 1])
        self.ends = np.concatenate([self.starts[1:], [len(cid)]])
        ps = p[self.order]
        self.lo = np.minimum.reduceat(ps, self.starts, axis=0)       # the bounds of each non-empty cell's samples
        self.hi = np.maximum.reduceat(ps, self.starts, axis=0)


def _cells(prep, o, u, tmin, tmax, radius):
    """The cells whose inflated sample bounds the widened segment crosses (float64), ordered by a lower bound of the t
    of their hits, with that bound; None when the bounds do not hold (overflow)."""
    far = np.sqrt((np.maximum(np.abs(prep.lo - o), np.abs(prep.hi - o)) ** 2).sum(axis=1))
    if not (far.max() < 1e37):
        return None
    slack = far * 1e-5 + 1e-30
    grow = radius * (1 + 1e-5) + slack
    enter = np.full(len(far), -np.inf)
    leave = np.full(len(far), np.inf)
    keep = np.ones(len(far), dtype=bool)
    for a in range(3):
        lo, hi = prep.lo[:, a] - grow - o[a], prep.hi[:, a] + grow - o[a]
        if u[a] == 0:
            keep &= (lo <= 0) & (hi >= 0)
        else:
            s0, s1 = lo / u[a], hi / u[a]
            enter = np.maximum(enter, np.minimum(s0, s1))
            leave = np.minimum(leave, np.maximum(s0, s1))
    keep &= (enter <= leave) & (leave >= tmin - slack) & (enter <= tmax + slack)
    cells = np.nonzero(keep)[0]
    first = (enter - slack)[cells]                          # no hit in the cell has a smaller t
    order = np.argsort(first, kind="stable")
    return cells[order], first[order]


def search(prep, r, radius):
    r = np.asarray(r, dtype=F)
    out = _empty(len(r))
    if not len(prep.cand):
        return out
    u_all, ok = normalise(r), valid(r)
    rr = _radius2(radius)
    for i in np.nonzero(ok)[0]:
        o, u, tmin, tmax = r[i, 0:3], u_all[i], r[i, 3], r[i, 7]
        found = None if np.isinf(rr) else _cells(prep, o.astype(np.float64), u.astype(np.float64), float(tmin), float(tmax),
                                                   float(radius))
        if found is None:
            t, h2 = key(prep.xyz, o, u)
            out[0][i], out[1][i], out[2][i] = _first(prep.cand, t, h2, tmin, tmax, rr)
            continue
        cells, first = found
        best = (-1, F(np.inf), F(np.inf))
        c0 = 0
        while c0 < len(cells):                              # front to back, until no later cell can hold a better hit
            if best[0] >= 0 and float(best[1]) < first[c0]:
                break
            c1 = c0 + 1 + int(np.searchsorted(np.cumsum(prep.ends[cells[c0:]] - prep.starts[cells[c0:]]), GROUP))
            members = prep.order[np.concatenate([np.arange(prep.starts[c], prep.ends[c]) for c in cells[c0:c1]])]
            c0 = c1
            t, h2 = key(tuple(v[members] for v in prep.xyz), o, u)
            idx = np.concatenate([prep.cand[members], [best[0]]]) if best[0] >= 0 else prep.cand[members]
            if best[0] >= 0:
                t, h2 = np.append(t, best[1]), np.append(h2, best[2])
            best = _first(idx, t, h2, tmin, tmax, rr)
        out[0][i], out[1][i], out[2][i] = best
    return out


def brute_force(export, r, radius, depth, box_min, box_max, rcp=None):
    r = np.asarray(r, dtype=F)
    cand = np.nonzero(N.candidates(export, depth, box_min, box_max, rcp))[0]
    xyz = tuple(v[cand] for v in N._xyz(export[1]))
    out = _empty(len(r))
    u_all, ok = normalise(r), valid(r)
    rr = _radius2(radius)
    for i in np.nonzero(ok)[0]:
        t, h2 = key(xyz, r[i, 0:3], u_all[i])
        out[0][i], out[1][i], out[2][i] = _first(cand, t, h2, r[i, 3], r[i, 7], rr)
    return out


def trace(export, r, radius, depth, box_min, box_max, rcp=None):
    return search(Prepared(export, depth, box_min, box_max, rcp), r, radius)


def trace_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, r, radius, depth, box_min, box_max, rcp=None):
    export = R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth)
    return trace(export, r, radius, depth, box_min, box_max, rcp)
