"""CPU restatement of kernel_render's bounding-box overlay (Uniforms::showBoundingBox): the line list the reference
builds and the line rasteriser it runs over it. Citations are to the reference's modules/progressive_octree/.

- Lines (render.cu:1195-1227, 637-688; rasterization.cuh:5-47): 8 frustum edges (colour 0x000000ff), NDC corners
  (+-1, +-1, -1) and (+-1, +-1, 0.99995) through transformInv_updateBound; then for every drawn node the 12 edges of its
  box (colour 0x0000ff00), centre cubeMin + float(X + 0.5f) * scale, corners centre -+ scale / 2. The reference appends
  each box four times (identical: s = 1 exactly), 48 lines per node; `reference_line_count` counts those.
- Rasterising (rasterization.cuh:90-183, math.cuh:22-152): endpoints outside the frustum of `transform` move along the
  normalised direction to the farthest finite positive plane distance (-Infinity when there is none); steps =
  clamp(length of the screen-space line, 0, 400); u runs 0, stepSize, ... while u <= 1 as a float recurrence; each step
  interpolates NDC x, y and the linear depth in double and does atomicMin(fb[pixel], depth bits << 32 | colour).

The device computes rcp, sqrt and rsqrt with MUFU approximations, the CPU correctly rounded, so `steps` and every depth
can differ in the last bits and a step can land one pixel over: compare against the device by coverage, not bits."""
import numpy as np

FRUSTUM_COLOR = 0x000000FF
BOX_COLOR = 0x0000FF00
FRUSTUM_LINES = 8
BOX_LINES = 12
# The reference's Lines list holds 1 000 000 vertices: 8 + 48 |D| lines fit while |D| <= 10 416 (structures.cuh:45-51,
# render.cu:1117-1120). Above that its vertices run into the framebuffer.
REFERENCE_VERTEX_CAPACITY = 1_000_000
REFERENCE_CAPACITY_NODES = (REFERENCE_VERTEX_CAPACITY // 2 - FRUSTUM_LINES) // 48
INF_DEPTH = np.uint64(0x7F800000)

f32, f64 = np.float32, np.float64


def reference_line_count(num_drawn):
    """Lines in the reference's list for |D| drawn nodes: 8 + 48 |D|."""
    return FRUSTUM_LINES + 48 * int(num_drawn)


def overlay_line_count(num_drawn):
    """Distinct lines drawn: 8 + 12 |D|."""
    return FRUSTUM_LINES + BOX_LINES * int(num_drawn)


def uniforms_from_bytes(b):
    """The fields of SimlodUniforms (include/simlod_abi.h) that the overlay reads."""
    b = bytes(b)
    fl = np.frombuffer(b[:448], dtype="<f4")
    return {"width": float(fl[0]), "height": float(fl[1]),
            "transform": fl[52:68].reshape(4, 4).copy(), "transformInv_updateBound": fl[84:100].reshape(4, 4).copy(),
            "boxMin": fl[106:109].copy(), "boxMax": fl[109:112].copy(), "showBoundingBox": b[448]}


def _fma(a, b, c):
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def _row_dot(r, x, y, z):
    """mat4 row * (x, y, z, 1) as the reference contracts it: w + fma(z, r.z, fma(x, r.x, y * r.y))."""
    return (f32(r[3]) + _fma(z, r[2], _fma(x, r[0], f32(y) * f32(r[1])))).astype(f32)


def _dot3(ax, ay, az, bx, by, bz):
    return _fma(az, bz, _fma(ax, bx, (np.asarray(ay, f32) * np.asarray(by, f32)).astype(f32)))


def cube_size(u):
    bs = (u["boxMax"] - u["boxMin"]).astype(f32)
    return f32(max(bs[0], bs[1], bs[2]))


def frustum_lines(u):
    """(starts, ends) of the 8 frustum edges (render.cu:1197-1223)."""
    fend = f32(0.99995)
    ti = u["transformInv_updateBound"]
    pairs = [((1, 1, -1), (1, 1, fend)), ((1, -1, -1), (1, -1, fend)), ((-1, 1, -1), (-1, 1, fend)), ((-1, -1, -1), (-1, -1, fend)),
             ((-1, -1, fend), (1, -1, fend)), ((-1, 1, fend), (1, 1, fend)), ((-1, -1, fend), (-1, 1, fend)), ((1, -1, fend), (1, 1, fend))]

    def project(c):
        x, y, z = (f32(v) for v in c)
        rw = f32(1.0) / _row_dot(ti[3], x, y, z)
        return [f32(_row_dot(ti[k], x, y, z) * rw) for k in range(3)]
    with np.errstate(all="ignore"):
        s = np.array([project(a) for a, _ in pairs], dtype=f32)
        e = np.array([project(b) for _, b in pairs], dtype=f32)
    return s, e


# start and end corner of each of drawBoundingBox's 12 edges, bits x = 4, y = 2, z = 1 (rasterization.cuh:25-47)
EDGE_FROM = (0, 4, 6, 2, 1, 5, 7, 3, 4, 6, 2, 0)
EDGE_TO = (4, 6, 2, 0, 5, 7, 3, 1, 5, 7, 3, 1)


def box_lines(u, lxyz):
    """(starts, ends) of the 12 box edges of every node (level, X, Y, Z) in `lxyz` (render.cu:646-687)."""
    lxyz = np.asarray(lxyz, dtype=np.int64).reshape(-1, 4)
    n = len(lxyz)
    cs = cube_size(u)
    scale = (cs * np.exp2(-lxyz[:, 0].astype(f32))).astype(f32)
    half = (scale * f32(0.5)).astype(f32)
    centre = np.stack([_fma(scale, (lxyz[:, 1 + i].astype(f32) + f32(0.5)).astype(f32), u["boxMin"][i]) for i in range(3)], axis=1)
    mn = (centre - half[:, None]).astype(f32)
    mx = (centre + half[:, None]).astype(f32)

    def corner(c):
        return np.stack([np.where(c & 4, mx[:, 0], mn[:, 0]), np.where(c & 2, mx[:, 1], mn[:, 1]), np.where(c & 1, mx[:, 2], mn[:, 2])], axis=1)
    s = np.stack([corner(c) for c in EDGE_FROM], axis=1).reshape(n * BOX_LINES, 3)
    e = np.stack([corner(c) for c in EDGE_TO], axis=1).reshape(n * BOX_LINES, 3)
    return s.astype(f32), e.astype(f32)


def line_list(u, lxyz):
    """The distinct lines of a frame: (starts, ends, colours), frustum first, then 12 per drawn node."""
    fs, fe = frustum_lines(u)
    bs, be = box_lines(u, lxyz)
    colors = np.concatenate([np.full(len(fs), FRUSTUM_COLOR, np.uint64), np.full(len(bs), BOX_COLOR, np.uint64)])
    return np.concatenate([fs, bs]), np.concatenate([fe, be]), colors


def frustum_planes(t):
    """Frustum::fromWorldViewProj (math.cuh:66-106): rows[3] -+ rows[0..2], normalised; (6, 4) normal and constant."""
    t = np.asarray(t, f32)
    raw = [t[3] - t[0], t[3] + t[0], t[3] + t[1], t[3] - t[1], t[3] - t[2], t[3] + t[2]]
    out = []
    with np.errstate(all="ignore"):
        for p in raw:
            p = p.astype(f32)
            inv = f32(1.0) / np.sqrt(_dot3(p[0], p[1], p[2], p[0], p[1], p[2]))
            out.append((p * inv).astype(f32))
    return np.array(out, dtype=f32)


def _contains(planes, p):
    inside = np.ones(len(p), dtype=bool)
    for q in planes:
        d = _dot3(q[0], q[1], q[2], p[:, 0], p[:, 1], p[:, 2])
        inside &= ~(q[3] < -d)
    return inside


def _intersect(planes, o, d):
    """Frustum::intersectRay (math.cuh:108-137): o + d * farthest."""
    farthest = np.full(len(o), -np.inf, dtype=f32)
    for q in planes:
        den = _dot3(q[0], q[1], q[2], d[:, 0], d[:, 1], d[:, 2])
        v = (q[3] + _dot3(q[0], q[1], q[2], o[:, 0], o[:, 1], o[:, 2])).astype(f32)
        t = (v * -(f32(1.0) / den)).astype(f32)
        dist = np.where(den < 0, np.inf, np.where(den == 0, np.where(v == 0, 0.0, np.inf), np.where(t >= 0, t, np.inf))).astype(f32)
        ok = (dist > 0) & (dist != np.inf)
        farthest = np.where(ok, np.fmax(farthest, dist), farthest).astype(f32)
    return np.stack([_fma(d[:, i], farthest, o[:, i]) for i in range(3)], axis=1)


def _d2i(x):
    """cvt.rzi.s32.f64: truncate, saturate, NaN -> 0."""
    x = np.where(np.isnan(x), 0.0, np.clip(x, -2147483648.0, 2147483647.0))
    return np.trunc(x).astype(np.int64)


MAX_STEPS = 403       # stepSize >= 1 / 400: u <= 1 holds for at most 401 values (402 with rounding), one more to see the end


def rasterize(u, starts, ends, colors, width, height):
    """rasterizeLines: (pixel index, 64-bit value) of every step drawn."""
    starts = np.array(starts, dtype=f32).reshape(-1, 3)
    ends = np.array(ends, dtype=f32).reshape(-1, 3)
    colors = np.asarray(colors, dtype=np.uint64)
    if len(starts) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.uint64)
    t = np.asarray(u["transform"], f32)
    planes = frustum_planes(t)
    with np.errstate(all="ignore"):
        d = (ends - starts).astype(f32)
        r = (f32(1.0) / np.sqrt(_dot3(d[:, 0], d[:, 1], d[:, 2], d[:, 0], d[:, 1], d[:, 2]))).astype(f32)
        d = (d * r[:, None]).astype(f32)
        s_in, e_in = _contains(planes, starts), _contains(planes, ends)
        starts = np.where(s_in[:, None], starts, _intersect(planes, starts, d))
        ends = np.where(e_in[:, None], ends, _intersect(planes, ends, (-d).astype(f32)))

        def proj(p):
            w = _row_dot(t[3], p[:, 0], p[:, 1], p[:, 2])
            rw = (f32(1.0) / w).astype(f32)
            return ((_row_dot(t[0], p[:, 0], p[:, 1], p[:, 2]) * rw).astype(f32), (_row_dot(t[1], p[:, 0], p[:, 1], p[:, 2]) * rw).astype(f32), w)
        xs, ys, ws = proj(starts)
        xe, ye, we = proj(ends)
        fw, fh = f32(width), f32(height)
        sdx = _fma(fw, _fma(xe, 0.5, 0.5), -(fw * _fma(xs, 0.5, 0.5)).astype(f32))
        sdy = _fma(fh, _fma(ye, 0.5, 0.5), -(fh * _fma(ys, 0.5, 0.5)).astype(f32))
        length = np.sqrt((f32(0.0) + _fma(sdx, sdx, (sdy * sdy).astype(f32))).astype(f32))
        steps = np.fmax(f32(0.0), np.fmin(length, f32(400.0))).astype(f32)
        step = (f32(1.0) / steps).astype(f32)
        uu = np.empty((len(starts), MAX_STEPS), dtype=f32)
        uu[:, 0] = 0
        uu[:, 1:] = step[:, None]
        uu = np.add.accumulate(uu, axis=1, dtype=f32)                   # the serial float recurrence u += stepSize
        assert (~(uu[:, -1] <= 1)).all(), "more steps than MAX_STEPS"
        take = uu <= 1
        line = np.repeat(np.arange(len(starts)), take.sum(axis=1))     # u increases: the steps taken are a prefix
        uk = uu[take]
        omu = 1.0 - uk.astype(f64)
        nx = (xs[line].astype(f64) * omu + (xe[line] * uk).astype(f32).astype(f64)).astype(f32)
        ny = (ys[line].astype(f64) * omu + (ye[line] * uk).astype(f32).astype(f64)).astype(f32)
        depth = (ws[line].astype(f64) * omu + (we[line] * uk).astype(f32).astype(f64)).astype(f32)
        keep = ~((nx < -1) | (nx > 1) | (ny < -1) | (ny > 1))
        x = _d2i(f64(width) * (nx.astype(f64) * 0.5 + 0.5))
        y = _d2i(f64(height) * (ny.astype(f64) * 0.5 + 0.5))
    x = np.clip(x, 0, width - 1)
    y = np.clip(y, 0, height - 1)
    pixel = (x + width * y)[keep]
    value = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | colors[line]
    return pixel, value[keep]


def overlay_frame(u, lxyz, width, height, fb=None):
    """The overlay drawn over `fb` (a cleared frame when None): every step's atomicMin."""
    if fb is None:
        fb = np.full(width * height, (INF_DEPTH << np.uint64(32)) | np.uint64(0x00332211), dtype=np.uint64)
    fb = np.array(fb, dtype=np.uint64).reshape(-1)
    s, e, c = line_list(u, lxyz)
    for k in range(0, len(s), LINES_PER_PASS):
        pixel, value = rasterize(u, s[k:k + LINES_PER_PASS], e[k:k + LINES_PER_PASS], c[k:k + LINES_PER_PASS], width, height)
        np.minimum.at(fb, pixel, value)
    return fb


LINES_PER_PASS = 16384        # host memory of one rasterize() call: lines x MAX_STEPS


def drawn_from_canon_flags(records, flags):
    """The LOD cut of a frame of oracle.Canon.render, from its flags (canonical order): a visible node that is large and a
    leaf, or not large below a large parent (render.cu:906-933). Returns (level, X, Y, Z) rows."""
    visible, large = flags[:, 0] != 0, flags[:, 1] != 0
    index = {(int(r["level"]), int(r["X"]), int(r["Y"]), int(r["Z"])): k for k, r in enumerate(records)}
    out = []
    for k, r in enumerate(records):
        if not visible[k]:
            continue
        level, x, y, z = int(r["level"]), int(r["X"]), int(r["Y"]), int(r["Z"])
        if large[k]:
            drawn = bool(r["isLeaf"])
        else:
            parent = index.get((level - 1, x >> 1, y >> 1, z >> 1))
            drawn = level > 0 and parent is not None and bool(large[parent])
        if drawn:
            out.append((level, x, y, z))
    return np.array(out, dtype=np.int64).reshape(-1, 4)


def canon_render(canon, uniforms_bytes, width, height):
    """oracle.Canon.render (the CPU model of kernel_render's draw, which does not draw the overlay) with the overlay drawn
    over its frame when the uniforms set showBoundingBox, as kernel_render does before EDL. Same return values."""
    fb, rs, flags = canon.render(uniforms_bytes, width, height)
    u = uniforms_from_bytes(uniforms_bytes)
    if u["showBoundingBox"]:
        fb = overlay_frame(u, drawn_from_canon_flags(canon.records, flags), width, height, fb).reshape(height, width)
    return fb, rs, flags


def coverage(fb):
    """Pixels a line was drawn into, on a frame without samples: every finite depth."""
    return (np.asarray(fb, dtype=np.uint64).reshape(-1) >> np.uint64(32)) != INF_DEPTH
