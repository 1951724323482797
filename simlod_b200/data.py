"""Synthetic point streams for the benchmark configurations (BASELINE.md §2, SURVEY.md §8d).

There is no network and no Morro Bay file on the box, so every configuration is generated:
  uniform_cube   config 1: N uniform-random points in a 2^k cube, one batch
  terrain        configs 2/3/5: fBm height field 4800 x 4300 x 300 m emitted in 50 m flight strips
                 (spatially coherent 1 M-point batches, as LiDAR is; the reference's spill buffers
                 rely on that coherence, SURVEY.md §7.3-3)
  shell          config 4: sphere shell in a 4096^3 cube, latitude/longitude tile order
All generators are counter-based (splitmix64 of the point index), so any sub-range can be produced
independently (per batch, per rank) and a CPU check sees exactly the bytes the GPU saw.
"""
import numpy as np

from .api import POINT_DTYPE

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x):
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & _M64
    z = x
    z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _M64
    z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _M64
    return z ^ (z >> np.uint64(31))


def _uniform24(counter):
    """24-bit uniform in [0, 1), exactly representable in float32."""
    return (splitmix64(counter) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)


def _counters(seed, first, count, lanes):
    with np.errstate(over="ignore"):
        base = (np.uint64(seed) << np.uint64(32)) + (np.arange(first, first + count, dtype=np.uint64) * np.uint64(lanes))
    return base


def uniform_cube(n, size=1024.0, seed=42, first=0):
    """Config 1. Cube [0,size)^3 with size a power of two (exact reciprocal on CPU and GPU)."""
    with np.errstate(over="ignore"):
        c = _counters(seed, first, n, 4)
        pts = np.empty(n, dtype=POINT_DTYPE)
        pts["x"] = _uniform24(c) * np.float32(size)
        pts["y"] = _uniform24(c + np.uint64(1)) * np.float32(size)
        pts["z"] = _uniform24(c + np.uint64(2)) * np.float32(size)
        pts["color"] = (splitmix64(c + np.uint64(3)) & np.uint64(0xFFFFFF)).astype(np.uint32) | np.uint32(0xFF000000)
    return pts, (0.0, 0.0, 0.0), (float(size), float(size), float(size))


# ---- terrain (Morro Bay stand-in) -------------------------------------------------------------
TERRAIN_EXTENT = (4800.0, 4300.0, 300.0)
_STRIP_WIDTH = 50.0


def _hash2(ix, iy, seed):
    with np.errstate(over="ignore"):
        k = (ix.astype(np.uint64) * np.uint64(0x9E3779B1)) ^ (iy.astype(np.uint64) * np.uint64(0x85EBCA77)) ^ np.uint64(seed)
    return (splitmix64(k) >> np.uint64(40)).astype(np.float64) * (2.0 ** -24)


def _value_noise(x, y, seed):
    ix, iy = np.floor(x), np.floor(y)
    fx, fy = x - ix, y - iy
    ix, iy = ix.astype(np.int64), iy.astype(np.int64)
    sx, sy = fx * fx * (3 - 2 * fx), fy * fy * (3 - 2 * fy)
    v00, v10 = _hash2(ix, iy, seed), _hash2(ix + 1, iy, seed)
    v01, v11 = _hash2(ix, iy + 1, seed), _hash2(ix + 1, iy + 1, seed)
    return (v00 * (1 - sx) + v10 * sx) * (1 - sy) + (v01 * (1 - sx) + v11 * sx) * sy


def terrain_height(x, y, seed=7):
    h = np.zeros_like(x, dtype=np.float64)
    amp, freq, norm = 1.0, 1.0 / 1600.0, 0.0
    for octave in range(5):
        h += amp * _value_noise(x * freq, y * freq, seed + 101 * octave)
        norm += amp
        amp *= 0.5
        freq *= 2.0
    return (h / norm) * (TERRAIN_EXTENT[2] - 1.0)


def terrain(n_total, first=0, count=None, seed=7):
    """Points first..first+count of an n_total-point scan of the synthetic terrain.

    The scan covers the 4800 x 4300 m area in 96 flight strips of 50 m; within a strip points
    advance along y and scatter across the strip, so consecutive 1 M-point batches cover compact
    patches. z = fBm height + 0.2 m scanner noise; colour = height ramp. boxMin = 0 (the loaders
    translate to the file's min, tools/las2simlod.mjs:130-132)."""
    count = n_total - first if count is None else count
    i = np.arange(first, first + count, dtype=np.uint64)
    num_strips = int(TERRAIN_EXTENT[0] / _STRIP_WIDTH)
    per_strip = -(-n_total // num_strips)
    strip = (i // np.uint64(per_strip)).astype(np.float64)
    t = (i % np.uint64(per_strip)).astype(np.float64) / float(per_strip)
    with np.errstate(over="ignore"):
        c = (np.uint64(seed) << np.uint64(40)) + i * np.uint64(4)
        u0 = _uniform24(c).astype(np.float64)
        u1 = _uniform24(c + np.uint64(1)).astype(np.float64)
        u2 = _uniform24(c + np.uint64(2)).astype(np.float64)
    x = np.minimum((strip + u0) * _STRIP_WIDTH, TERRAIN_EXTENT[0] - 0.01)
    # serpentine flight lines; a few metres of along-track jitter
    along = np.where((strip.astype(np.int64) & 1) == 0, t, 1.0 - t)
    y = np.clip(along * TERRAIN_EXTENT[1] + (u1 - 0.5) * 4.0, 0.0, TERRAIN_EXTENT[1] - 0.01)
    z = np.clip(terrain_height(x, y, seed) + (u2 - 0.5) * 0.4, 0.0, TERRAIN_EXTENT[2] - 0.01)
    pts = np.empty(count, dtype=POINT_DTYPE)
    pts["x"], pts["y"], pts["z"] = x.astype(np.float32), y.astype(np.float32), z.astype(np.float32)
    hn = np.clip(z / TERRAIN_EXTENT[2], 0.0, 1.0)
    r = (40 + 200 * hn).astype(np.uint32)
    g = (90 + 140 * (1.0 - np.abs(hn - 0.5) * 2.0)).astype(np.uint32)
    b = (60 + 120 * (1.0 - hn)).astype(np.uint32)
    pts["color"] = r | (g << np.uint32(8)) | (b << np.uint32(16)) | np.uint32(0xFF000000)
    return pts, (0.0, 0.0, 0.0), TERRAIN_EXTENT


# ---- sphere shell (config 4) --------------------------------------------------------------------
SHELL_CUBE = 4096.0


def shell(n_total, first=0, count=None, seed=1234, tiles_lat=64, tiles_lon=128):
    """Sphere shell R = 1800 +- 0.25 centred in a 4096^3 cube, emitted tile by tile in latitude /
    longitude order (equal-area tiles), so that 1 M-point batches cover compact patches."""
    count = n_total - first if count is None else count
    i = np.arange(first, first + count, dtype=np.uint64)
    num_tiles = tiles_lat * tiles_lon
    per_tile = -(-n_total // num_tiles)
    tile = (i // np.uint64(per_tile)).astype(np.int64)
    tlat, tlon = tile // tiles_lon, tile % tiles_lon
    with np.errstate(over="ignore"):
        c = (np.uint64(seed) << np.uint64(40)) + i * np.uint64(4)
        u0 = _uniform24(c).astype(np.float64)
        u1 = _uniform24(c + np.uint64(1)).astype(np.float64)
        u2 = _uniform24(c + np.uint64(2)).astype(np.float64)
        col = (splitmix64(c + np.uint64(3)) & np.uint64(0xFFFFFF)).astype(np.uint32)
    cz = -1.0 + 2.0 * (tlat + u0) / tiles_lat             # equal-area in z
    phi = 2.0 * np.pi * (tlon + u1) / tiles_lon
    r = 1800.0 + (u2 - 0.5) * 0.5
    s = np.sqrt(np.maximum(0.0, 1.0 - cz * cz))
    ctr = SHELL_CUBE / 2
    pts = np.empty(count, dtype=POINT_DTYPE)
    pts["x"] = (ctr + r * s * np.cos(phi)).astype(np.float32)
    pts["y"] = (ctr + r * s * np.sin(phi)).astype(np.float32)
    pts["z"] = (ctr + r * cz).astype(np.float32)
    pts["color"] = col | np.uint32(0xFF000000)
    return pts, (0.0, 0.0, 0.0), (SHELL_CUBE, SHELL_CUBE, SHELL_CUBE)


def terrain_batches(total_batches, mine, threads=None, seed=7, batch_size=1_000_000):
    """Host copies of the batches `mine` of a (total_batches x batch_size)-point terrain scan (numpy, several threads)."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    n_total = total_batches * batch_size
    threads = threads or min(16, os.cpu_count() or 4)
    with ThreadPoolExecutor(threads) as ex:
        out = list(ex.map(lambda b: terrain(n_total, b * batch_size, batch_size, seed)[0], mine))
    return out, (0.0, 0.0, 0.0), TERRAIN_EXTENT


def batches(points, batch_size=1_000_000):
    for s in range(0, points.shape[0], batch_size):
        yield points[s:s + batch_size]


# ---- LAS files (for the LAS front-end row) ------------------------------------------------------------
LAS_RECORD_BYTES = {0: 20, 1: 28, 2: 26, 3: 34, 5: 63, 7: 36}      # 5: odd record size (waveform packet); 7: LAS 1.4
LAS_RGB_OFFSET = {2: 20, 3: 28, 5: 28, 7: 30}


def las_records(points, fmt=2, scale=(0.001, 0.001, 0.001), offset=(0.0, 0.0, 0.0), wide_colors=True, extra_bytes=0):
    """Raw LAS point records (uint8, n x bytesPerPoint) for 16-byte points: int32 XYZ = round((p - offset) / scale),
    intensity/flags zero, RGB as 16-bit channels (x 257 when wide_colors, as most LAS writers do)."""
    n = points.shape[0]
    bpp = LAS_RECORD_BYTES[fmt] + extra_bytes
    rec = np.zeros((n, bpp), dtype=np.uint8)
    if bpp > LAS_RECORD_BYTES[fmt]:
        rec[:, LAS_RECORD_BYTES[fmt]:] = 0xA5                    # "extra bytes" of the record: anything
    for k, ax in enumerate("xyz"):
        q = np.rint((points[ax].astype(np.float64) - offset[k]) / scale[k]).astype("<i4")
        rec[:, 4 * k:4 * k + 4] = q.view(np.uint8).reshape(n, 4)
    rec[:, 12:14] = (np.arange(n, dtype=np.uint32) & 0xFFFF).astype("<u2").view(np.uint8).reshape(n, 2)     # intensity: anything
    if fmt in LAS_RGB_OFFSET:
        o = LAS_RGB_OFFSET[fmt]
        c = points["color"]
        for k in range(3):
            ch = ((c >> np.uint32(8 * k)) & np.uint32(0xFF)).astype(np.uint32)
            ch16 = (ch * 257 if wide_colors else ch).astype("<u2")
            rec[:, o + 2 * k:o + 2 * k + 2] = ch16.view(np.uint8).reshape(n, 2)
    return rec


LAS_HEADER_SIZE = {(1, 2): 227, (1, 3): 235, (1, 4): 375}


def write_las(path, points, fmt=2, scale=(0.001, 0.001, 0.001), offset=(0.0, 0.0, 0.0), wide_colors=True, extra_bytes=0,
              version=(1, 2), vlr_bytes=0):
    """Minimal LAS file with the header fields the reference reads (LasLoader.h:21-55). version (1, 2) writes the 227-byte
    1.2 header, (1, 3) the 235-byte 1.3 header, (1, 4) the 375-byte 1.4 header with the 64-bit point count at byte 247
    and a legacy count of 0. `vlr_bytes` zero bytes between header and records stand for variable length records, so
    that offset_to_point_data = header size + vlr_bytes."""
    import struct
    rec = las_records(points, fmt, scale, offset, wide_colors, extra_bytes)
    n, bpp = rec.shape
    size = LAS_HEADER_SIZE[tuple(version)]
    hdr = bytearray(size + vlr_bytes)
    hdr[0:4] = b"LASF"
    hdr[24], hdr[25] = version
    struct.pack_into("<H", hdr, 94, size)
    struct.pack_into("<I", hdr, 96, size + vlr_bytes)
    hdr[104] = fmt
    struct.pack_into("<H", hdr, 105, bpp)
    struct.pack_into("<I", hdr, 107, n if tuple(version) != (1, 4) else 0)
    if tuple(version) == (1, 4):
        struct.pack_into("<Q", hdr, 247, n)
    struct.pack_into("<3d", hdr, 131, *scale)
    struct.pack_into("<3d", hdr, 155, *offset)
    mx = [float(points[a].max()) for a in "xyz"] if n else [0.0] * 3
    mn = [float(points[a].min()) for a in "xyz"] if n else [0.0] * 3
    struct.pack_into("<6d", hdr, 179, mx[0], mn[0], mx[1], mn[1], mx[2], mn[2])
    with open(path, "wb") as f:
        f.write(bytes(hdr))
        f.write(rec.tobytes())
    return rec


def write_simlod(path, points, box_min, box_max):
    """The .simlod container (tools/las2simlod.mjs:95-101,130-132): 6 x f32 (min, max) then 16-byte points, already
    translated so that the box minimum is the origin."""
    import struct
    with open(path, "wb") as f:
        f.write(struct.pack("<6f", *[float(v) for v in box_min], *[float(v) for v in box_max]))
        f.write(np.ascontiguousarray(points).tobytes())
