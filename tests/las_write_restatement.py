"""TEST INFRASTRUCTURE — numpy restatement of the LAS files SimLOD.write_las writes (DESIGN.md §9.13), from the samples
and the parameters alone; it does not use the package's writer.

  q       per axis, in IEEE double: rint(((double(p) + translation) - offset) / scale), half to even; a sample with a
          non-finite coordinate or a q outside int32 is invalid, and any invalid sample refuses the whole file
  header  LAS 1.2, 227 bytes, no VLRs, point format 2, record length 26, generating software "simlod_b200", creation
          day and year 0, legacy count n, points by return [n, 0, 0, 0, 0], scale and offset as given, and per axis
          max = double(q_max) * scale + offset, min likewise (0 when n = 0)
  record  int32 X, Y, Z = q; intensity 0; flags 0x09; classification, scan angle, user data, point source ID 0;
          R, G, B = 257 * colour bits 0-7, 8-15, 16-23"""
import struct

import numpy as np

POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("color", "<u4")])
RECORD_DTYPE = np.dtype([("xyz", "<i4", (3,)), ("intensity", "<u2"), ("flags", "u1"), ("classification", "u1"),
                         ("scan_angle", "i1"), ("user_data", "u1"), ("point_source", "<u2"), ("rgb", "<u2", (3,))])
assert RECORD_DTYPE.itemsize == 26
HEADER_BYTES = 227
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


def params(scale=0.001, offset=None, translation=(0.0, 0.0, 0.0)):
    """(scale, offset, translation) as float64[3] each, with write_las's defaults: a scalar scale applies to every axis,
    offset None is the translation."""
    s = np.full(3, float(scale)) if np.ndim(scale) == 0 else np.asarray(scale, dtype=np.float64)
    t = np.asarray(translation, dtype=np.float64)
    o = t.copy() if offset is None else np.asarray(offset, dtype=np.float64)
    return s, o, t


def as_points(samples):
    a = np.asarray(samples)
    if a.dtype != POINT_DTYPE:
        a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1).view(POINT_DTYPE)
    return a


def quantise(samples, scale, offset, translation):
    """(q int64 (n, 3), valid bool (n,)) by the file contract's rule."""
    pts = as_points(samples)
    p = np.stack([pts["x"], pts["y"], pts["z"]], axis=1).astype(np.float64)
    with np.errstate(all="ignore"):
        r = np.rint(((p + translation) - offset) / scale)
    valid = np.all((r >= INT32_MIN) & (r <= INT32_MAX), axis=1)          # NaN and inf fail both tests
    q = np.where(valid[:, None], r, 0.0).astype(np.int64)
    return q, valid


def records(q, color):
    rec = np.zeros(len(q), dtype=RECORD_DTYPE)
    rec["xyz"] = q.astype(np.int32)
    rec["flags"] = 0x09
    c = np.asarray(color, dtype=np.uint32)
    for k in range(3):
        rec["rgb"][:, k] = (((c >> np.uint32(8 * k)) & np.uint32(0xFF)) * np.uint32(257)).astype(np.uint16)
    return rec


def bounds(q, scale, offset):
    """(min, max) float64[3] of the header: double(q) * scale + offset, multiply then add."""
    if len(q) == 0:
        return np.zeros(3), np.zeros(3)
    return q.min(axis=0).astype(np.float64) * scale + offset, q.max(axis=0).astype(np.float64) * scale + offset


def header(n, scale, offset, mn, mx):
    h = bytearray(HEADER_BYTES)
    h[0:4] = b"LASF"
    h[24], h[25] = 1, 2
    h[58:58 + 11] = b"simlod_b200"
    struct.pack_into("<H", h, 94, HEADER_BYTES)
    struct.pack_into("<I", h, 96, HEADER_BYTES)
    struct.pack_into("<I", h, 100, 0)
    h[104] = 2
    struct.pack_into("<H", h, 105, RECORD_DTYPE.itemsize)
    struct.pack_into("<I", h, 107, n)
    struct.pack_into("<5I", h, 111, n, 0, 0, 0, 0)
    struct.pack_into("<3d", h, 131, *scale)
    struct.pack_into("<3d", h, 155, *offset)
    struct.pack_into("<6d", h, 179, mx[0], mn[0], mx[1], mn[1], mx[2], mn[2])
    return bytes(h)


def file_bytes(samples, scale=0.001, offset=None, translation=(0.0, 0.0, 0.0)):
    """(file bytes, first invalid index): the bytes are None when a sample is invalid, the index None when none is."""
    s, o, t = params(scale, offset, translation)
    pts = as_points(samples)
    if len(pts) > 2 ** 32 - 1:
        raise ValueError("a LAS 1.2 file holds at most 2^32 - 1 points")
    q, valid = quantise(pts, s, o, t)
    if not valid.all():
        return None, int(np.argmin(valid))
    mn, mx = bounds(q, s, o)
    return header(len(pts), s, o, mn, mx) + records(q, pts["color"]).tobytes(), None


def decode(buf):
    """(header fields dict, records RECORD_DTYPE) of a point-format-2 file written by the rules above."""
    n = struct.unpack_from("<I", buf, 107)[0]
    h = {"signature": buf[0:4], "version": (buf[24], buf[25]), "software": buf[58:90], "day_year": struct.unpack_from("<2H", buf, 90),
         "header_size": struct.unpack_from("<H", buf, 94)[0], "offset_to_point_data": struct.unpack_from("<I", buf, 96)[0],
         "num_vlrs": struct.unpack_from("<I", buf, 100)[0], "format": buf[104], "bytes_per_point": struct.unpack_from("<H", buf, 105)[0],
         "num_points": n, "by_return": struct.unpack_from("<5I", buf, 111), "scale": struct.unpack_from("<3d", buf, 131),
         "offset": struct.unpack_from("<3d", buf, 155), "max": struct.unpack_from("<6d", buf, 179)[0::2],
         "min": struct.unpack_from("<6d", buf, 179)[1::2]}
    rec = np.frombuffer(buf, dtype=RECORD_DTYPE, count=n, offset=HEADER_BYTES)
    return h, rec
