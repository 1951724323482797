"""TEST INFRASTRUCTURE — CPU restatement of the reference's reload() for a list of point-cloud files
(main_progressive_octree.cpp:644-773) and of the loader's per-batch work (:855-941), from the files' header fields:
the box, the translation and the batch list, each batch as (file, first, count, kind); and the points each batch
becomes, which is what simlod_insert_files must insert.

LAS headers are read as the reference's loadHeader reads them (LasLoader.h:21-55): through the reference's own code
(oracle/_ref/libref_las.so, `ref_las_header`) where it has been built, else by `las_header` below, whose fields the
CPU tests pin against the reference."""
import ctypes as C
import os
import struct

import numpy as np

import oracle

MAX_BATCH_SIZE = 1_000_000          # main.cpp:37


def las_header(path):
    """loadHeader (LasLoader.h:21-55): the fields at their byte offsets; the point count at 107 (u32) for versions
    1.0-1.3, else at 247 (u64) (:31-35)."""
    with open(path, "rb") as f:
        b = f.read(375).ljust(375, b"\0")
    major, minor = b[24], b[25]
    h = {"version_major": major, "version_minor": minor, "header_size": struct.unpack_from("<H", b, 94)[0],
         "offset_to_point_data": struct.unpack_from("<I", b, 96)[0], "format": b[104],
         "bytes_per_point": struct.unpack_from("<H", b, 105)[0],
         "num_points": struct.unpack_from("<I", b, 107)[0] if (major == 1 and minor <= 3) else struct.unpack_from("<Q", b, 247)[0],
         "scale": struct.unpack_from("<3d", b, 131), "offset": struct.unpack_from("<3d", b, 155),
         "min": tuple(struct.unpack_from("<d", b, o)[0] for o in (187, 203, 219)),
         "max": tuple(struct.unpack_from("<d", b, o)[0] for o in (179, 195, 211))}
    return h


def ref_las_header(path):
    """The reference's own loadHeader (oracle/_ref/libref_las.so): the fields LasHeader keeps, or None where the
    reference loader has not been built."""
    L = oracle.ref_las()
    if L is None:
        return None
    n, bpp, fmt, off = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
    arr = [(C.c_double * 3)() for _ in range(4)]
    L.ref_las_header(path.encode(), C.byref(n), C.byref(bpp), C.byref(fmt), C.byref(off), *arr)
    return {"num_points": n.value, "bytes_per_point": bpp.value, "format": fmt.value, "offset_to_point_data": off.value,
            "scale": tuple(arr[0]), "offset": tuple(arr[1]), "min": tuple(arr[2]), "max": tuple(arr[3])}


def header(path):
    h = las_header(path)
    ref = ref_las_header(path)
    if ref is not None:
        h.update(ref)
    return h


def is_las(path):
    return path.lower().endswith(".las")          # iEndsWith(path, "las"), main.cpp:693


def reload(paths):
    """(box_min, box_max, translation, batches) of reload() for `paths` in list order:
      box_min / box_max  float32[3]: the union of float(header.min / max) of the LAS files (main.cpp:700-709) and the
                         six header floats of the .simlod files (:724-733)
      translation        float64[3]: double of the negated float box minimum (main.cpp:868)
      batches            [(path, first, count, kind)], kind "las" or "simlod": ceil(n / 1 000 000) batches per file, the
                         last one partial (main.cpp:711-720, 737-745)
    The uniforms then hold boxMin = 0 and boxMax = box_max - box_min in float (main.cpp:312-313, 763-765)."""
    bmin = np.full(3, np.inf, np.float32)
    bmax = np.full(3, -np.inf, np.float32)
    batches = []
    for path in paths:
        if is_las(path):
            h = header(path)
            n, kind = h["num_points"], "las"
            lo, hi = np.float32(h["min"]), np.float32(h["max"])
        else:
            hdr = np.fromfile(path, dtype="<f4", count=6)
            n, kind = (os.path.getsize(path) - 24) // 16, "simlod"
            lo, hi = hdr[:3], hdr[3:]
        bmin, bmax = np.minimum(bmin, lo), np.maximum(bmax, hi)
        for first in range(0, n, MAX_BATCH_SIZE):
            batches.append((path, first, min(n - first, MAX_BATCH_SIZE), kind))
    translation = (-bmin).astype(np.float64)
    return bmin, bmax, translation, batches


def batch_points(batch, translation):
    """The 16-byte points one batch becomes: LAS records decoded by oracle.decode_las with the union translation
    (loadLasNative, main.cpp:866-869; alpha 0xff as the device decode writes it), .simlod points copied as they are
    stored, untranslated (main.cpp:927-941)."""
    path, first, count, kind = batch
    if kind == "simlod":
        return np.fromfile(path, dtype=oracle.POINT_DTYPE, count=count, offset=24 + 16 * first)
    h = header(path)
    bpp = h["bytes_per_point"]
    rec = np.fromfile(path, dtype=np.uint8, count=count * bpp, offset=h["offset_to_point_data"] + first * bpp)
    pts = oracle.decode_las(rec, count, bpp, h["format"], h["scale"], h["offset"], translation)
    return pts


# ---- the reference's results, stored -------------------------------------------------------------------------------
# What the reference's own loader computes on the test inputs, kept as digests in tests/golden/las_files_reference.json
# so that the comparison runs where the reference has not been built (a checkout without the original sources). Where it has been built, the
# reference runs live and must agree with what is stored; SIMLOD_RECORD_GOLDEN=1 rewrites the stored values instead.
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "las_files_reference.json")
_stored = None


def reference(key, run):
    import json
    global _stored
    if _stored is None:
        _stored = json.load(open(GOLDEN)) if os.path.exists(GOLDEN) else {}
    if oracle.ref_las() is None:
        assert key in _stored, "no stored reference result for %r in %s" % (key, GOLDEN)
        return _stored[key]
    value = json.loads(json.dumps(run()))
    if os.environ.get("SIMLOD_RECORD_GOLDEN"):
        _stored[key] = value
        with open(GOLDEN, "w") as f:
            json.dump(_stored, f, indent=1, sort_keys=True)
    elif key in _stored:
        assert _stored[key] == value, "reference result for %r differs from the stored one" % key
    return value


# ---- inputs shared by the CPU and GPU tests ------------------------------------------------------------------------
SHIFT = (1000.0, 2000.0, 50.0)          # the tiles sit away from the origin, so the translation is not trivial
SCALE = (0.001, 0.001, 0.001)
OFFSET = (1000.0, 2000.0, 0.0)
# name: (format, extra bytes, version, VLR bytes): 2.5 M terrain points as one LAS file
FORMAT_CASES = {"fmt2": (2, 0, (1, 2), 0), "fmt3": (3, 0, (1, 2), 0), "fmt0": (0, 0, (1, 3), 0), "fmt5": (5, 0, (1, 3), 0),
                "fmt7": (7, 0, (1, 4), 54), "fmt3_extra1": (3, 1, (1, 4), 0)}
FORMAT_CASE_POINTS = 2_500_000


def shifted_terrain(n_total, first=0, count=None, shift=SHIFT):
    from simlod_b200 import data
    pts, _, _ = data.terrain(n_total, first, count)
    for k, ax in enumerate("xyz"):
        pts[ax] = pts[ax] + np.float32(shift[k])
    return pts


def write_format_case(directory, name):
    from simlod_b200 import data
    fmt, extra, version, vlr = FORMAT_CASES[name]
    path = os.path.join(str(directory), name + ".las")
    data.write_las(path, shifted_terrain(FORMAT_CASE_POINTS), fmt=fmt, scale=SCALE, offset=OFFSET, extra_bytes=extra,
                   version=version, vlr_bytes=vlr)
    return path


def check_batches_against_reference(key, paths):
    """The points of every LAS batch of reload(paths), as batch_points decodes them, against the reference's own
    loadLasNative (oracle.ref_las_load) with the same translation: xyz bit for bit, colour under the RGB mask for the
    formats with RGB. Returns the restatement (box_min, box_max, translation, batches)."""
    import reference_golden as golden
    restated = reload(paths)
    translation, batches = restated[2], restated[3]
    for k, b in enumerate(batches):
        if b[3] != "las":
            continue
        rgb = header(b[0])["format"] in (2, 3, 5, 7)
        got = golden.points(batch_points(b, translation), rgb)
        want = reference("%s/batch%d" % (key, k), lambda: golden.points(oracle.ref_las_load(b[0], b[1], b[2], translation), rgb))
        assert got == want, (key, k)
    return restated
