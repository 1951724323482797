"""CPU-only checks of the file-list front end (simlod_insert_files): the LAS header reader against the reference's
loadHeader, every rejection of the validation pass, and the reload() restatement (tests/files_restatement.py) on
hand-computed cases. Rejections are checked with a null context: the list is validated before the context is used."""
import ctypes as C
import os

import numpy as np
import pytest

import files_restatement as fr
import oracle
from simlod_b200 import api, data, read_las_header, SimlodError

SIMLOD_ERR_INVALID = -2


def insert_files_no_context(paths):
    """simlod_insert_files with a null context: (return code, last error)."""
    lib = api.load_library()
    arr = (C.c_char_p * max(1, len(paths)))(*[os.fsencode(str(p)) for p in paths])
    rc = lib.simlod_insert_files(None, arr, len(paths), 4, 0, None, None, None)
    return rc, lib.simlod_last_error().decode()


# (version, format, extra bytes, VLR bytes): 1.2 / 1.3 / 1.4 headers, the formats the decoder colours and two it does
# not, odd record sizes, offset_to_point_data 227, 235, 375 and 375 + 54
HEADER_CASES = [((1, 2), 2, 0, 0), ((1, 2), 0, 0, 0), ((1, 2), 1, 0, 0), ((1, 3), 3, 0, 0), ((1, 3), 5, 0, 0),
                ((1, 4), 7, 0, 0), ((1, 4), 7, 0, 54), ((1, 2), 2, 3, 0), ((1, 4), 3, 1, 54), ((1, 2), 0, 0, 100)]


@pytest.mark.parametrize("version,fmt,extra,vlr", HEADER_CASES)
def test_read_las_header_matches_reference_loadheader(tmp_path, version, fmt, extra, vlr):
    pts = fr.shifted_terrain(12_345)
    path = str(tmp_path / "h.las")
    data.write_las(path, pts, fmt=fmt, scale=(0.001, 0.002, 0.0005), offset=(1000.0, 2000.0, 1.5), extra_bytes=extra,
                   version=version, vlr_bytes=vlr)
    got = read_las_header(path).as_dict()
    assert got == fr.las_header(path)
    assert got["num_points"] == 12_345 and got["offset_to_point_data"] == data.LAS_HEADER_SIZE[version] + vlr
    assert (got["version_major"], got["version_minor"]) == version and got["bytes_per_point"] == data.LAS_RECORD_BYTES[fmt] + extra
    keys = ("num_points", "bytes_per_point", "format", "offset_to_point_data", "scale", "offset", "min", "max")
    want = fr.reference("header/%d.%d/fmt%d/extra%d/vlr%d" % (version + (fmt, extra, vlr)),
                        lambda: {k: list(v) if isinstance(v, tuple) else v for k, v in fr.ref_las_header(path).items()})
    assert {k: list(got[k]) if isinstance(got[k], tuple) else got[k] for k in keys} == want


def test_write_las_default_output_is_the_las_1_2_file(tmp_path):
    pts = fr.shifted_terrain(1000)
    a, b = str(tmp_path / "a.las"), str(tmp_path / "b.las")
    data.write_las(a, pts, fmt=3)
    data.write_las(b, pts, fmt=3, version=(1, 2), vlr_bytes=0)
    raw = open(a, "rb").read()
    assert raw == open(b, "rb").read() and len(raw) == 227 + 1000 * 34 and raw[94:96] == b"\xe3\x00"


def test_read_las_header_rejects_files_that_are_not_las(tmp_path):
    for name, content in (("none.las", None), ("text.las", b"hello world" * 40), ("short.las", b"LASF" + bytes(100))):
        p = tmp_path / name
        if content is not None:
            p.write_bytes(content)
        with pytest.raises(SimlodError) as e:
            read_las_header(str(p))
        assert e.value.code == SIMLOD_ERR_INVALID and name in str(e.value)


def las_file(path, n=1000, **kw):
    data.write_las(str(path), fr.shifted_terrain(max(n, 1))[:n], **kw)
    return str(path)


def test_every_rejection_names_the_file(tmp_path):
    good = las_file(tmp_path / "good.las")
    sml = str(tmp_path / "good.simlod")
    data.write_simlod(sml, fr.shifted_terrain(10), (0, 0, 0), (1, 1, 1))
    rc, msg = insert_files_no_context([])
    assert rc == SIMLOD_ERR_INVALID and "empty" in msg
    cases = []
    cases.append(("missing", str(tmp_path / "missing.las"), "does not exist"))
    p = tmp_path / "scan.xyz"; p.write_bytes(b"1 2 3\n")
    cases.append(("extension", str(p), "unsupported file type"))
    p = tmp_path / "scan.LAZ"; p.write_bytes(open(good, "rb").read())
    cases.append(("laz", str(p), "LAZ is not supported"))
    p = tmp_path / "nosig.las"; p.write_bytes(b"XXXX" + open(good, "rb").read()[4:])
    cases.append(("signature", str(p), "LASF"))
    p = tmp_path / "bpp.las"; raw = bytearray(open(good, "rb").read()); raw[105:107] = (11).to_bytes(2, "little")
    p.write_bytes(bytes(raw))
    cases.append(("record size", str(p), "record size 11"))
    p = tmp_path / "fmt.las"; raw = bytearray(open(las_file(tmp_path / "f0.las", fmt=0), "rb").read()); raw[104] = 2
    p.write_bytes(bytes(raw))                                    # format 2 needs RGB at byte 20 of a 20-byte record
    cases.append(("format", str(p), "does not fit"))
    p = tmp_path / "truncated.las"; p.write_bytes(open(good, "rb").read()[:-1])
    cases.append(("truncated", str(p), "past the end"))
    p = tmp_path / "trunc14.las"; raw = open(las_file(tmp_path / "v14.las", version=(1, 4), vlr_bytes=54), "rb").read()
    p.write_bytes(raw[:-26])
    cases.append(("truncated 1.4", str(p), "past the end"))
    p = tmp_path / "short.simlod"; p.write_bytes(b"\0" * 23)
    cases.append(("short simlod", str(p), "24-byte header"))
    for what, bad, text in cases:
        for paths in ([bad], [good, sml, bad], [bad, good]):
            rc, msg = insert_files_no_context(paths)
            assert rc == SIMLOD_ERR_INVALID, (what, rc, msg)
            assert bad in msg and text in msg, (what, msg)
    # a valid list gets as far as the context
    rc, msg = insert_files_no_context([good, sml, good])
    assert rc == SIMLOD_ERR_INVALID and "null context" in msg


def test_extensions_compare_case_insensitively(tmp_path):
    good = las_file(tmp_path / "TILE.LaS")
    sml = str(tmp_path / "SCAN.SimLOD")
    data.write_simlod(sml, fr.shifted_terrain(10), (0, 0, 0), (1, 1, 1))
    rc, msg = insert_files_no_context([good, sml])
    assert "null context" in msg, msg


def test_restatement_box_and_batches_on_hand_computed_lists(tmp_path):
    # a: 1 000 000 points, b: 1 000 001 points, e: no points, s: a .simlod file, c: a tile far from the others
    a = las_file(tmp_path / "a.las", 1_000_000, fmt=2)
    b = las_file(tmp_path / "b.las", 1_000_001, fmt=3, version=(1, 4), vlr_bytes=54)
    e = str(tmp_path / "e.las")
    data.write_las(e, np.zeros(0, dtype=oracle.POINT_DTYPE), fmt=0)
    s = str(tmp_path / "s.simlod")
    data.write_simlod(s, fr.shifted_terrain(2_000_500)[:2_000_500], (-5.0, 7.0, 1.0), (8000.0, 9000.0, 400.0))
    c = str(tmp_path / "c.las")
    pc = fr.shifted_terrain(10)
    pc["x"] += np.float32(3000.0)
    data.write_las(c, pc, fmt=7, version=(1, 4))

    bmin, bmax, tr, batches = fr.reload([a, b])
    pa, pb = fr.shifted_terrain(1_000_000), fr.shifted_terrain(1_000_001)
    for k, ax in enumerate("xyz"):
        assert bmin[k] == min(pa[ax].min(), pb[ax].min()) and bmax[k] == max(pa[ax].max(), pb[ax].max())
    assert tr.dtype == np.float64 and (tr == -bmin.astype(np.float64)).all()
    assert batches == [(a, 0, 1_000_000, "las"), (b, 0, 1_000_000, "las"), (b, 1_000_000, 1, "las")]

    # the empty file contributes its (zero) box and no batch; the .simlod header floats widen the box
    bmin, bmax, tr, batches = fr.reload([e, a, s, c, b])
    assert [list(bmin), list(bmax)] == [[-5.0, 0.0, 0.0], [8000.0, 9000.0, 400.0]]
    assert batches == [(a, 0, 1_000_000, "las"), (s, 0, 1_000_000, "simlod"), (s, 1_000_000, 1_000_000, "simlod"),
                       (s, 2_000_000, 500, "simlod"), (c, 0, 10, "las"), (b, 0, 1_000_000, "las"), (b, 1_000_000, 1, "las")]
    # without the empty file, the union of the tiles' own boxes
    bmin, _, _, _ = fr.reload([a, c])
    assert list(bmin) == [min(pa[ax].min(), pc[ax].min()) for ax in "xyz"]


@pytest.mark.parametrize("case", sorted(fr.FORMAT_CASES))
def test_restated_batches_decode_as_the_reference_loader(tmp_path, case):
    """The points the restatement gives every batch of the one-file cases the GPU test builds: those of the reference's
    loadLasNative with the union translation."""
    path = fr.write_format_case(tmp_path, case)
    _, _, _, batches = fr.check_batches_against_reference("format/" + case, [path])
    assert [b[2] for b in batches] == [1_000_000, 1_000_000, 500_000]
