"""CPU-only tests of the octree file (simlod_read_octree_header, DESIGN.md §9.7): the header's ctypes mirror against the C
layout, the header reader on well-formed and crafted files, the restatement, and the import kernels' resources."""
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import octree_file_restatement as F
from conftest import ROOT
from simlod_b200 import SimlodError, api
from simlod_b200 import build as B


def test_ctypes_mirror_matches_the_c_layout(tmp_path):
    src = tmp_path / "hdr.c"
    fields = [f for f, _ in api.OctreeFileHeader._fields_]
    src.write_text('#include <stdio.h>\n#include "simlod_abi.h"\nint main(void){printf("%zu\\n", sizeof(SimlodOctreeFileHeader));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodOctreeFileHeader, %s));\n' % f for f in fields) + "return 0;}\n")
    exe = tmp_path / "hdr"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    import ctypes as C
    assert got == [C.sizeof(api.OctreeFileHeader)] + [getattr(api.OctreeFileHeader, f).offset for f in fields]
    assert got[0] == F.HEADER_SIZE


def small_octree():
    """A root leaf with 3 points: its full export, as the restatement builds it"""
    nodes = np.zeros(1, dtype=R.EXPORT_NODE_DTYPE)
    nodes["name"] = b"r"
    nodes["flags"] = R.LEAF | R.SAMPLED
    nodes["parent"] = -1
    nodes["first_child"] = -1
    nodes["num_points"] = 3
    samples = np.zeros(3, dtype=R.POINT_DTYPE)
    samples["x"] = [1.0, 2.0, 3.0]
    info = R.ExportInfo(1, 0, 3, 3, 0)
    return nodes, samples, info


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def test_read_header_accepts_a_well_formed_file(tmp_path):
    nodes, samples, info = small_octree()
    data = F.encode(nodes, samples, info, [3], (0, 0, 0), (8, 8, 8), 1, 3)
    h = api.read_octree_header(write(tmp_path, "ok.octree", data))
    want, _, _, _ = F.decode(data)
    assert h.magic == b"SIMLODOT" and h.version == 1 and h.header_size == 128
    assert (h.info.num_nodes, h.info.num_samples, h.info.num_points, h.info.num_voxels) == (1, 3, 3, 0)
    assert tuple(h.box_max) == (8.0, 8.0, 8.0) and h.batchlet_index == 1 and h.num_points_processed == 3
    for f in ("records_offset", "counters_offset", "samples_offset", "file_size"):
        assert getattr(h, f) == want[f], f
    assert h.file_size == len(data) and h.samples_offset % 16 == 0


def header_with(data, **fields):
    h, _, _, _ = F.decode(data)
    h.update(fields)
    vals = []
    for f in F.FIELDS:
        vals.extend(h[f] if f in ("box_min", "box_max") else [h[f]])
    return F.HEADER.pack(*vals) + data[F.HEADER_SIZE:]


def test_read_header_rejects_crafted_files(tmp_path):
    nodes, samples, info = small_octree()
    data = F.encode(nodes, samples, info, [3], (0, 0, 0), (8, 8, 8), 1, 3)
    h, _, _, _ = F.decode(data)
    cases = {
        "missing.octree": None,
        "short.octree": data[:100],
        "truncated.octree": data[:-1],
        "longer.octree": data + b"\0" * 16,
        "magic.octree": b"SIMLODOX" + data[8:],
        "version.octree": header_with(data, version=2),
        "counters.octree": header_with(data, counters_offset=h["counters_offset"] + 16),
        "samples.octree": header_with(data, samples_offset=h["samples_offset"] + 16, file_size=h["file_size"] + 16),
        "size.octree": header_with(data, file_size=h["file_size"] + 16),
        "counts.octree": header_with(data, num_points=2),
    }
    for name, blob in cases.items():
        path = str(tmp_path / name) if blob is None else write(tmp_path, name, blob)
        with pytest.raises(SimlodError) as e:
            api.read_octree_header(path)
        assert e.value.code == -2, name
        assert name in str(e.value), (name, str(e.value))


def test_restatement_round_trip():
    nodes, samples, info = small_octree()
    data = F.encode(nodes, samples, info, [3], (0.5, 0, 0), (8, 8, 8), 4, 12)
    h, n2, c2, s2 = F.decode(data)
    assert n2.tobytes() == nodes.tobytes() and s2.tobytes() == samples.tobytes() and list(c2) == [3]
    assert h["box_min"] == (0.5, 0.0, 0.0) and h["batchlet_index"] == 4 and h["num_points_processed"] == 12
    assert h["samples_offset"] == 208 and h["file_size"] == 208 + 48


def test_import_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit not found")
    cubin = str(tmp_path / "import.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v", "-cubin", "-o", cubin, os.path.join(B.CSRC, "import.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", res.stdout)
    names = {p[0] for p in props}
    assert {"simlod_import_nodes", "simlod_import_link", "simlod_import_clear_grids", "simlod_import_scatter", "simlod_import_voxels",
            "simlod_import_count_grids"} <= names, res.stdout
    assert all(p[1:] == ("0", "0", "0") for p in props), props
