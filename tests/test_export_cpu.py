"""CPU-only: the octree export's layout and its restatement (export_restatement.py) on oracle-built octrees and
hand-made device images. The GPU export is pinned byte for byte to this restatement in test_export_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import export_restatement as R
import oracle
from conftest import ROOT
from simlod_b200 import api, data


# ---- properties every export has (also used by test_export_gpu.py) ----------------------------------------------

def morton(level, X, Y, Z):
    """Morton code of (X, Y, Z) at `level`: bit triples x<<2 | y<<1 | z, root first (the reference's child index)."""
    code = np.zeros(len(X), dtype=np.uint64)
    for b in range(int(level.max(initial=0)) - 1, -1, -1):
        on = level > b
        bits = (((X >> b) & 1) << 2 | ((Y >> b) & 1) << 1 | ((Z >> b) & 1)).astype(np.uint64)
        code = np.where(on, (code << np.uint64(3)) | bits, code)
    return code


def check_structure(nodes, info):
    """(level, Morton) order, parent / first-child links, 8 consecutive children, contiguous sample offsets."""
    n = len(nodes)
    assert n == info.num_nodes and n >= 1
    lv, X, Y, Z = (nodes[f].astype(np.uint64) for f in ("level", "X", "Y", "Z"))
    key = list(zip(lv.tolist(), morton(lv, X, Y, Z).tolist()))
    assert all(a < b for a, b in zip(key, key[1:])), "records are not in (level, Morton) order"
    assert nodes["parent"][0] == -1 and nodes["level"][0] == 0
    for i in np.nonzero(nodes["first_child"] >= 0)[0]:
        fc = int(nodes["first_child"][i])
        kids = nodes[fc:fc + 8]
        assert len(kids) == 8 and (kids["parent"] == i).all() and (kids["level"] == nodes["level"][i] + 1).all()
        k = np.arange(8, dtype=np.uint32)
        assert (kids["X"] == 2 * nodes["X"][i] + (k >> 2 & 1)).all()
        assert (kids["Y"] == 2 * nodes["Y"][i] + (k >> 1 & 1)).all()
        assert (kids["Z"] == 2 * nodes["Z"][i] + (k & 1)).all()
        assert not nodes["flags"][i] & api.EXPORT_LEAF
    for i in range(1, n):
        p = int(nodes["parent"][i])
        assert 0 <= p < i and nodes["first_child"][p] <= i < nodes["first_child"][p] + 8
    counts = nodes["num_points"].astype(np.uint64) + nodes["num_voxels"]
    assert (nodes["sample_offset"] == np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint64)).all()
    assert int(counts.sum()) == info.num_samples == info.num_points + info.num_voxels
    assert int(nodes["num_points"].sum()) == info.num_points and int(nodes["num_voxels"].sum()) == info.num_voxels
    # samples only where flagged
    assert (counts[(nodes["flags"] & api.EXPORT_SAMPLED) == 0] == 0).all()


def cut_count(records, depth):
    """Samples of the cut at `depth` from the canonical records: voxels of the inner nodes at `depth`, points of the leaves above."""
    inner = records["isLeaf"] == 0
    return int(records["numVoxelsStored"][inner & (records["level"] == depth)].sum()) + \
        int(records["numPoints"][~inner & (records["level"] <= depth)].sum())


def sorted_points(p):
    """16-byte samples as (N, 2) uint64 rows in a canonical order (for multiset comparisons)."""
    a = np.ascontiguousarray(p).view(np.uint64).reshape(-1, 2)
    return a[np.lexsort((a[:, 1], a[:, 0]))]


def check_against_canon(canon, points=None):
    """The restatement of `canon` at every depth against the canonical records; `points`: the inserted point set."""
    rec = canon.records
    nodes, samples, info = R.export_canon(canon)
    check_structure(nodes, info)
    assert (nodes["flags"] & api.EXPORT_SAMPLED).all()
    assert info.max_level == int(rec["level"].max()) and info.num_nodes == len(rec)
    # the full export holds every node with both of its lists: per node, the same multisets as the canonical form
    order = np.lexsort((nodes["Z"], nodes["Y"], nodes["X"], nodes["level"]))
    for f in ("level", "X", "Y", "Z", "name"):
        assert (nodes[f][order] == rec[f]).all(), f
    assert (nodes["num_points"][order] == rec["numPoints"]).all() and (nodes["num_voxels"][order] == rec["numVoxelsStored"]).all()
    assert ((nodes["flags"][order] & api.EXPORT_LEAF) == rec["isLeaf"]).all()
    for k, i in enumerate(order):
        o, np_, nv = int(nodes["sample_offset"][i]), int(nodes["num_points"][i]), int(nodes["num_voxels"][i])
        assert np.array_equal(sorted_points(samples[o:o + np_]), sorted_points(canon.samples(k)))
        assert np.array_equal(sorted_points(samples[o + np_:o + np_ + nv]), sorted_points(canon.samples(k, voxels=True)))
    deepest_leaf = int(rec["level"][rec["isLeaf"] == 1].max())
    for depth in range(0, info.max_level + 2):
        cn, cs, ci = R.export_canon(canon, depth)
        check_structure(cn, ci)
        assert ci.max_level == info.max_level
        assert (cn["level"] <= depth).all() and ci.num_nodes == int((rec["level"] <= depth).sum())
        assert ci.num_samples == cut_count(rec, depth)
        # records are the full export's first records, with the cut's flags and counts
        head = nodes[:ci.num_nodes]
        for f in ("level", "X", "Y", "Z", "name", "parent"):
            assert (cn[f] == head[f]).all()
        if depth >= deepest_leaf:
            assert ci.num_voxels == 0
            if points is not None:
                assert np.array_equal(sorted_points(cs), sorted_points(points))
    return nodes, samples, info


# ---- layout ---------------------------------------------------------------------------------------------------------

def test_export_dtypes_match_the_c_structs(tmp_path):
    src = tmp_path / "layout.c"
    fields = [n for n in api.EXPORT_NODE_DTYPE.names]
    src.write_text('#include <stdio.h>\n#include "simlod_abi.h"\nint main(void){\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodExportNode, %s));\n' % f for f in fields) +
                   'printf("%zu\\n%zu\\n", sizeof(SimlodExportNode), sizeof(SimlodExportInfo));\n' +
                   "".join('printf("%%zu\\n", offsetof(SimlodExportInfo, %s));\n' % f for f, _ in api.ExportInfo._fields_) +
                   "return 0;}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert out[:len(fields)] == [api.EXPORT_NODE_DTYPE.fields[f][1] for f in fields]
    assert out[len(fields):len(fields) + 2] == [api.EXPORT_NODE_DTYPE.itemsize, C.sizeof(api.ExportInfo)] == [64, 32]
    assert out[len(fields) + 2:] == [getattr(api.ExportInfo, f).offset for f, _ in api.ExportInfo._fields_]
    assert R.EXPORT_NODE_DTYPE == api.EXPORT_NODE_DTYPE and (R.LEAF, R.SAMPLED) == (api.EXPORT_LEAF, api.EXPORT_SAMPLED)
    assert R.ExportInfo._fields_ == api.ExportInfo._fields_


def test_morton_helper_orders_children_by_child_index():
    k = np.arange(8, dtype=np.uint64)
    lv = np.ones(8, dtype=np.uint64)
    assert (morton(lv, k >> np.uint64(2) & np.uint64(1), k >> np.uint64(1) & np.uint64(1), k & np.uint64(1)) == k).all()


# ---- oracle-built octrees --------------------------------------------------------------------------------------------

def build(batches, box):
    o = oracle.Oracle(box[0], box[1])
    for b in batches:
        o.add_batch(b)
    return o


def test_uniform_1m():
    pts, mn, mx = data.uniform_cube(1_000_000)
    o = build([pts], (mn, mx))
    check_against_canon(o.canon(), pts)


def test_ragged_terrain_stream():
    n = 3_300_000
    pts, mn, mx = data.terrain(n)
    sizes = [1_000_000, 1_000_000, 7, 0, 900_000, n - 2_900_007]
    batches = np.split(pts, np.cumsum(sizes)[:-1])
    o = build(batches, (mn, mx))
    check_against_canon(o.canon(), pts)


@pytest.mark.parametrize("case", ["empty", "one_point", "leaf_root", "corner_cascade"])
def test_hand_made_streams(case):
    rng = np.random.default_rng(4)
    box = ((0.0, 0.0, 0.0), (64.0, 64.0, 64.0))
    if case == "empty":
        pts = np.zeros(0, dtype=api.POINT_DTYPE)
    elif case == "one_point":
        pts = api.make_points([[1.0, 2.0, 3.0]], [0xFF112233])
    elif case == "leaf_root":           # 50 000 points: the root stays a leaf and keeps its voxels
        pts = api.make_points(rng.random((50_000, 3), dtype=np.float32) * np.float32(64.0), rng.integers(0, 2**32, 50_000, dtype=np.uint32))
    else:                               # 120 000 points in a tiny corner: a split cascade several levels deep
        pts = api.make_points(rng.random((120_000, 3), dtype=np.float32) * np.float32(0.5), rng.integers(0, 2**32, 120_000, dtype=np.uint32))
    batches = [pts[i:i + 40_000] for i in range(0, max(len(pts), 1), 40_000)]
    o = build(batches, box)
    nodes, samples, info = check_against_canon(o.canon(), pts)
    if case in ("empty", "one_point", "leaf_root"):
        assert info.num_nodes == 1 and nodes["flags"][0] == api.EXPORT_LEAF | api.EXPORT_SAMPLED
        assert info.num_points == len(pts)
    if case == "leaf_root":
        assert info.num_voxels > 0                                     # the full export keeps a leaf root's voxels
        _, _, cut = R.export_canon(o.canon(), 0)
        assert cut.num_voxels == 0 and cut.num_points == len(pts)      # the cut does not
    if case == "corner_cascade":
        assert info.max_level >= 4


# ---- hand-made device images: list order and the validation paths ---------------------------------------------------

NODES_ADDR, HEAP_ADDR = 0x7000_0000_0000, 0x7100_0000_0000
NODE_DTYPE = np.dtype({"names": ["children", "numPoints", "level", "X", "Y", "Z", "name", "points", "voxelChunks", "numVoxels", "numVoxelsStored"],
                       "formats": [("<u8", 8), "<u4", "<u4", "<u4", "<u4", "<u4", "S20", "<u8", "<u8", "<u4", "<u4"],
                       "offsets": [0, 68, 72, 76, 80, 84, 96, 128, 136, 144, 148], "itemsize": 152})


class Image:
    """A root with 8 leaf children; chunk lists laid out out of address order so that list order is observable."""

    def __init__(self):
        rng = np.random.default_rng(9)
        self.nodes = np.zeros(9, dtype=NODE_DTYPE)
        self.nodes["name"][0] = b"r"
        self.nodes["children"][0] = [NODES_ADDR + 152 * (k + 1) for k in range(8)]
        self.chunks = []            # (list of points) per heap chunk, in allocation order
        self.lists = {}
        counts = {("v", 0): 1500}
        for k in range(8):
            for f, v in (("level", 1), ("X", k >> 2 & 1), ("Y", k >> 1 & 1), ("Z", k & 1), ("name", b"r" + bytes([48 + k]))):
                self.nodes[f][k + 1] = v
            counts[("p", k + 1)] = [0, 1, 999, 1000, 1001, 2500, 7, 3000][k]
        for (kind, i), n in counts.items():
            samples = np.zeros(n, dtype=api.POINT_DTYPE)
            samples["x"] = rng.random(n, dtype=np.float32)
            samples["color"] = rng.integers(0, 2**32, n, dtype=np.uint32)
            self.lists[(kind, i)] = samples
        # allocate chunks round robin over the lists, then link every list back to front
        pending = {key: [s[j:j + 1000] for j in range(0, len(s), 1000)] for key, s in self.lists.items()}
        addr = {key: [] for key in pending}
        while any(pending.values()):
            for key in sorted(pending, reverse=True):
                if pending[key]:
                    addr[key].append(16 + 16032 * len(self.chunks))
                    self.chunks.append(pending[key].pop(0))
        self.heap = np.zeros(16 + 16032 * len(self.chunks), dtype=np.uint8)
        self.heap[8:16].view(np.uint64)[0] = len(self.heap)
        for key, offs in addr.items():
            for j, off in enumerate(offs):
                nxt = HEAP_ADDR + offs[j + 1] if j + 1 < len(offs) else 0
                self.heap[off + 16008:off + 16016].view(np.uint64)[0] = nxt
            kind, i = key
            field = "points" if kind == "p" else "voxelChunks"
            self.nodes[field][i] = HEAP_ADDR + offs[0] if offs else 0
            if kind == "p":
                self.nodes["numPoints"][i] = len(self.lists[key])
            else:
                self.nodes["numVoxels"][i] = self.nodes["numVoxelsStored"][i] = len(self.lists[key])
        for off, pts in zip([16 + 16032 * c for c in range(len(self.chunks))], self.chunks):
            self.heap[off:off + 16 * len(pts)] = pts.view(np.uint8)

    def image(self):
        return np.ascontiguousarray(self.nodes).view(np.uint8), self.heap, NODES_ADDR, HEAP_ADDR

    def canon_error(self):
        nb = np.ascontiguousarray(self.nodes).view(np.uint8)
        h = oracle.lib().canon_from_image(nb.ctypes.data, len(self.nodes), self.heap.ctypes.data, len(self.heap), NODES_ADDR, HEAP_ADDR)
        try:
            return oracle.lib().canon_error(h)
        finally:
            oracle.lib().canon_destroy(h)

    def export(self, depth):
        """(restatement's error code, the canonicaliser's error code, nodes, samples) of this image."""
        try:
            nodes, samples, _ = R.export_image(*self.image(), depth)
            rc = 0
        except R.ExportError as e:
            rc, nodes, samples = e.code, None, None
        return rc, self.canon_error(), nodes, samples


def test_image_export_keeps_chunk_list_order():
    img = Image()
    rc, err, nodes, samples = img.export(-1)
    assert rc == 0 and err == 0 and len(nodes) == 9
    want = [img.lists[("v", 0)]] + [img.lists[("p", k + 1)] for k in range(8)]
    assert samples.tobytes() == np.concatenate(want).tobytes()
    assert nodes["first_child"][0] == 1 and (nodes["parent"][1:] == 0).all()
    rc, _, nodes0, samples0 = img.export(0)
    assert rc == 0 and len(nodes0) == 1 and nodes0["first_child"][0] == -1 and samples0.tobytes() == img.lists[("v", 0)].tobytes()
    rc, _, nodes1, samples1 = img.export(1)
    assert rc == 0 and not nodes1["flags"][0] & api.EXPORT_SAMPLED and samples1.tobytes() == np.concatenate(want[1:]).tobytes()
    with pytest.raises(ValueError):
        img.export(21)
    # the canonical-form path of the restatement gives the same node table and, per node, the same samples
    for depth in (-1, 0, 1):
        _, _, nodes, samples = img.export(depth)
        cn, cs, ci = R.export_canon(oracle.canon_from_image(*img.image()), depth)
        assert cn.tobytes() == nodes.tobytes() and ci.num_samples == len(samples)
        for i in range(len(cn)):
            a, m = int(cn["sample_offset"][i]), int(cn["num_points"][i] + cn["num_voxels"][i])
            assert np.array_equal(sorted_points(cs[a:a + m]), sorted_points(samples[a:a + m]))


@pytest.mark.parametrize("corruption,code,canon_code", [
    ("child_outside_nodes", 1, 1), ("chunk_outside_heap", 2, 2), ("list_shorter_than_count", 4, 4), ("seven_children", 5, 0)])
def test_image_inconsistencies_are_reported(corruption, code, canon_code):
    img = Image()
    if corruption == "child_outside_nodes":
        img.nodes["children"][0, 3] = NODES_ADDR + 152 * 9
    elif corruption == "chunk_outside_heap":
        img.nodes["points"][6] = HEAP_ADDR + len(img.heap) - 16000
    elif corruption == "list_shorter_than_count":
        img.nodes["numPoints"][5] = 2001
    else:
        img.nodes["children"][0, 7] = 0
    rc, err, _, _ = img.export(-1)
    assert (rc, err) == (code, canon_code)
