"""CPU-only: the view export's restatement (export_view_restatement.export_view_image, drawn_from_flags) on hand-made device
images and drawn sets, and the register budget of export.cu's kernels. The GPU view export is pinned byte for byte to
this restatement in test_export_view_gpu.py."""
import os
import re
import subprocess

import numpy as np
import pytest

import export_restatement as R
import export_view_restatement as V
from simlod_b200 import api
from simlod_b200 import build as B
from test_export_cpu import HEAP_ADDR, NODE_DTYPE, NODES_ADDR, check_structure

SAMPLED, LEAF = api.EXPORT_SAMPLED, api.EXPORT_LEAF


class Tree:
    """A hand-made device image: the root (0) with 8 children (1-8); child 3 (node 4) split into 9-16, and its child 5
    (node 14) into 17-24, so the deepest leaves are at level 3. Leaves hold points, inner nodes voxels; every list is a
    chain of chunks laid out back to front in the heap. `extra` appends unreferenced leaves to nodes[]."""

    SPLIT = {0: 1, 4: 9, 14: 17}

    def __init__(self, root_only=False, extra=0):
        rng = np.random.default_rng(5)
        n = (1 if root_only else 25) + extra
        self.nodes = np.zeros(n, dtype=NODE_DTYPE)
        self.nodes["name"][0] = b"r"
        if not root_only:
            for parent, first in self.SPLIT.items():
                self.nodes["children"][parent] = [NODES_ADDR + 152 * (first + k) for k in range(8)]
                for k in range(8):
                    c = first + k
                    self.nodes["level"][c] = self.nodes["level"][parent] + 1
                    self.nodes["X"][c] = 2 * self.nodes["X"][parent] + (k >> 2 & 1)
                    self.nodes["Y"][c] = 2 * self.nodes["Y"][parent] + (k >> 1 & 1)
                    self.nodes["Z"][c] = 2 * self.nodes["Z"][parent] + (k & 1)
                    self.nodes["name"][c] = self.nodes["name"][parent] + bytes([48 + k])
        for i in range(len(self.nodes) - extra, len(self.nodes)):       # unreferenced leaves: level 1, name "r9"
            self.nodes["level"][i], self.nodes["name"][i] = 1, b"r9"
        self.lists = {}
        for i in range(len(self.nodes)):
            inner = self.nodes["children"][i][0] != 0
            if root_only or inner:
                self.lists[("v", i)] = 700 + 450 * i
            if root_only or not inner:
                self.lists[("p", i)] = [0, 1, 999, 1000, 1001, 2500, 7][i % 7]
        chunks = []
        self.samples = {}
        for key, count in self.lists.items():
            s = np.zeros(count, dtype=api.POINT_DTYPE)
            s["x"] = rng.random(count, dtype=np.float32)
            s["color"] = rng.integers(0, 2**32, count, dtype=np.uint32)
            self.samples[key] = s
            chunks += [(key, j) for j in range(0, count, 1000)]
        chunks.reverse()
        self.heap = np.zeros(16 + 16032 * len(chunks), dtype=np.uint8)
        self.heap[8:16].view(np.uint64)[0] = len(self.heap)
        where = {c: 16 + 16032 * k for k, c in enumerate(chunks)}
        for (key, j), off in where.items():
            part = self.samples[key][j:j + 1000]
            self.heap[off:off + 16 * len(part)] = part.view(np.uint8)
            nxt = where.get((key, j + 1000))
            self.heap[off + 16008:off + 16016].view(np.uint64)[0] = HEAP_ADDR + nxt if nxt is not None else 0
        for (kind, i), count in self.lists.items():
            head = where.get(((kind, i), 0))
            self.nodes["voxelChunks" if kind == "v" else "points"][i] = HEAP_ADDR + head if head is not None else 0
            if kind == "v":
                self.nodes["numVoxels"][i] = self.nodes["numVoxelsStored"][i] = count
            else:
                self.nodes["numPoints"][i] = count

    def image(self):
        return np.ascontiguousarray(self.nodes).view(np.uint8), self.heap, NODES_ADDR, HEAP_ADDR

    def drawn(self, *indices):
        d = np.zeros(len(self.nodes), dtype=bool)
        d[list(indices)] = True
        return d

    def view(self, *indices):
        return V.export_view_image(*self.image(), self.drawn(*indices))

    def node_samples(self, i):
        empty = np.zeros(0, dtype=api.POINT_DTYPE)
        return np.concatenate([self.samples.get(("p", i), empty), self.samples.get(("v", i), empty)])


def record_of(nodes, name):
    return int(np.nonzero(nodes["name"] == name)[0][0])


def test_nothing_drawn_gives_the_root_alone():
    t = Tree()
    nodes, samples, info = t.view()
    check_structure(nodes, info)
    assert info.num_nodes == 1 and info.num_samples == 0 and len(samples) == 0 and info.max_level == 3
    assert nodes["flags"][0] == 0 and nodes["parent"][0] == -1 and nodes["first_child"][0] == -1 and nodes["name"][0] == b"r"


def test_one_deep_leaf_gives_its_path_and_the_siblings_on_it():
    t = Tree()
    leaf = 17 + 6                                             # level 3, name r356
    nodes, samples, info = t.view(leaf)
    check_structure(nodes, info)
    assert info.num_nodes == 1 + 3 * 8
    assert [bytes(n) for n in nodes["name"][[0, 4, 14]]] == [b"r", b"r3", b"r35"]
    assert (nodes["first_child"] >= 0).sum() == 3                 # root, r3, r35 expanded; their siblings are not
    r = record_of(nodes, b"r356")
    assert nodes["flags"][r] == SAMPLED | LEAF and ((nodes["flags"] & SAMPLED) != 0).sum() == 1
    assert samples.tobytes() == t.node_samples(leaf).tobytes()
    assert info.num_points == t.nodes["numPoints"][leaf] and info.num_voxels == 0


def test_drawn_inner_node_carries_its_voxels_and_leaves_elsewhere_their_points():
    t = Tree()
    nodes, samples, info = t.view(14, 2, 17)                  # r35 (inner, level 2), r1 (leaf, level 1), r350 (below r35)
    check_structure(nodes, info)
    flagged = sorted(bytes(n) for n in nodes["name"][(nodes["flags"] & SAMPLED) != 0])
    assert flagged == [b"r1", b"r35", b"r350"]
    r = record_of(nodes, b"r35")
    assert nodes["num_voxels"][r] == t.nodes["numVoxelsStored"][14] and nodes["num_points"][r] == 0
    order = [record_of(nodes, n) for n in (b"r1", b"r35", b"r350")]
    assert order == sorted(order)
    assert samples.tobytes() == np.concatenate([t.node_samples(i) for i in (2, 14, 17)]).tobytes()


def test_drawn_leaf_root_carries_points_and_voxels():
    t = Tree(root_only=True)
    nodes, samples, info = t.view(0)
    check_structure(nodes, info)
    assert info.num_nodes == 1 and nodes["flags"][0] == SAMPLED | LEAF
    assert info.num_points == t.nodes["numPoints"][0] and info.num_voxels == t.nodes["numVoxelsStored"][0] > 0
    assert samples.tobytes() == t.node_samples(0).tobytes()
    n0, s0, i0 = t.view()
    assert i0.num_nodes == 1 and n0["flags"][0] == LEAF and i0.num_samples == 0


def test_all_leaves_drawn_gives_the_full_node_table():
    t = Tree()
    leaves = [i for i in range(len(t.nodes)) if t.nodes["children"][i][0] == 0]
    nodes, samples, info = t.view(*leaves)
    full, _, finfo = R.export_image(*t.image())
    check_structure(nodes, info)
    assert info.num_nodes == finfo.num_nodes == len(t.nodes)
    for f in ("level", "X", "Y", "Z", "name", "parent", "first_child", "num_points"):
        assert (nodes[f] == full[f]).all(), f
    assert ((nodes["flags"] & SAMPLED != 0) == (nodes["flags"] & LEAF != 0)).all()
    assert (nodes["flags"] & LEAF == full["flags"] & LEAF).all()
    assert info.num_voxels == 0 and info.num_points == finfo.num_points


def test_every_drawn_set_keeps_the_structure():
    t = Tree()
    rng = np.random.default_rng(11)
    for _ in range(40):
        d = rng.random(len(t.nodes)) < 0.2
        nodes, samples, info = V.export_view_image(*t.image(), d)
        check_structure(nodes, info)
        assert (nodes["flags"] & SAMPLED != 0).sum() == d.sum()
        got = sorted(bytes(n) for n in nodes["name"][(nodes["flags"] & SAMPLED) != 0])
        assert got == sorted(bytes(n) for n in t.nodes["name"][d])
        assert info.num_samples == sum(len(t.node_samples(i)) for i in np.nonzero(d)[0])
        # the smallest set: a record is expanded exactly when a drawn node lies below it
        for r in range(len(nodes)):
            below = any(bytes(n).startswith(bytes(nodes["name"][r])) and len(n) > len(nodes["name"][r]) for n in t.nodes["name"][d])
            assert (nodes["first_child"][r] >= 0) == below


def flags_image(t, visible, large):
    raw = np.ascontiguousarray(t.nodes).view(np.uint8).reshape(-1, 152).copy()
    raw[:, V.VISIBLE_BYTE] = visible
    raw[:, V.IS_LARGE_BYTE] = large
    return raw.reshape(-1)


def test_drawn_from_flags_is_the_renderers_second_pass():
    t = Tree()
    n = len(t.nodes)
    visible, large = np.ones(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    large[[0, 4]] = 1                     # root and r3 large: the children of both are drawn unless large themselves
    large[7] = 1                          # r6: a large leaf, drawn
    large[14] = 1                         # r35: large inner, so its children are drawn and it is not
    visible[9] = 0                        # r30: not visible
    d = V.drawn_from_flags(flags_image(t, visible, large))
    want = {1, 2, 3, 5, 6, 7, 8} | {10, 11, 12, 13, 15, 16} | set(range(17, 25))
    assert set(np.nonzero(d)[0].tolist()) == want
    # a large visible leaf under a parent that is not large is drawn; a large invisible leaf is not
    large2, visible2 = np.zeros(n, dtype=np.uint8), np.ones(n, dtype=np.uint8)
    large2[[20, 21]] = 1
    visible2[21] = 0
    d2 = V.drawn_from_flags(flags_image(t, visible2, large2))
    assert set(np.nonzero(d2)[0].tolist()) == {20}
    nodes, _, info = V.export_view_image(*t.image(), d2)
    check_structure(nodes, info)
    assert [bytes(x) for x in nodes["name"][(nodes["flags"] & SAMPLED) != 0]] == [b"r353"]


@pytest.mark.parametrize("corruption,code", [
    ("child_outside_nodes", 1), ("chunk_outside_heap", 2), ("list_shorter_than_count", 4), ("seven_children", 5),
    ("unreachable_drawn_node", 1), ("drawn_node_reached_twice", 1)])
def test_view_errors(corruption, code):
    t = Tree(extra=1 if corruption == "unreachable_drawn_node" else 0)
    drawn = [17]
    if corruption == "child_outside_nodes":
        t.nodes["children"][4, 2] = NODES_ADDR + 152 * len(t.nodes)
    elif corruption == "chunk_outside_heap":
        t.nodes["points"][17] = HEAP_ADDR + len(t.heap) - 16000
    elif corruption == "list_shorter_than_count":
        t.nodes["numPoints"][17] += 1000
    elif corruption == "seven_children":
        t.nodes["children"][0, 7] = 0
    elif corruption == "unreachable_drawn_node":
        drawn.append(len(t.nodes) - 1)
    else:                                 # r34 and r35 share their children: r35's subtree is reached twice
        t.nodes["children"][13] = t.nodes["children"][14]
    with pytest.raises(R.ExportError) as err:
        t.view(*drawn)
    assert err.value.code == code


def test_lists_of_nodes_that_are_not_drawn_are_not_followed():
    t = Tree()
    t.nodes["points"][18] = HEAP_ADDR + len(t.heap) - 16000     # r351: its chunk pointer lies outside the heap
    with pytest.raises(R.ExportError):
        R.export_image(*t.image())
    nodes, samples, _ = t.view(17)
    assert samples.tobytes() == t.node_samples(17).tobytes()


def test_drawn_set_must_cover_nodes():
    t = Tree()
    with pytest.raises(ValueError):
        V.export_view_image(*t.image(), np.zeros(len(t.nodes) - 1, dtype=bool))


# ---- export.cu: no kernel uses local memory -------------------------------------------------------------------------

def test_export_kernels_use_no_local_memory(tmp_path):
    if not os.path.exists(B.NVCC):
        pytest.skip("CUDA toolkit (nvcc) not found")
    cubin = str(tmp_path / "export.cubin")
    cmd = [B.NVCC] + B.ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v"] + B.EXTRA_FLAGS.get("export", []) + \
        ["-cubin", "-o", cubin, os.path.join(B.CSRC, "export.cu")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                       res.stdout)
    names = {f for f, *_ in found}
    assert {"simlod_export_view_flags", "simlod_export_plan", "simlod_export_collect", "simlod_export_gather"} <= names, res.stdout
    for f, stack, stores, loads in found:
        assert (int(stack), int(stores), int(loads)) == (0, 0, 0), "%s uses local memory: %s" % (f, res.stdout)
