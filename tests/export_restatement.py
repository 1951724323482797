"""TEST INFRASTRUCTURE — CPU restatement of simlod_export_octree (DESIGN.md §9.4): what the device must write for an
octree, computed independently of simlod_b200 (which it checks).

  export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth)   a raw device image (SimLOD.download_octree()):
      walks the children pointers and the chunk lists itself, so its output is the byte-exact expectation for the same
      buffers (samples in chunk-list order), and it reports an inconsistent image with the export's error codes
  export_canon(canon, depth)   a canonical form (oracle.Canon, e.g. of the oracle builder): the same node table; the
      samples of each node come in the canonical form's sorted order, so they compare per node as multisets

Both return (nodes as EXPORT_NODE_DTYPE, samples as POINT_DTYPE, ExportInfo); export_image raises ExportError."""
import ctypes as C

import numpy as np

POINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("color", "<u4")])
# SimlodExportNode / SimlodExportInfo (include/simlod_abi.h), restated so that the checker does not import the code it checks
EXPORT_NODE_DTYPE = np.dtype([
    ("level", "<u4"), ("X", "<u4"), ("Y", "<u4"), ("Z", "<u4"), ("name", "S20"), ("flags", "<u4"),
    ("parent", "<i4"), ("first_child", "<i4"), ("sample_offset", "<u8"), ("num_points", "<u4"), ("num_voxels", "<u4")])
assert EXPORT_NODE_DTYPE.itemsize == 64
LEAF, SAMPLED = 1, 2
MAX_DEPTH = 20
PPC = 1000                      # samples per chunk
CHUNK_BYTES = 16016             # SimlodChunk: 1000 points, size, padding, next (at byte 16008)

# the fields of SimlodNode the export reads (include/simlod_abi.h)
NODE_DTYPE = np.dtype({"names": ["children", "numPoints", "level", "X", "Y", "Z", "name", "points", "voxelChunks", "numVoxelsStored"],
                       "formats": [("<u8", 8), "<u4", "<u4", "<u4", "<u4", "<u4", "S20", "<u8", "<u8", "<u4"],
                       "offsets": [0, 68, 72, 76, 80, 84, 96, 128, 136, 148], "itemsize": 152})

# error codes (as the export reports them in its message; the canonicaliser uses 1, 2 and 4 for the same conditions)
ERR_CHILD, ERR_CHUNK, ERR_SHORT, ERR_PARTIAL = 1, 2, 4, 5


class ExportInfo(C.Structure):
    _fields_ = [("num_nodes", C.c_uint32), ("max_level", C.c_uint32), ("num_samples", C.c_uint64), ("num_points", C.c_uint64),
                ("num_voxels", C.c_uint64)]


class ExportError(RuntimeError):
    def __init__(self, code):
        super().__init__("inconsistent octree image (export error %d)" % code)
        self.code = code


def _plan(num_nodes, children, depth):
    """Breadth-first records from node 0. children(i) -> None for a leaf or the 8 child node indices; raises ExportError.
    Returns (record -> node index, parent, first_child, flags, sampled points?, sampled voxels?)."""
    if depth is not None and depth > MAX_DEPTH:
        raise ValueError("depth %d > %d" % (depth, MAX_DEPTH))
    full = depth is None or depth < 0
    rec_node, parent = [0], [-1]
    first_child, flags, take_points, take_voxels = [], [], [], []
    begin, end, level = 0, 1, 0
    while begin < end:
        expand = full or level < depth
        for r in range(begin, end):
            kids = children(rec_node[r])
            inner = kids is not None
            fc = -1
            if expand and inner:
                if len(rec_node) + 8 > num_nodes:           # more records than nodes: a node reached twice
                    raise ExportError(ERR_CHILD)
                fc = len(rec_node)
                rec_node.extend(kids)
                parent.extend([r] * 8)
            first_child.append(fc)
            flags.append((0 if inner else LEAF) | (SAMPLED if full or not inner or level == depth else 0))
            take_points.append(full or not inner)
            take_voxels.append(full or (inner and level == depth))
        begin, end, level = end, len(rec_node), level + 1
    return rec_node, parent, first_child, flags, take_points, take_voxels


def _assemble(fields, rec_node, parent, first_child, flags, take_points, take_voxels, samples_of, max_level):
    n = len(rec_node)
    nodes = np.zeros(n, dtype=EXPORT_NODE_DTYPE)
    idx = np.asarray(rec_node, dtype=np.int64)
    for f in ("level", "X", "Y", "Z", "name"):
        nodes[f] = fields[f][idx]
    nodes["flags"], nodes["parent"], nodes["first_child"] = flags, parent, first_child
    parts, offset = [], 0
    for r in range(n):
        pts, vox = samples_of(rec_node[r], take_points[r], take_voxels[r])
        nodes["sample_offset"][r] = offset
        nodes["num_points"][r], nodes["num_voxels"][r] = len(pts), len(vox)
        parts += [pts, vox]
        offset += len(pts) + len(vox)
    samples = np.concatenate(parts) if parts else np.zeros(0, dtype=POINT_DTYPE)
    info = ExportInfo(n, max_level, offset, int(nodes["num_points"].sum()), int(nodes["num_voxels"].sum()))
    return nodes, samples.view(POINT_DTYPE), info


def export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, depth=None):
    """The export of a raw device image: nodes_bytes = nodes[0, Stats::numNodes), heap_bytes = the used heap."""
    nodes = np.frombuffer(np.ascontiguousarray(nodes_bytes, dtype=np.uint8).tobytes(), dtype=NODE_DTYPE)
    heap = np.ascontiguousarray(heap_bytes, dtype=np.uint8)
    num_nodes, heap_used = len(nodes), len(heap)

    def children(i):
        ptrs = [int(p) for p in nodes["children"][i]]
        nonzero = [p for p in ptrs if p]
        for p in nonzero:
            if p < nodes_addr or (p - nodes_addr) % 152 or (p - nodes_addr) // 152 >= num_nodes:
                raise ExportError(ERR_CHILD)
        if not nonzero:
            return None
        if len(nonzero) != 8:
            raise ExportError(ERR_PARTIAL)
        return [(p - nodes_addr) // 152 for p in ptrs]

    def walk(head, count):
        """`count` samples of the list at `head`, chunk by chunk; every chunk is tested before it is read."""
        out, addr, left = [], int(head), int(count)
        while left > 0:
            if addr == 0:
                raise ExportError(ERR_SHORT)
            off = addr - heap_addr
            if addr < heap_addr or off + CHUNK_BYTES > heap_used or off % 16:
                raise ExportError(ERR_CHUNK)
            take = min(left, PPC)
            out.append(heap[off:off + 16 * take])
            left -= take
            addr = int(heap[off + 16008:off + 16016].view(np.uint64)[0])
        return np.concatenate(out).view(POINT_DTYPE) if out else np.zeros(0, dtype=POINT_DTYPE)

    def samples_of(i, points, voxels):
        pts = walk(nodes["points"][i], nodes["numPoints"][i]) if points else np.zeros(0, dtype=POINT_DTYPE)
        vox = walk(nodes["voxelChunks"][i], nodes["numVoxelsStored"][i]) if voxels else np.zeros(0, dtype=POINT_DTYPE)
        return pts, vox

    plan = _plan(num_nodes, children, depth)
    return _assemble(nodes, *plan, samples_of, int(nodes["level"].max(initial=0)))


def export_canon(canon, depth=None):
    """The export of a canonical form (oracle.Canon): children are the records one level down at (2X+x, 2Y+y, 2Z+z)."""
    rec = canon.records
    index = {(int(r["level"]), int(r["X"]), int(r["Y"]), int(r["Z"])): k for k, r in enumerate(rec)}

    def children(k):
        if int(rec["isLeaf"][k]):
            return None
        l, X, Y, Z = (int(rec[f][k]) for f in ("level", "X", "Y", "Z"))
        return [index[(l + 1, 2 * X + (c >> 2 & 1), 2 * Y + (c >> 1 & 1), 2 * Z + (c & 1))] for c in range(8)]

    def samples_of(k, points, voxels):
        empty = np.zeros(0, dtype=POINT_DTYPE)
        return (canon.samples(k) if points else empty), (canon.samples(k, voxels=True) if voxels else empty)

    plan = _plan(len(rec), children, depth)
    return _assemble(rec, *plan, samples_of, int(rec["level"].max(initial=0)))
