"""TEST INFRASTRUCTURE — CPU restatement of the octree file (simlod_save_octree, DESIGN.md §9.7): the bytes a saved
octree must consist of, computed independently of simlod_b200 (which it checks), on top of the export's restatement.

  file_bytes(nodes_bytes, heap_bytes, nodes_addr, heap_addr, box_min, box_max, batchlet_index, num_points_processed)
      a raw device image (SimLOD.download_octree()) plus the box and the two batch counters of Stats: the expected file
  encode(nodes, samples, info, counters, box_min, box_max, batchlet_index, num_points_processed)
      the file of a given export and counters (also used to craft files)
  decode(buf)   the header fields as a dict, the records, the counters and the samples of a file's bytes"""
import struct

import numpy as np

import export_restatement as R

MAGIC = b"SIMLODOT"
VERSION = 1
HEADER_SIZE = 128
# magic, version, header_size, info (num_nodes, max_level, num_samples, num_points, num_voxels), box_min, box_max,
# batchlet_index, reserved0, num_points_processed, records_offset, counters_offset, samples_offset, file_size, reserved1
HEADER = struct.Struct("<8sII IIQQQ 3f3f II QQQQQQ")
assert HEADER.size == HEADER_SIZE
FIELDS = ("magic", "version", "header_size", "num_nodes", "max_level", "num_samples", "num_points", "num_voxels",
          "box_min", "box_max", "batchlet_index", "reserved0", "num_points_processed", "records_offset", "counters_offset",
          "samples_offset", "file_size", "reserved1")
COUNTER_OFFSET = 64            # Node::counter


def layout(num_nodes, num_samples):
    records = HEADER_SIZE
    counters = records + 64 * num_nodes
    samples = (counters + 4 * num_nodes + 15) & ~15
    return records, counters, samples, samples + 16 * num_samples


def encode(nodes, samples, info, counters, box_min, box_max, batchlet_index, num_points_processed):
    n, s = len(nodes), len(samples)
    records, counters_at, samples_at, size = layout(n, s)
    head = HEADER.pack(MAGIC, VERSION, HEADER_SIZE, n, int(info.max_level), s, int(info.num_points), int(info.num_voxels),
                       *[float(v) for v in box_min], *[float(v) for v in box_max], int(batchlet_index), 0,
                       int(num_points_processed), records, counters_at, samples_at, size, 0)
    out = bytearray(size)
    out[:HEADER_SIZE] = head
    out[records:counters_at] = np.ascontiguousarray(nodes).tobytes()
    out[counters_at:counters_at + 4 * n] = np.asarray(counters, dtype="<u4").tobytes()
    out[samples_at:] = np.ascontiguousarray(samples).tobytes()
    return bytes(out)


def counters_of(nodes_bytes, records):
    """Node::counter of each record's node: the node of nodes[] with the record's (level, X, Y, Z)."""
    raw = np.frombuffer(np.ascontiguousarray(nodes_bytes, dtype=np.uint8).tobytes(), dtype=np.uint8).reshape(-1, 152)
    words = raw[:, 64:88].copy().view("<u4")                 # counter, numPoints, level, X, Y, Z
    key = {(int(w[2]), int(w[3]), int(w[4]), int(w[5])): int(w[0]) for w in words}
    return np.array([key[(int(r["level"]), int(r["X"]), int(r["Y"]), int(r["Z"]))] for r in records], dtype="<u4")


def file_bytes(nodes_bytes, heap_bytes, nodes_addr, heap_addr, box_min, box_max, batchlet_index, num_points_processed):
    nodes, samples, info = R.export_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr)
    return encode(nodes, samples, info, counters_of(nodes_bytes, nodes), box_min, box_max, batchlet_index, num_points_processed)


def decode(buf):
    vals = HEADER.unpack_from(buf, 0)
    h = {}
    it = iter(vals)
    for f in FIELDS:
        h[f] = tuple(next(it) for _ in range(3)) if f in ("box_min", "box_max") else next(it)
    n, s = h["num_nodes"], h["num_samples"]
    nodes = np.frombuffer(buf, dtype=R.EXPORT_NODE_DTYPE, count=n, offset=h["records_offset"])
    counters = np.frombuffer(buf, dtype="<u4", count=n, offset=h["counters_offset"])
    samples = np.frombuffer(buf, dtype=R.POINT_DTYPE, count=s, offset=h["samples_offset"])
    return h, nodes, counters, samples
