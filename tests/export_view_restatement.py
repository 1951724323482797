"""TEST INFRASTRUCTURE — CPU restatement of simlod_export_view (DESIGN.md §9.5): what the device must write for the LOD
cut of a frame, computed independently of simlod_b200 (which it checks), on top of export_restatement (§9.4).

  drawn_from_flags(nodes_bytes)   the nodes a kernel_render frame drew, from the visible / isLarge flags it left in
      nodes[] (the renderer's second pass, integer logic only)
  export_view_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, drawn)   the view export of a raw device image for
      the drawn set `drawn` (one bool per node of nodes[]), byte-exact like export_restatement.export_image, whose
      breadth-first walk, validation, chunk-list walk and error codes it uses

Both return what export_restatement does; export_view_image raises export_restatement.ExportError."""
import numpy as np

import export_restatement as R

# Node::visible, Node::isLarge (include/simlod_abi.h): written for every node by kernel_render
VISIBLE_BYTE, IS_LARGE_BYTE = 116, 119
NODE_BYTES = 152


def drawn_from_flags(nodes_bytes):
    """The nodes a kernel_render frame drew, from the flags it left in nodes[] (render.cu's second pass, integer logic
    only, so exact): a node is drawn when it is visible and either it is a large leaf, or it is not large and its parent
    is large. The parent is the node one level up at (X/2, Y/2, Z/2), whose flags the same frame wrote."""
    raw = np.ascontiguousarray(nodes_bytes, dtype=np.uint8).reshape(-1, NODE_BYTES)
    nodes = np.frombuffer(raw.tobytes(), dtype=R.NODE_DTYPE)
    visible, large = raw[:, VISIBLE_BYTE] != 0, raw[:, IS_LARGE_BYTE] != 0
    leaf = (nodes["children"] == 0).all(axis=1)
    key = {(int(l), int(x), int(y), int(z)): i for i, (l, x, y, z) in enumerate(zip(nodes["level"], nodes["X"], nodes["Y"], nodes["Z"]))}
    drawn = visible & large & leaf
    for i in np.nonzero(visible & ~large & (nodes["level"] > 0))[0]:
        p = key.get((int(nodes["level"][i]) - 1, int(nodes["X"][i]) >> 1, int(nodes["Y"][i]) >> 1, int(nodes["Z"][i]) >> 1))
        drawn[i] = p is not None and bool(large[p])
    return drawn


def _with_counts(nodes, keep):
    """nodes[] as bytes with numPoints / numVoxelsStored zeroed wherever `keep` is False: export_image then walks those
    nodes' children but none of their lists."""
    out = nodes.copy()
    out["numPoints"][~keep] = 0
    out["numVoxelsStored"][~keep] = 0
    return out.view(np.uint8)


def _kept_records(drawn, rec_node, parent):
    """Of the full breadth-first records: the kept ones (the root and the 8 children of every record with a drawn record
    strictly below it), in order, and which records are marked (have one below)."""
    n = len(rec_node)
    marked = np.zeros(n, dtype=bool)
    for r in range(n):
        if drawn[rec_node[r]]:
            p = parent[r]
            while p >= 0 and not marked[p]:
                marked[p] = True
                p = parent[p]
    kept = [r for r in range(n) if parent[r] < 0 or marked[parent[r]]]
    return kept, marked


def export_view_image(nodes_bytes, heap_bytes, nodes_addr, heap_addr, drawn):
    """The view export of a raw device image for the drawn set `drawn` (one bool per node of nodes[]): the same
    validation and error codes as export_image, plus ERR_CHILD for a drawn node the breadth-first pass does not reach
    exactly once. Stages as on the device: the full breadth-first records (errors in the hierarchy), the drawn count,
    then the lists of the drawn nodes alone (errors in those lists)."""
    nodes = np.frombuffer(np.ascontiguousarray(nodes_bytes, dtype=np.uint8).tobytes(), dtype=R.NODE_DTYPE)
    drawn = np.asarray(drawn, dtype=bool)
    if len(drawn) != len(nodes):
        raise ValueError("%d drawn flags for %d nodes" % (len(drawn), len(nodes)))
    # every reachable node's record, no list walked
    full, _, _ = R.export_image(_with_counts(nodes, np.zeros(len(nodes), dtype=bool)), heap_bytes, nodes_addr, heap_addr)
    rec_node = [0] * len(full)
    for r in np.nonzero(full["first_child"] >= 0)[0]:
        fc = int(full["first_child"][r])
        for k in range(8):
            rec_node[fc + k] = (int(nodes["children"][rec_node[r]][k]) - nodes_addr) // NODE_BYTES
    if sum(bool(drawn[i]) for i in rec_node) != int(drawn.sum()):
        raise R.ExportError(R.ERR_CHILD)
    kept, marked = _kept_records(drawn, rec_node, full["parent"])
    # the same records with both lists of every drawn node and nothing else; the records dropped carry no samples, so
    # the sample array and the kept records' offsets are the view's
    rec, samples, info = R.export_image(_with_counts(nodes, drawn), heap_bytes, nodes_addr, heap_addr)
    index = np.full(len(rec), -1, dtype=np.int64)
    index[kept] = np.arange(len(kept))
    out = rec[kept].copy()
    out["parent"] = [-1 if p < 0 else index[p] for p in rec["parent"][kept]]
    out["first_child"] = [index[fc] if marked[r] else -1 for r, fc in zip(kept, rec["first_child"][kept])]
    out["flags"] = [(int(f) & R.LEAF) | (R.SAMPLED if drawn[rec_node[r]] else 0) for r, f in zip(kept, rec["flags"][kept])]
    info.num_nodes = len(kept)
    return out, samples, info
