"""What the original SimLOD computes on the inputs of the tests, kept as digests in tests/golden/reference.json so
that every comparison with the original runs without its sources.

The digests were recorded by the unmodified reference code that build() compiles into oracle/_ref/ when the original
sources are at hand: its kernels (oracle/build_ref.cpp), run on an H100 through the same C ABI, buffers and inputs as
ours, and its LAS / .simlod loaders (oracle/ref_*_shim.cpp). To record them again, build oracle/_ref and run the tests
with SIMLOD_RECORD_GOLDEN=<output .json>: each comparison then runs the reference live, checks ours against it, and
writes what the reference computed to that file."""
import hashlib
import json
import os

import numpy as np

import oracle

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference.json")
RECORD = os.environ.get("SIMLOD_RECORD_GOLDEN")
_stored = None
_recorded = {}


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def stats(st):
    """The deterministic Stats fields (oracle.STATS_FIELDS)."""
    return {"stats": {f: int(getattr(st, f)) for f in oracle.STATS_FIELDS}}


def octree(st, canon):
    """Stats plus a digest of the canonical form (every field oracle.compare_canon compares)."""
    rec = canon.records.copy()
    rec["nodeIndex"] = 0
    rec["_pad"] = 0
    return dict(stats(st), nodes=len(rec), canon=sha256(rec))


def points(pts, with_color=True):
    """Points by their float bits; colour under the 24-bit mask (the reference leaves alpha uninitialised)."""
    xyz = [np.ascontiguousarray(pts[ax]).view(np.uint32) for ax in "xyz"]
    return {"count": len(pts), "points": sha256(*xyz, *([pts["color"] & np.uint32(0x00FFFFFF)] if with_color else []))}


def frame(fb, surface, visible, voxels, nodes=None):
    """A rendered frame: the depth word of every pixel, the visible counts, (optionally) the visibility flags of every
    node in canonical (level, X, Y, Z) order and, when no voxel is drawn (`voxels` == 0), the raw u64 framebuffer and
    the RGBA8 surface. Which point donates a voxel's colour is a race in the builders, so the colours of a frame that
    draws voxels differ from build to build; every other colour (point colours, node / LOD colours, HQS sums, EDL) is
    deterministic and compared bit for bit."""
    out = {"depth": sha256(fb >> np.uint64(32)), "visible": [int(v) for v in visible]}
    if voxels == 0:
        out["framebuffer"] = sha256(fb)
        out["surface"] = sha256(surface)
    if nodes is not None:
        rec = nodes.reshape(-1, 152)
        key = rec[:, 72:88].copy().view(np.uint32)
        order = np.lexsort((key[:, 3], key[:, 2], key[:, 1], key[:, 0]))
        out["flags"] = sha256(rec[order][:, [116, 119]])
    return out


def reference(key, run):
    """The reference's result for `key`: run() live (and recorded) with SIMLOD_RECORD_GOLDEN set, else the stored one."""
    global _stored
    if RECORD:
        value = json.loads(json.dumps(run()))
        _recorded[key] = value
        with open(RECORD, "w") as f:
            json.dump(_recorded, f, indent=1, sort_keys=True)
        return value
    if _stored is None:
        with open(PATH) as f:
            _stored = json.load(f)
    assert key in _stored, "no stored reference result for %r in %s" % (key, PATH)
    return _stored[key]


def assert_same(ours, ref, label):
    """Every entry of ours must be identical in the reference result."""
    diffs = []
    for k, got in ours.items():
        want = ref.get(k)
        if isinstance(got, dict):
            diffs += ["%s.%s: %r != %r" % (k, f, v, (want or {}).get(f)) for f, v in got.items() if (want or {}).get(f) != v]
        elif got != want:
            diffs.append("%s: %r != %r" % (k, got, want))
    assert not diffs, "%s:\n%s" % (label, "\n".join(diffs))
