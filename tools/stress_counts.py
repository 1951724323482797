"""Repeat full builds of a device-generated stream and check that no point is lost (developer aid for rare races).
usage: stress_counts.py [batches=120] [passes=20]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from simlod_b200 import SimLOD, data  # noqa: E402

NB = int(sys.argv[1]) if len(sys.argv) > 1 else 120
P = int(sys.argv[2]) if len(sys.argv) > 2 else 20
n = NB * 1_000_000
sim = SimLOD(640, 360, persistent_bytes=max(4 << 30, NB * (60 << 20)))
sim.set_box((0, 0, 0), data.TERRAIN_EXTENT)
dptr = sim.device_alloc(n * 16)
sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
NODE = np.dtype({"names": ["child0", "counter", "numPoints", "level", "X", "Y", "Z", "numVoxels", "numVoxelsStored"], "formats": ["<u8", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4", "<u4"],
                 "offsets": [0, 64, 68, 72, 76, 80, 84, 144, 148], "itemsize": 152})
good = None
bad = 0
ref = None
if len(sys.argv) > 3 and sys.argv[3] != "-":
    import subprocess
    out = os.path.join(ROOT, "tools", "exp", "stress_variant.cubin")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin"] + sys.argv[3].split(",") + ["-o", out, os.path.join(ROOT, "simlod_b200", "csrc", "construct.cu")])
    sim.use_module(0, out)
    print("variant", sys.argv[3], flush=True)
for p in range(P):
    sim.reset()
    sim.insert_device(dptr, n)
    st = sim.stats()
    nodes = np.frombuffer(sim.memcpy_dtoh(sim.buffers().nodes, st.numNodes * 152).tobytes(), dtype=NODE)
    leaf = nodes["child0"] == 0
    key = (st.numNodes, st.numPoints, st.numVoxels, int(nodes["counter"][leaf].sum()), int(nodes["numPoints"][leaf].sum()), int(nodes["counter"][~leaf].astype(np.uint64).sum()))
    ev = sim.memcpy_dtoh(sim.buffers().momentary + 976, 16).view(np.uint32)
    keys = {(int(r["level"]), int(r["X"]), int(r["Y"]), int(r["Z"])): (int(r["numPoints"]), int(r["counter"]), int(r["numVoxels"]), bool(r["child0"] == 0)) for r in nodes}
    ok = st.numPoints == n and st.dbg & 0x7f == 0
    if ref is None and ok:
        ref = key
        good = keys
    if not ok or (ref is not None and key != ref):
        bad += 1
        print("pass", p, "MISMATCH", key, "expected", ref, "dbg", st.dbg, "events(legacy rounds, list-full warps, table-full, refused)", ev.tolist(), flush=True)
        if good is not None:
            shown = 0
            for k_, v in sorted(keys.items()):
                g = good.get(k_)
                if g != v and shown < 12:
                    print("     node level %d X %d Y %d Z %d: numPoints/counter/numVoxels/leaf got %s expected %s" % (k_ + (v, g)), flush=True)
                    shown += 1
    else:
        print("pass", p, "ok", key, "events", ev.tolist(), flush=True)
print("bad passes", bad, "of", P)
sim.close()
