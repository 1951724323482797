"""Developer tool (not part of bench.py): times the reference's OWN kernels (oracle/_ref/*.cubin) on
the same H100, same harness, same inputs as bench.py's workload — the "R-GPU" baseline of
BASELINE.md §2. Writes one JSON object."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from simlod_b200 import SimLOD, camera, data# noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 36
out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "gpurun_out", "reference_gpu.json")
batches, mn, mx = data.terrain_batches(K, list(range(K)))
npts = K * 1_000_000
res = {"workload": "terrain_synth_%dM, %d x 1M batches" % (K, K)}
for impl in ("reference", "ours"):
    sim = SimLOD(1920, 1080, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=max(8 << 30, K * (220 << 20)),
                 construct_blocks_per_sm=1 if impl == "reference" else 0)
    if impl == "reference":
        for p in (0, 1, 2):
            sim.use_module(p, oracle.REF_CUBINS[p])
    sim.set_box(mn, mx)
    dptr = sim.device_alloc(npts * 16)
    sim.memcpy_htod(dptr, np.concatenate(batches).view(np.uint8))
    sim.reset(); sim.insert_device(dptr, 3 * 1_000_000); sim.reset(); sim.flush_l2()
    kms, tms = sim.insert_device(dptr, npts)
    st = sim.stats()
    assert st.numPoints == npts, (st.numPoints, st.dbg)
    r = {"insert_kernel_ms": kms, "insert_total_ms": tms, "mpoints_per_s_kernel": npts / kms / 1e3, "mpoints_per_s_total": npts / tms / 1e3,
         "construct_blocks": sim.launch_info()["construct_blocks"], "numNodes": st.numNodes, "numVoxels": st.numVoxels}
    frames = []
    for hqs in (0, 1):
        sim.set_settings(useHighQualityShading=hqs)
        for k in range(4):
            view, proj = camera.autofocus(mx, 1920, 1080, yaw_offset=k * np.pi / 2)
            sim.set_camera(view, proj)
            sim.render()
            ms = min(sim.render() for _ in range(3))
            s = sim.stats()
            frames.append({"hqs": hqs, "camera": k, "ms": ms, "samples": s.numVisiblePoints + s.numVisibleVoxels})
    r["render_blocks"] = sim.launch_info()["render_blocks"]
    r["render_frames"] = frames
    for hqs in (0, 1):
        f = [x for x in frames if x["hqs"] == hqs]
        r["render_msamples_per_s_hqs%d" % hqs] = sum(x["samples"] for x in f) / sum(x["ms"] for x in f) / 1e3
    res[impl] = r
    sim.close()
    print(impl, json.dumps({k: v for k, v in r.items() if k != "render_frames"}), flush=True)
res["speedup_insert_kernel"] = res["ours"]["mpoints_per_s_kernel"] / res["reference"]["mpoints_per_s_kernel"]
res["speedup_render_hqs0"] = res["ours"]["render_msamples_per_s_hqs0"] / res["reference"]["render_msamples_per_s_hqs0"]
res["speedup_render_hqs1"] = res["ours"]["render_msamples_per_s_hqs1"] / res["reference"]["render_msamples_per_s_hqs1"]
json.dump(res, open(out, "w"), indent=1)
print("speedups", res["speedup_insert_kernel"], res["speedup_render_hqs0"], res["speedup_render_hqs1"])
