"""Octree export throughput on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device): the full export and the cuts at depths 3, 5 and 7, each the median of --runs runs with the L2 flushed
before every run, after a warm-up. Reports kernel time (plan + collect + gather events), Gsamples/s and achieved
bandwidth in algorithmic bytes (16 B read + 16 B written per sample, 152 B read + 64 B written per node) against the
H100 SXM data sheet's 3.35 TB/s, the host path (download_octree + canon_from_image) once, the card and its power
limit, and whether the repeated exports were byte-identical.

    python tools/bench_export.py [--batches 350] [--runs 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

PEAK_GBS = 3350.0
BATCH = 1_000_000
TERRAIN_SEED = 7


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import oracle
    from simlod_b200 import SimLOD, data

    sim = SimLOD(640, 360, persistent_bytes=a.persistent_gb << 30)
    n = a.batches * BATCH
    dptr = sim.device_alloc(n * 16)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, TERRAIN_SEED)
        sim.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.reset()
        sim.insert_device(dptr, n)
    finally:
        sim.device_free(dptr)
    st = sim.stats()
    assert st.dbg == 0 and st.numPointsProcessed == n, (st.dbg, st.numPointsProcessed)
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "heap_bytes": int(st.allocatedBytes_persistent),
              "runs": a.runs, "exports": []}

    full, _ = sim.export_octree_into(None, 0, 0, 0, 0)
    dev = torch.device("cuda", 0)
    nodes_buf = torch.empty(full.num_nodes * 64, dtype=torch.uint8, device=dev)
    samples_buf = torch.empty(full.num_samples * 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    for depth in (None, 3, 5, 7):
        info, plan_ms = sim.export_octree_into(depth, 0, 0, 0, 0)     # size query: plan + collect only
        args = (depth, nodes_buf.data_ptr(), info.num_nodes, samples_buf.data_ptr() if info.num_samples else 0, info.num_samples)
        sim.export_octree_into(*args)                                  # warm-up
        torch.cuda.synchronize(dev)
        first_nodes = nodes_buf[:info.num_nodes * 64].clone()
        first_samples = samples_buf[:info.num_samples * 16].clone()
        kernel_ms, wall_ms, identical = [], [], True
        for _ in range(a.runs):
            sim.flush_l2()
            t0 = time.perf_counter()
            _, ms = sim.export_octree_into(*args)
            wall_ms.append((time.perf_counter() - t0) * 1e3)
            kernel_ms.append(ms)
            identical &= bool(torch.equal(nodes_buf[:info.num_nodes * 64], first_nodes)) and \
                bool(torch.equal(samples_buf[:info.num_samples * 16], first_samples))
        del first_nodes, first_samples
        torch.cuda.empty_cache()
        ms = float(np.median(kernel_ms))
        nbytes = 32 * info.num_samples + (152 + 64) * info.num_nodes
        result["exports"].append({
            "depth": "full" if depth is None else depth, "nodes": info.num_nodes, "samples": info.num_samples,
            "points": info.num_points, "voxels": info.num_voxels,
            "kernel_ms_median": round(ms, 4), "kernel_ms_min": round(min(kernel_ms), 4), "kernel_ms_max": round(max(kernel_ms), 4),
            "plan_collect_ms": round(plan_ms, 4), "wall_ms_median": round(float(np.median(wall_ms)), 4),
            "gsamples_per_s": round(info.num_samples / ms / 1e6, 3), "algorithmic_bytes": nbytes,
            "achieved_gb_per_s": round(nbytes / ms / 1e6, 1), "share_of_3350_gb_per_s": round(nbytes / ms / 1e6 / PEAK_GBS, 4),
            "repeated_exports_identical": identical})
        print(json.dumps(result["exports"][-1]), flush=True)
    del nodes_buf, samples_buf
    torch.cuda.empty_cache()

    t0 = time.perf_counter()
    image = sim.download_octree()
    t1 = time.perf_counter()
    canon = oracle.canon_from_image(*image)
    t2 = time.perf_counter()
    result["host_path"] = {"download_octree_s": round(t1 - t0, 3), "canon_from_image_s": round(t2 - t1, 3),
                           "image_bytes": int(len(image[0]) + len(image[1])), "nodes": len(canon.records)}
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
