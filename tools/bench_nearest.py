"""k-nearest query cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device). Queries: 1 k, 64 k and 1 M, either stored points of the stream jittered on the surface (sigma 5 cm) or
uniform in the cube; k = 1, 8, 32; depth None (the inserted points) and 5. Per row, after a warm-up, --runs runs with the
L2 flushed before each: kernel ms by stage from the query's events (the export's plan + collect, locate + bucketing,
search; the search writes the destinations, so the write is not timed on its own) as median / min / max, samples tested
and records visited per query, queries/s over the whole kernel time, and whether the repeats were byte-identical.
Beside it what a user does today: scipy cKDTree on the host over the same samples (the eligible ones of the export at
that depth), its build and a 64 k-query k = 8 search timed separately, with the core count; with depth None only when
--host-full is given (the tree over 350 M points takes minutes). Also the card and its power limit.

    python tools/bench_nearest.py [--batches 350] [--runs 5] [--sizes 1000,65536,1048576] [--host-full] [--out result.json]
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

BATCH = 1_000_000
TERRAIN_SEED = 7
SIZES = (1000, 65536, 1 << 20)


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def stats(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(min(v)), 4), "max": round(float(max(v)), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--sizes", default=",".join(str(v) for v in SIZES), help="query counts, comma-separated")
    ap.add_argument("--host-full", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    sizes = [int(v) for v in a.sizes.split(",")]
    import torch
    from simlod_b200 import SimLOD, data

    sim = SimLOD(640, 360, persistent_bytes=a.persistent_gb << 30)
    n = a.batches * BATCH
    dptr = sim.device_alloc(n * 16)
    rng = np.random.default_rng(3)
    try:
        sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, TERRAIN_SEED)
        sim.set_box((0.0, 0.0, 0.0), data.TERRAIN_EXTENT)
        sim.reset()
        sim.insert_device(dptr, n)
        # stored points from all over the scan: 1024 slices of 1024 consecutive points at random positions of the stream
        parts = []
        for first in rng.choice(n // 1024, 1024, replace=False) * 1024:
            sim.generate(sim.GEN_TERRAIN, dptr, n, int(first), 1024, TERRAIN_SEED)
            parts.append(sim.memcpy_dtoh(dptr, 1024 * 16).view(np.float32).reshape(-1, 4)[:, :3].copy())
        stream = np.concatenate(parts)
    finally:
        sim.device_free(dptr)
    st = sim.stats()
    assert st.dbg == 0 and st.numPointsProcessed == n, (st.dbg, st.numPointsProcessed)
    size = float(max(data.TERRAIN_EXTENT))
    kinds = {"surface": stream + rng.normal(0, 0.05, stream.shape).astype(np.float32),
             "uniform": rng.uniform(0, size, (max(SIZES), 3)).astype(np.float32)}
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "runs": a.runs, "rows": [], "host": []}

    dev = torch.device("cuda", 0)
    kmax = 32
    index = torch.empty(max(SIZES) * kmax, dtype=torch.int64, device=dev)
    dist2 = torch.empty(max(SIZES) * kmax, dtype=torch.float32, device=dev)
    for kind, xyz in kinds.items():
        q4 = torch.zeros((max(SIZES), 4), dtype=torch.float32, device=dev)
        q4[:, :3] = torch.from_numpy(xyz).to(dev)
        torch.cuda.synchronize(dev)
        for nq in sizes:
            for k in (1, 8, 32):
                for depth in (None, 5):
                    args = (q4.data_ptr(), nq, k, depth, None, index.data_ptr(), dist2.data_ptr(), 0)
                    sim.query_nearest_into(*args)                                  # warm-up
                    first_i, first_d = index[:nq * k].clone(), dist2[:nq * k].clone()
                    plan, bucket, search, total, identical = [], [], [], [], True
                    for _ in range(a.runs):
                        sim.flush_l2()
                        info, ms = sim.query_nearest_into(*args)
                        plan.append(info.plan_ms); bucket.append(info.bucket_ms); search.append(info.search_ms); total.append(ms)
                        identical &= bool(torch.equal(index[:nq * k], first_i) and torch.equal(dist2[:nq * k], first_d))
                    del first_i, first_d
                    row = {"queries": nq, "kind": kind, "k": k, "depth": "points" if depth is None else depth,
                           "index_space": info.num_samples, "plan_ms": stats(plan), "locate_bucket_ms": stats(bucket),
                           "search_ms": stats(search), "total_ms": stats(total),
                           "samples_tested_per_query": round(info.samples_tested / nq, 1),
                           "records_visited_per_query": round(info.records_visited / nq, 2),
                           "queries_per_s": round(nq / (float(np.median(total)) / 1e3)), "found": info.num_found,
                           "repeats_identical": identical}
                    print(json.dumps(row), flush=True)
                    result["rows"].append(row)

    # what a user does today: download the samples, a k-d tree on the host
    from scipy.spatial import cKDTree
    for depth in ((None, 5) if a.host_full else (5,)):
        ex = sim.export_octree(depth, device="cpu")
        s = ex.samples
        keep = np.ones(len(s), dtype=bool)
        nodes = ex.nodes
        for r in range(len(nodes)):                       # depth None: the points of the leaves only
            o, p, v = int(nodes["sample_offset"][r]), int(nodes["num_points"][r]), int(nodes["num_voxels"][r])
            if depth is None:
                keep[o + p:o + p + v] = False
                if not nodes["flags"][r] & 1:
                    keep[o:o + p] = False
        pts = np.stack([s["x"][keep], s["y"][keep], s["z"][keep]], axis=1).astype(np.float64)
        t0 = time.perf_counter()
        tree = cKDTree(pts)
        build_s = time.perf_counter() - t0
        for kind, xyz in kinds.items():
            t0 = time.perf_counter()
            tree.query(xyz[:65536].astype(np.float64), k=8, workers=-1)
            query_s = time.perf_counter() - t0
            row = {"depth": "points" if depth is None else depth, "samples": int(len(pts)), "kind": kind, "queries": 65536, "k": 8,
                   "build_s": round(build_s, 2), "query_s": round(query_s, 3), "cores": os.cpu_count()}
            print(json.dumps(row), flush=True)
            result["host"].append(row)
        del tree, pts, ex
    sim.close()
    print(json.dumps({"card": result["card"], "points": n, "nodes_in_octree": st.numNodes}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
