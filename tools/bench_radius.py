"""Radius query cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device). Queries: 1 k, 64 k and 1 M, either stored points of the stream jittered on the surface (sigma 5 cm) or
uniform in the cube; r = 0.25, 1 and 4 m; depth None (the inserted points) and 5. Per row, after a warm-up, --runs full
calls with the L2 flushed before each: kernel ms by stage from the query's events (the export's plan + collect, locate +
bucketing, count + offset scan, write) and the size query's kernel ms, as median / min / max; neighbours per query (mean
and max), samples tested and records visited per query (count pass), queries/s over the full call's kernel time, and
whether the repeats were byte-identical (offsets, index, dist2). Beside each row, what a user does today:
query_nearest(k=32, max_radius=r), its kernel ms and the fraction of queries it truncates (more than 32 neighbours);
and for the first 1 k queries, query_region(Region.sphere) once per query, wall ms of the loop. Then scipy cKDTree on the
host over the samples of the depth-5 cut: its build, and query_ball_point of 64 k queries with workers=-1, with the core
count. Also the card and its power limit.

    python tools/bench_radius.py [--batches 350] [--runs 5] [--sizes 1000,65536,1048576] [--out result.json]
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
RADII = (0.25, 1.0, 4.0)


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
    ap.add_argument("--out")
    a = ap.parse_args()
    sizes = [int(v) for v in a.sizes.split(",")]
    import torch
    from simlod_b200 import Region, SimLOD, data

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
    nn_index = torch.empty(max(sizes) * 32, dtype=torch.int64, device=dev)
    nn_dist2 = torch.empty(max(sizes) * 32, dtype=torch.float32, device=dev)
    offsets = torch.empty(max(sizes) + 1, dtype=torch.int64, device=dev)
    for kind, xyz in kinds.items():
        q4 = torch.zeros((max(SIZES), 4), dtype=torch.float32, device=dev)
        q4[:, :3] = torch.from_numpy(xyz).to(dev)
        torch.cuda.synchronize(dev)
        for nq in sizes:
            for r in RADII:
                for depth in (None, 5):
                    qp = q4.data_ptr()
                    sinfo, _ = sim.query_radius_into(qp, nq, r, depth, 0, 0, 0, 0, 0)
                    m = sinfo.num_found
                    index = torch.empty(max(m, 1), dtype=torch.int64, device=dev)
                    dist2 = torch.empty(max(m, 1), dtype=torch.float32, device=dev)
                    args = (qp, nq, r, depth, offsets.data_ptr(), index.data_ptr(), dist2.data_ptr(), 0, m)
                    sim.query_radius_into(*args)                                   # warm-up
                    first = (offsets[:nq + 1].clone(), index[:m].clone(), dist2[:m].clone())
                    plan, bucket, count, write, total, size_ms, identical = [], [], [], [], [], [], True
                    for _ in range(a.runs):
                        sim.flush_l2()
                        _, ms = sim.query_radius_into(qp, nq, r, depth, 0, 0, 0, 0, 0)
                        size_ms.append(ms)
                        sim.flush_l2()
                        info, ms = sim.query_radius_into(*args)
                        plan.append(info.plan_ms); bucket.append(info.bucket_ms); count.append(info.count_ms)
                        write.append(info.write_ms); total.append(ms)
                        identical &= bool(torch.equal(offsets[:nq + 1], first[0]) and torch.equal(index[:m], first[1]) and
                                          torch.equal(dist2[:m], first[2]))
                    counts = torch.diff(first[0]).cpu().numpy()
                    del first, index, dist2
                    # what a user does today: the 32 nearest within r (truncated beyond 32), and a sphere per query
                    nargs = (qp, nq, 32, depth, r, nn_index.data_ptr(), nn_dist2.data_ptr(), 0)
                    sim.query_nearest_into(*nargs)
                    nn_ms = []
                    for _ in range(a.runs):
                        sim.flush_l2()
                        nn_ms.append(sim.query_nearest_into(*nargs)[1])
                    row = {"queries": nq, "kind": kind, "radius": r, "depth": "points" if depth is None else depth,
                           "index_space": info.num_samples, "plan_ms": stats(plan), "locate_bucket_ms": stats(bucket),
                           "count_scan_ms": stats(count), "write_ms": stats(write), "total_ms": stats(total),
                           "size_query_ms": stats(size_ms), "found": int(m),
                           "neighbours_per_query": round(m / nq, 1), "max_found": info.max_found,
                           "samples_tested_per_query": round(info.samples_tested / nq, 1),
                           "records_visited_per_query": round(info.records_visited / nq, 2),
                           "queries_per_s": round(nq / (float(np.median(total)) / 1e3)), "repeats_identical": identical,
                           "nearest32_ms": stats(nn_ms), "nearest32_truncated": round(float((counts > 32).mean()), 4)}
                    if nq == sizes[0]:
                        host = q4[:nq, :3].cpu().numpy()
                        t0 = time.perf_counter()
                        for t in range(nq):
                            sim.query_region(Region.sphere(host[t], r), depth, device="cuda")
                        row["region_sphere_loop_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                    print(json.dumps(row), flush=True)
                    result["rows"].append(row)

    # what a user does today on the host: download the cut at depth 5, a k-d tree, query_ball_point
    from scipy.spatial import cKDTree
    ex = sim.export_octree(5, device="cpu")
    s = ex.samples
    pts = np.stack([s["x"], s["y"], s["z"]], axis=1).astype(np.float64)
    t0 = time.perf_counter()
    tree = cKDTree(pts)
    build_s = time.perf_counter() - t0
    for kind, xyz in kinds.items():
        for r in RADII:
            t0 = time.perf_counter()
            found = tree.query_ball_point(xyz[:65536].astype(np.float64), r, workers=-1, return_length=True)
            query_s = time.perf_counter() - t0
            row = {"depth": 5, "samples": int(len(pts)), "kind": kind, "queries": 65536, "radius": r,
                   "neighbours_per_query": round(float(np.mean(found)), 1), "build_s": round(build_s, 2),
                   "query_s": round(query_s, 3), "cores": os.cpu_count()}
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
