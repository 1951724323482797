"""Region query cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device): a box over 1 % and over 10 % of the ground area, the whole cube, a 50 m sphere around a position picked on the surface,
a 5 m-wide diagonal corridor across the scene (6 planes) and the frustum of the Morro close camera (6 planes), each at
depth None (the inserted points) and at depth 5. Per row the median of --runs runs with the L2 flushed before every
run, after a warm-up: kernel time of the whole query (plan + collect + count + scan + write events) and of the size
query alone (everything but the write), nodes visited, samples tested and returned, algorithmic bytes (16 B read per
tested sample, counted once although the count and the write kernel each read it, + 16 B written per returned sample)
and the bandwidth they amount to, beside the full export of the same octree, which is what a region query replaces.
Also the card and its power limit, and whether repeated queries were byte-identical.

    python tools/bench_query.py [--batches 350] [--runs 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

BATCH = 1_000_000
TERRAIN_SEED = 7


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def regions():
    from simlod_b200 import Region, camera, data
    ex, ey, ez = data.TERRAIN_EXTENT
    cx, cy = ex / 2, ey / 2

    def ground_box(share):
        f = np.sqrt(share) / 2
        return Region.box((cx - f * ex, cy - f * ey, -1.0), (cx + f * ex, cy + f * ey, ez + 1.0))
    # the corridor follows the diagonal (0, 0) -> (ex, ey): |n . p| <= 2.5 with n the unit normal of the diagonal
    length = float(np.hypot(ex, ey))
    tx, ty = ex / length, ey / length
    nx, ny = -ty, tx
    corridor = [[nx, ny, 0, 2.5], [-nx, -ny, 0, 2.5], [tx, ty, 0, 0], [-tx, -ty, 0, length], [0, 0, 1, 1], [0, 0, -1, ez + 1]]
    view, proj = camera.orbit_camera(width=1920, height=1080, **camera.MORRO_CLOSE)
    m = (np.asarray(proj, dtype=np.float32) @ np.asarray(view, dtype=np.float32)).astype(np.float32)
    frustum = [m[3] + m[0], m[3] - m[0], m[3] + m[1], m[3] - m[1], m[3] + m[2], m[3] - m[2]]
    return [("box 1 % of the ground", ground_box(0.01)), ("box 10 % of the ground", ground_box(0.10)),
            ("whole cube", Region.box((-1.0, -1.0, -1.0), (ex + 1, ex + 1, ex + 1))),
            ("sphere 50 m", Region.sphere((cx, cy, float(data.terrain_height(np.array([cx]), np.array([cy]))[0])), 50.0)),
            ("corridor 5 m", Region.planes(corridor)), ("frustum Morro close", Region.planes(frustum))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
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
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "runs": a.runs, "queries": []}

    dev = torch.device("cuda", 0)
    full, _ = sim.export_octree_into(None, 0, 0, 0, 0)
    nodes_buf = torch.empty(full.num_nodes * 64, dtype=torch.uint8, device=dev)
    buf = torch.empty(full.num_samples * 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    export_args = (None, nodes_buf.data_ptr(), full.num_nodes, buf.data_ptr(), full.num_samples)
    sim.export_octree_into(*export_args)
    export_ms = []
    for _ in range(a.runs):
        sim.flush_l2()
        export_ms.append(sim.export_octree_into(*export_args)[1])
    result["full_export"] = {"samples": full.num_samples, "kernel_ms_median": round(float(np.median(export_ms)), 4)}
    print(json.dumps(result["full_export"]), flush=True)

    for name, region in regions():
        for depth in (None, 5):
            info, _ = sim.query_region_into(region, depth, 0, 0)
            m = info.num_samples
            args = (region, depth, buf.data_ptr() if m else 0, m)
            sim.query_region_into(*args)                                  # warm-up
            first = buf[:m * 16].clone()
            size_ms, kernel_ms, identical = [], [], True
            for _ in range(a.runs):
                sim.flush_l2()
                size_ms.append(sim.query_region_into(region, depth, 0, 0)[1])
                sim.flush_l2()
                kernel_ms.append(sim.query_region_into(*args)[1])
                identical &= bool(torch.equal(buf[:m * 16], first))
            del first
            ms = float(np.median(kernel_ms))
            nbytes = 16 * info.samples_tested + 16 * m
            row = {"region": name, "depth": "points" if depth is None else depth, "nodes_visited": info.nodes_visited,
                   "samples_tested": info.samples_tested, "samples_returned": m, "points": info.num_points, "voxels": info.num_voxels,
                   "kernel_ms_median": round(ms, 4), "kernel_ms_min": round(min(kernel_ms), 4), "kernel_ms_max": round(max(kernel_ms), 4),
                   "size_query_ms_median": round(float(np.median(size_ms)), 4), "algorithmic_bytes": nbytes,
                   "achieved_gb_per_s": round(nbytes / ms / 1e6, 1), "repeated_queries_identical": identical}
            print(json.dumps(row), flush=True)
            result["queries"].append(row)
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
