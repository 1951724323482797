"""Height map cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with insert_device).
Grids: 10 m and 1 m over the whole terrain, 0.25 m over a 1 km x 1 km tile; depth None (the inserted points) and 5; all
six destinations and the count alone. Per row, after a warm-up, --runs runs with the L2 flushed before each: kernel ms
by stage from the query's events (the export's plan + collect; the reset + accumulate; the finalize) as median / min /
max, samples tested, the bytes the algorithm must move (16 B per sample tested, the accumulators' reset and read-back,
the destinations) and the achieved rate against the H100 SXM data sheet's 3.35 TB/s, and whether the repeats were
byte-identical. Baselines in the same run: export_octree(depth) followed by torch ops that give the same count, z_min
and z_max (wall ms with the L2 flushed before each run, peak torch device memory, and whether the bytes match), and for
the 10 m grid one vertical query_ray per cell centre. Also the card and its power limit.

    python tools/bench_heightmap.py [--batches 350] [--runs 5] [--grids 10m,1m,tile] [--out result.json]
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
HBM_TBPS = 3.35                       # H100 SXM data sheet, not a measured figure


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def stats(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(min(v)), 4), "max": round(float(max(v)), 4)}


def grid_list(ext):
    return {"10m": ((0.0, 0.0), 10.0, (int(np.ceil(ext[1] / 10)), int(np.ceil(ext[0] / 10)))),
            "1m": ((0.0, 0.0), 1.0, (int(np.ceil(ext[1])), int(np.ceil(ext[0])))),
            "tile": ((1900.0, 1600.0), 0.25, (4000, 4000))}


def torch_baseline(sim, torch, depth, origin, cell, shape, rcp, mn, size):
    """export_octree(depth), then the sample set, the cell of every sample and count / z_min / z_max with torch ops."""
    ny, nx = shape
    ex = sim.export_octree(depth)
    nodes, s = ex.nodes, ex.samples
    dev = s.device
    counts = np.stack([nodes["num_points"], nodes["num_voxels"]], axis=1).reshape(-1).astype(np.int64)
    if depth is None:                                      # the leaves' points only
        leaf = (nodes["flags"] & 1) != 0
        keep = np.stack([leaf, np.zeros(len(nodes), dtype=bool)], axis=1).reshape(-1)
    else:                                                  # every point and voxel of the cut
        keep = np.ones(2 * len(nodes), dtype=bool)
    voxel = np.tile([False, True], len(nodes))
    kind = torch.repeat_interleave(torch.as_tensor(keep * 1 + voxel * 2, device=dev), torch.as_tensor(counts, device=dev))
    x, y, z = s[:, 0], s[:, 1], s[:, 2]
    ok = (kind & 1) == 1
    pt = ok & ((kind & 2) == 0)
    for p, m in ((x, mn[0]), (y, mn[1]), (z, mn[2])):     # the in-cube test of the points
        q = ((p + np.float32(-m)) * np.float32(1048576.0)) * np.float32(rcp)
        inside = (p >= np.float32(m)) & (q >= 0) & (torch.trunc(q) < 1048576.0)
        ok &= ~pt | inside
    u = (x - np.float32(origin[0])) / np.float32(cell)
    v = (y - np.float32(origin[1])) / np.float32(cell)
    ok &= (u >= 0) & (v >= 0) & (torch.trunc(u) < nx) & (torch.trunc(v) < ny)
    cid = (torch.trunc(v[ok]).to(torch.int64) * nx + torch.trunc(u[ok]).to(torch.int64))
    zb = z[ok].contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    oz = torch.where(zb >= 0x80000000, zb ^ 0xFFFFFFFF, zb | 0x80000000)
    count = torch.bincount(cid, minlength=nx * ny)
    lo = torch.full((nx * ny,), 1 << 33, dtype=torch.int64, device=dev).scatter_reduce_(0, cid, oz, "amin")
    hi = torch.full((nx * ny,), -1, dtype=torch.int64, device=dev).scatter_reduce_(0, cid, oz, "amax")

    def back(o, empty):
        b = torch.where(o >= 0x80000000, o & 0x7FFFFFFF, o ^ 0xFFFFFFFF)
        b = torch.where(empty, torch.full_like(b, 0x7FC00000), b)
        return b.to(torch.int32).view(torch.float32).reshape(ny, nx)
    empty = count == 0
    out = count.reshape(ny, nx), back(lo, empty), back(hi, empty)
    torch.cuda.synchronize(dev)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--grids", default="10m,1m,tile")
    ap.add_argument("--radius", type=float, default=0.05, help="radius of the vertical-ray baseline")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    from simlod_b200 import SimLOD, api, data

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
    ext = np.asarray(data.TERRAIN_EXTENT, dtype=np.float64)
    mn = np.zeros(3, dtype=np.float32)
    size = float(np.float32(ext.max()))
    rcp = sim.device_rcp(size)
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "runs": a.runs, "rows": [], "baselines": []}
    dev = torch.device("cuda", 0)
    grids = grid_list(ext)
    for gname in a.grids.split(","):
        origin, cell, shape = grids[gname]
        cells = shape[0] * shape[1]
        g = api.SimlodHeightmap(cell=cell, nx=shape[1], ny=shape[0])
        g.origin[:] = list(origin)
        for depth in (None, 5):
            for dests in ("all", "count"):
                bufs = [torch.empty(shape, dtype=t, device=dev) for t in (torch.int64, torch.float32, torch.float32, torch.float32, torch.int64)]
                bufs.append(torch.empty(shape + (4,), dtype=torch.float32, device=dev))
                ptrs = [b.data_ptr() for b in bufs] if dests == "all" else [bufs[0].data_ptr(), 0, 0, 0, 0, 0]
                torch.cuda.synchronize(dev)
                sim.query_heightmap_into(g, depth, *ptrs)                          # warm-up
                first = [b.clone() for b in bufs]
                plan, acc, fin, total, identical = [], [], [], [], True
                for _ in range(a.runs):
                    sim.flush_l2()
                    info, ms = sim.query_heightmap_into(g, depth, *ptrs)
                    plan.append(info.plan_ms); acc.append(info.accumulate_ms); fin.append(info.finalize_ms); total.append(ms)
                    identical &= all(torch.equal(b.view(torch.uint8) if b.dtype != torch.int64 else b, f.view(torch.uint8) if f.dtype != torch.int64 else f)
                                     for b, f in zip(bufs, first))
                acc_bytes = 4 + (24 - 4 if dests == "all" else 0)                 # accumulators per cell
                out_bytes = 44 if dests == "all" else 8                           # destinations per cell
                moved = 16 * info.samples_tested + cells * (2 * acc_bytes + out_bytes)
                work_ms = float(np.median(acc)) + float(np.median(fin))
                row = {"grid": gname, "cells": cells, "depth": "points" if depth is None else depth, "dests": dests,
                       "index_space": info.num_samples, "samples_tested": info.samples_tested, "binned": info.num_binned,
                       "nonempty_cells": info.nonempty_cells, "records_visited": info.records_visited,
                       "plan_ms": stats(plan), "accumulate_ms": stats(acc), "finalize_ms": stats(fin), "total_ms": stats(total),
                       "bytes_moved": moved, "accumulate_finalize_GBps": round(moved / work_ms / 1e6, 1),
                       "share_of_3.35TBps_datasheet": round(moved / work_ms / 1e6 / (HBM_TBPS * 1e3), 3),
                       "repeats_identical": identical}
                print(json.dumps(row), flush=True)
                result["rows"].append(row)
                if dests == "all":
                    want = [b.cpu() for b in bufs[:3]]
                del bufs
            # baseline: export + torch for count, z_min, z_max
            torch.cuda.synchronize(dev)
            torch.cuda.empty_cache()
            walls, peak, match = [], 0, True
            for r in range(a.runs + 1):
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                sim.flush_l2()
                t0 = time.perf_counter()
                out = torch_baseline(sim, torch, depth, origin, cell, shape, rcp, mn, size)
                wall = (time.perf_counter() - t0) * 1e3
                if r:
                    walls.append(wall)
                peak = max(peak, torch.cuda.max_memory_allocated(dev) - base)
                match &= all(o.cpu().numpy().tobytes() == w.numpy().tobytes() for o, w in zip(out, want))
                del out
                torch.cuda.empty_cache()
            brow = {"grid": gname, "depth": "points" if depth is None else depth, "baseline": "export + torch",
                    "wall_ms": stats(walls), "peak_torch_bytes": int(peak), "same_bytes_as_heightmap": bool(match)}
            print(json.dumps(brow), flush=True)
            result["baselines"].append(brow)
        if gname == "10m":                                 # one vertical ray per cell centre
            ny, nx = shape
            jj, ii = np.meshgrid(np.arange(ny), np.arange(nx), indexing="ij")
            r = np.zeros((cells, 8), dtype=np.float32)
            r[:, 0] = origin[0] + (ii.reshape(-1) + 0.5) * cell
            r[:, 1] = origin[1] + (jj.reshape(-1) + 0.5) * cell
            r[:, 2] = ext[2] + 100.0
            r[:, 6], r[:, 7] = -1.0, np.inf
            rays = torch.from_numpy(r).to(dev)
            index = torch.empty(cells, dtype=torch.int64, device=dev)
            torch.cuda.synchronize(dev)
            args = (rays.data_ptr(), cells, a.radius, None, index.data_ptr(), 0, 0, 0)
            sim.query_ray_into(*args)
            total = []
            for _ in range(a.runs):
                sim.flush_l2()
                info, ms = sim.query_ray_into(*args)
                total.append(ms)
            brow = {"grid": gname, "depth": "points", "baseline": "vertical query_ray per cell", "radius": a.radius,
                    "total_ms": stats(total), "hits": info.num_hits}
            print(json.dumps(brow), flush=True)
            result["baselines"].append(brow)
            del rays, index
    sim.close()
    print(json.dumps({"card": result["card"], "points": n, "nodes_in_octree": st.numNodes}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
