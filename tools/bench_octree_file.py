"""Octree files on one GPU (DESIGN.md §9.7): save and load of the config-3 octree (the 350 M-point device terrain stream)
on tmpfs, beside the rebuild of the same points from a .simlod file through insert_files. For each: wall time and file
GB/s; for save and load also the export / import kernel ms and, for the import, the algorithmic bytes (16 B read + 16 B
written per sample, each grid zeroed and read once, each voxel read back three times) over its kernel time. Best of
--runs. Card name and power limit are read in the same run.

    python tools/bench_octree_file.py [--points 350000000] [--runs 3] [--dir /dev/shm] [--out f.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from simlod_b200 import SimLOD, api, data  # noqa: E402

BATCH = 1_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def write_simlod(path, sim, n, chunk=10 * BATCH):
    """The n-point device terrain stream as a .simlod file (24-byte box header, then 16-byte points)."""
    dptr = sim.device_alloc(chunk * 16)
    try:
        with open(path, "wb") as f:
            f.write(np.array([0, 0, 0, *data.TERRAIN_EXTENT], dtype="<f4").tobytes())
            for first in range(0, n, chunk):
                c = min(chunk, n - first)
                sim.generate(sim.GEN_TERRAIN, dptr, n, first, c, 7)
                f.write(sim.memcpy_dtoh(dptr, c * 16).tobytes())
    finally:
        sim.device_free(dptr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=350_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--dir", default="/dev/shm")
    ap.add_argument("--out")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(dir=args.dir, prefix="simlod_octree_")
    try:
        sim = SimLOD(640, 360)
        src, octree = os.path.join(tmp, "terrain.simlod"), os.path.join(tmp, "terrain.octree")
        write_simlod(src, sim, args.points)
        res = {"card": card(), "points": args.points, "simlod_bytes": os.path.getsize(src)}
        best = {}

        def keep(key, wall, ms):
            if key not in best or wall < best[key][0]:
                best[key] = (wall, ms)
        for _ in range(args.runs):
            t = time.perf_counter()
            _, kms, _ = sim.insert_files([src])
            keep("rebuild", time.perf_counter() - t, kms)
        st = sim.stats()
        assert st.dbg == 0 and st.numPointsProcessed == args.points
        for _ in range(args.runs):
            t = time.perf_counter()
            info, ms = sim.save_octree(octree)
            keep("save", time.perf_counter() - t, ms)
        res["octree_bytes"] = os.path.getsize(octree)
        res["samples"] = info.num_samples
        for _ in range(args.runs):
            t = time.perf_counter()
            _, ms = sim.load_octree(octree)
            keep("load", time.perf_counter() - t, ms)
        st2 = sim.stats()
        assert st2.numNodes == st.numNodes and st2.numPoints == st.numPoints and st2.numVoxels == st.numVoxels
        grids = st.numInner + 1
        # each sample read and written once, each grid zeroed and read for its count, each voxel read back three times
        algo = info.num_samples * 32 + grids * 2 * api.GRID_STRIDE + info.num_voxels * 3 * 16
        for key, (wall, ms) in best.items():
            size = res["simlod_bytes"] if key == "rebuild" else res["octree_bytes"]
            row = {"wall_s": round(wall, 3), "file_GBps": round(size / wall / 1e9, 2), "kernel_ms": round(ms, 1)}
            if key == "load":
                row["algorithmic_GB"] = round(algo / 1e9, 2)
                row["kernel_GBps"] = round(algo / (ms * 1e-3) / 1e9, 1) if ms > 0 else None
            if key == "rebuild":
                row["Gpoints_per_s"] = round(args.points / wall / 1e9, 3)
            res[key] = row
        sim.close()
        line = json.dumps(res)
        print(line)
        if args.out:
            with open(args.out, "w") as f:
                f.write(line + "\n")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
