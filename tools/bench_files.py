"""File-list front end (simlod_insert_files) on one GPU: a terrain scan on tmpfs written as one .simlod file, one LAS
format 2 file (26 B/point), one LAS format 3 file (34 B/point) and 8 format 3 tiles. For each input: the end-to-end wall
rate (reset, box, read, upload, decode, insert), file GB/s, device and kernel ms (best of --runs), beside the reference's
CPU loader on the same files (oracle.ref_las_bench / ref_simlod_bench: host memory only, best of 1 / 8 / all cores).
--profile: one torch.profiler run of the format 3 file; the share of host-to-device copy time that overlaps
kernel_construct launches (the Chrome trace goes to --trace-dir, default profiles/). --parent-tree DIR: bench.py's stream_file row (bench_stream_file) for this tree and for DIR (a
built checkout of another commit), alternating --rounds times. Card name and power limit are read in the same run.

    python tools/bench_files.py [--points 100000000] [--runs 3] [--profile [--trace-dir DIR]] [--parent-tree DIR] [--out f.json]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from simlod_b200 import SimLOD, data  # noqa: E402

BATCH = 1_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def write_las_chunked(path, sim, n, first, count, fmt, chunk=10 * BATCH):
    """A LAS 1.2 file of points [first, first + count) of the n-point device terrain stream, written chunk by chunk."""
    dptr = sim.device_alloc(chunk * 16)
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    try:
        with open(path, "wb") as f:
            f.write(bytes(227))
            for s in range(first, first + count, chunk):
                c = min(chunk, first + count - s)
                sim.generate(sim.GEN_TERRAIN, dptr, n, s, c, 7)
                pts = sim.memcpy_dtoh(dptr, c * 16).view(oracle.POINT_DTYPE)
                for k, ax in enumerate("xyz"):
                    lo[k], hi[k] = min(lo[k], float(pts[ax].min())), max(hi[k], float(pts[ax].max()))
                f.write(data.las_records(pts, fmt).tobytes())
    finally:
        sim.device_free(dptr)
    one = path + ".hdr"
    data.write_las(one, np.zeros(0, dtype=oracle.POINT_DTYPE), fmt=fmt)
    hdr = bytearray(open(one, "rb").read(227))
    os.remove(one)
    struct.pack_into("<I", hdr, 107, count)
    struct.pack_into("<6d", hdr, 179, hi[0], lo[0], hi[1], lo[1], hi[2], lo[2])
    with open(path, "r+b") as f:
        f.write(bytes(hdr))


def write_simlod_chunked(path, sim, n, chunk=10 * BATCH):
    dptr = sim.device_alloc(chunk * 16)
    try:
        with open(path, "wb") as f:
            f.write(struct.pack("<6f", 0.0, 0.0, 0.0, *data.TERRAIN_EXTENT))
            for s in range(0, n, chunk):
                c = min(chunk, n - s)
                sim.generate(sim.GEN_TERRAIN, dptr, n, s, c, 7)
                f.write(sim.memcpy_dtoh(dptr, c * 16).tobytes())
    finally:
        sim.device_free(dptr)


def time_insert(sim, paths, n, runs, threads):
    best = None
    for _ in range(runs):
        t0 = time.perf_counter()
        got, kms, tms = sim.insert_files(paths, loader_threads=threads)
        dt = time.perf_counter() - t0
        assert got == n and sim.stats().numPoints == n, (got, sim.stats().numPoints)
        if best is None or dt < best[0]:
            best = (dt, kms, tms)
    nbytes = sum(os.path.getsize(p) for p in paths)
    return {"points": n, "file_bytes": nbytes, "wall_s": round(best[0], 4), "Mpoints_per_s": round(n / best[0] / 1e6, 1),
            "file_GB_per_s": round(nbytes / best[0] / 1e9, 2), "device_ms": round(best[2], 2), "kernel_ms": round(best[1], 2)}


def reference_loader(paths, n):
    """The reference's CPU loader on the same files into host memory: best of 1 / 8 / all cores, files one after another."""
    if oracle.ref_las() is None:
        return None
    best = None
    for threads in sorted({1, min(8, os.cpu_count() or 1), os.cpu_count() or 1}):
        dt = 0.0
        for p in paths:
            if p.endswith(".las"):
                dt += oracle.ref_las_bench(p, oracle_count(p), BATCH, threads)
            else:
                dt += oracle.ref_simlod_bench(p, (os.path.getsize(p) - 24) // 16, BATCH, threads)
        if best is None or dt < best[0]:
            best = (dt, threads)
    return {"Mpoints_per_s": round(n / best[0] / 1e6, 1), "cores": best[1], "wall_s": round(best[0], 4)}


def oracle_count(path):
    return struct.unpack_from("<I", open(path, "rb").read(111), 107)[0]


def profile_overlap(sim, paths, out_dir):
    """One insert under torch.profiler: H2D copy time, and the part of it that overlaps kernel_construct launches."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        sim.insert_files(paths, loader_threads=16)
    trace = os.path.join(out_dir, "bench_files_trace.json")
    prof.export_chrome_trace(trace)
    ev = json.load(open(trace))["traceEvents"]
    kern = sorted((e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "kernel" and "kernel_construct" in e.get("name", ""))
    h2d = [(e["ts"], e["ts"] + e["dur"]) for e in ev if e.get("cat") == "gpu_memcpy" and "HtoD" in e.get("name", "") and e.get("dur", 0) > 50]
    overlap = 0.0
    for a, b in h2d:
        for c, d in kern:
            overlap += max(0.0, min(b, d) - max(a, c))
    total = sum(b - a for a, b in h2d)
    return {"trace": trace, "construct_launches": len(kern), "h2d_copies": len(h2d),
            "h2d_us": round(total, 1), "h2d_us_during_construct": round(overlap, 1),
            "h2d_share_during_construct": round(overlap / total, 3) if total else None,
            "construct_us": round(sum(d - c for c, d in kern), 1)}


STREAM_ROW = r"""
import json, sys
sys.path.insert(0, '.')
import bench
from simlod_b200 import data
mine = list(range(%d))
batches, mn, mx = data.terrain_batches(%d, mine)
print(json.dumps(bench.bench_stream_file(0, batches, mn, mx)["e2e"]))
"""


def stream_rows(trees, rounds, batches):
    """bench.py's stream_file row in each tree, alternating."""
    rows = {t: [] for t in trees}
    for _ in range(rounds):
        for t in trees:
            r = subprocess.run([sys.executable, "-c", STREAM_ROW % (batches, batches)], cwd=t, stdout=subprocess.PIPE, text=True, check=True)
            rows[t].append(json.loads(r.stdout.strip().splitlines()[-1]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100 * BATCH)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--trace-dir", default=os.path.join(ROOT, "profiles"), help="where --profile writes its Chrome trace")
    ap.add_argument("--parent-tree")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stream-batches", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    n = args.points
    out = {"card": card(), "points": n}
    d = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    base = os.path.join(d, "simlod_files_%d" % os.getpid())
    sim = SimLOD(320, 176, persistent_bytes=max(8 << 30, n * 220))
    results = {}
    try:
        inputs = [("simlod", None), ("las_fmt2", 2), ("las_fmt3", 3), ("las_fmt3_8_tiles", 3)]
        for name, fmt in inputs:
            if fmt is None:
                paths = [base + ".simlod"]
                write_simlod_chunked(paths[0], sim, n)
            elif "tiles" in name:
                paths = [base + "_tile%d.las" % k for k in range(8)]
                for k, p in enumerate(paths):
                    write_las_chunked(p, sim, n, k * n // 8, (k + 1) * n // 8 - k * n // 8, fmt)
            else:
                paths = [base + "_%s.las" % name]
                write_las_chunked(paths[0], sim, n, 0, n, fmt)
            try:
                sim.insert_files(paths, loader_threads=args.threads)          # warm-up: pool, staging, page cache
                r = time_insert(sim, paths, n, args.runs, args.threads)
                r["reference_cpu_loader"] = reference_loader(paths, n)
                if args.profile and name == "las_fmt3":
                    os.makedirs(args.trace_dir, exist_ok=True)
                    r["profile"] = profile_overlap(sim, paths, args.trace_dir)
                results[name] = r
                print(name, json.dumps(r), flush=True)
            finally:
                for p in paths:
                    os.remove(p)
    finally:
        sim.close()
    out["inputs"] = results
    if args.parent_tree:
        rows = stream_rows([ROOT, os.path.abspath(args.parent_tree)], args.rounds, args.stream_batches)
        out["stream_file_alternating"] = {"this": rows[ROOT], "parent": rows[os.path.abspath(args.parent_tree)]}
    out["card_after"] = card()
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
