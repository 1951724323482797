"""LAS writer rates on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device). Three writes: depth None (every inserted point), depth 5 (the cut at 5), and a 64 k-sample
query_region result. Each at 1, 4, 8 and 16 writer threads: wall s of the call, file GB/s, and from the call's info the
plan, gather + encode and device-to-host copy event times. Beside them, the path users had before: data.write_las of
export_octree(20, device="cpu").samples, for depth 5 and, when the host has the memory and the target the space, the
full cloud; and save_octree of the same octree as the file-rate reference. One file per run is read back and checked
against tests/las_write_restatement.py. Also the card and its power limit.

The target directory's free space is checked before every write; a row that does not fit is skipped and says so.

    python tools/bench_write_las.py [--dir /dev/shm] [--batches 350] [--threads 1,4,8,16] [--out result.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))



BATCH = 1_000_000
TERRAIN_SEED = 7


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def fits(directory, nbytes):
    return shutil.disk_usage(directory).free > nbytes + (1 << 30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default="/dev/shm")
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--threads", default="1,4,8,16")
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--out")
    a = ap.parse_args()
    threads = [int(v) for v in a.threads.split(",")]
    import las_write_restatement as W
    from simlod_b200 import Region, SimLOD, data

    work = os.path.join(a.dir, "bench_write_las.%d" % os.getpid())
    os.makedirs(work)
    sim = SimLOD(640, 360, persistent_bytes=a.persistent_gb << 30)
    try:
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
        assert st.dbg == 0 and st.numPointsProcessed == n
        region, _ = sim.query_region(Region.box((1000.0, 1000.0, 0.0), (1070.0, 1070.0, 300.0)), None)
        region = region[:65536].contiguous()
        result = {"card": card(), "points": n, "dir": a.dir, "host_cores": os.cpu_count(), "rows": [], "host": [], "skipped": []}
        path = os.path.join(work, "out.las")
        sources = [("depth None", None, None), ("depth 5", None, 5), ("query_region 64k", region, None)]
        verified = False
        for label, samples, depth in sources:
            for th in threads:
                count = len(samples) if samples is not None else sim.export_octree_into(20 if depth is None else depth, 0, 0, 0, 0)[0].num_samples
                size = 227 + 26 * count
                if not fits(a.dir, size):
                    result["skipped"].append({"write": label, "threads": th, "bytes": size})
                    continue
                t0 = time.perf_counter()
                info = sim.write_las(path, samples, depth, scale=0.001, writer_threads=th)
                wall = time.perf_counter() - t0
                row = {"write": label, "threads": th, "records": info.num_points, "bytes": info.file_size, "windows": info.num_windows,
                       "wall_s": round(wall, 4), "file_GBps": round(info.file_size / wall / 1e9, 3), "plan_ms": round(info.plan_ms, 3),
                       "gather_encode_ms": round(info.encode_ms, 3), "d2h_ms": round(info.copy_ms, 3)}
                if not verified and depth == 5:
                    want, _ = W.file_bytes(sim.export_octree(5, device="cpu").samples, 0.001)
                    with open(path, "rb") as f:
                        row["verified"] = f.read() == want
                    assert row["verified"], "written file differs from the restatement"
                    verified = True
                result["rows"].append(row)
                print(json.dumps(row), flush=True)
                os.unlink(path)
        # the path users had before: export to the host, encode in numpy, write
        need_full = 227 + 26 * n
        for label, depth in (("depth 5", 5), ("depth None", None)):
            e_samples = sim.export_octree_into(20 if depth is None else depth, 0, 0, 0, 0)[0].num_samples
            size = 227 + 26 * e_samples
            # the export (16 B), the records (26 B) and numpy's float64 temporaries (about 48 B) per sample
            if not fits(a.dir, size) or mem_available() < 100 * e_samples:
                result["skipped"].append({"write": "data.write_las " + label, "bytes": size, "mem_available": mem_available()})
                continue
            t0 = time.perf_counter()
            s = sim.export_octree(20 if depth is None else depth, device="cpu").samples
            t1 = time.perf_counter()
            data.write_las(path, s, fmt=2, scale=(0.001,) * 3)
            t2 = time.perf_counter()
            row = {"write": "data.write_las " + label, "records": len(s), "bytes": size, "export_s": round(t1 - t0, 3),
                   "encode_write_s": round(t2 - t1, 3), "wall_s": round(t2 - t0, 3), "file_GBps": round(size / (t2 - t0) / 1e9, 3)}
            del s
            result["host"].append(row)
            print(json.dumps(row), flush=True)
            os.unlink(path)
        # save_octree of the same octree: the file-rate reference (one fwrite thread)
        octree = os.path.join(work, "o.octree")
        if fits(a.dir, 16 * need_full // 26 + (1 << 30)):
            t0 = time.perf_counter()
            info, ms = sim.save_octree(octree)
            wall = time.perf_counter() - t0
            size = os.path.getsize(octree)
            row = {"write": "save_octree", "bytes": size, "wall_s": round(wall, 3), "file_GBps": round(size / wall / 1e9, 3), "kernel_ms": round(ms, 3)}
            result["host"].append(row)
            print(json.dumps(row), flush=True)
            os.unlink(octree)
        else:
            result["skipped"].append({"write": "save_octree"})
    finally:
        sim.close()
        shutil.rmtree(work, ignore_errors=True)
    print(json.dumps({"card": result["card"], "skipped": result["skipped"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
