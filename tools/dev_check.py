"""Developer loop on the GPU box: parity of the builder against the CPU oracle and the reference kernels on a handful of
streams — each once with one batch per launch and once with multi-batch launches (the pipelined path) — then timing
and per-phase times on device-generated terrain streams. Uses oracle/ as the checker (see oracle/README.md).

  python tools/dev_check.py [--quick] [--sizes 36,120]
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from simlod_b200 import SimLOD, data  # noqa: E402

BATCH = 1_000_000
PHASES = ["fused", "split", "rewalk", "deferred", "final_alloc", "final_insert", "rounds(count)", "prologue"]
quick = "--quick" in sys.argv
sizes = [36]
if "--sizes" in sys.argv:
    sizes = [int(x) for x in sys.argv[sys.argv.index("--sizes") + 1].split(",")]
HAVE_REF = all(os.path.exists(p) for p in oracle.REF_CUBINS.values())
fails = 0


def report(label, diffs):
    global fails
    if diffs:
        fails += 1
        print("FAIL", label, diffs[:3], flush=True)
    else:
        print("ok  ", label, flush=True)


def build(sim, batches, box, per_launch, reference=False):
    for p in (0, 2):
        sim.use_module(p, oracle.REF_CUBINS[p] if reference else None)
    sim.set_box(*box)
    sim.reset()
    if per_launch == 1:
        sim.insert_batches(batches)
    else:
        done, i = 0, 0
        while i < len(batches):
            for b in batches[i:i + per_launch]:
                sim.upload_batch(b)
            i += per_launch
            while sim.stats().batchletIndex < min(i, len(batches)):
                sim.update_octree()
    st = sim.stats()
    cn = oracle.canon_from_image(*sim.download_octree())
    for p in (0, 2):
        sim.use_module(p, None)
    return st, cn


def split(points, sizes):
    out, s = [], 0
    for n in sizes:
        out.append(points[s:s + n]); s += n
    return out


sim = SimLOD(1920, 1080, momentary_bytes=oracle.REF_MOMENTARY_BYTES, persistent_bytes=24 << 30)
print(sim.launch_info(), flush=True)

cases = []
pts, mn, mx = data.uniform_cube(1_000_000)
cases.append(("uniform 1M single batch", [pts], (mn, mx), 0.0))
pts, mn, mx = data.terrain(3_300_000)
cases.append(("terrain ragged", split(pts, [1_000_000, 1_000_000, 7, 0, 900_000, 3_300_000 - 2_900_007]), (mn, mx), None))
pts, mn, mx = data.uniform_cube(120_000, size=64.0, seed=5)
cases.append(("leaf root grows then splits", split(pts, [20_000, 20_000, 10_000, 1, 30_000, 39_999]), (mn, mx), 0.0))
if not quick:
    pts, mn, mx = data.shell(2_400_000)
    cases.append(("shell 2.4M", list(data.batches(pts)), (mn, mx), 0.0))
    pts, mn, mx = data.uniform_cube(3_000_000, size=2048.0, seed=77)
    cases.append(("uniform 3x1M incoherent", list(data.batches(pts)), (mn, mx), 0.0))
    pts, mn, mx = data.terrain(12_000_000)
    cases.append(("terrain 12M", list(data.batches(pts)), (mn, mx), None))

for name, batches, box, rcp in cases:
    if rcp is None:
        rcp = float(sim.device_rcp(max(b - a for a, b in zip(*box))))
    t0 = time.time()
    o = oracle.Oracle(box[0], box[1], rcp)
    for b in batches:
        o.add_batch(b)
    ost, ocn = o.stats(), o.canon()
    for per_launch in (1, 20, 3):
        st, cn = build(sim, batches, box, per_launch)
        d = oracle.compare_canon(cn, ocn, "ours") + oracle.compare_stats(st, ost)
        if st.dbg:
            d.append("dbg=%#x" % st.dbg)
        bad = o.check_voxel_colors(cn)
        if bad:
            d.append("%d voxel colour violations" % bad)
        report("%s | %d batch(es)/launch vs oracle" % (name, per_launch), d)
    if HAVE_REF:
        st_r, cn_r = build(sim, batches, box, 1, reference=True)
        report("%s | reference kernels vs oracle" % name, oracle.compare_canon(cn_r, ocn, "ref") + oracle.compare_stats(st_r, ost))
    print("     (%.1f s)" % (time.time() - t0), flush=True)

# ---- timing on device-generated terrain streams ---------------------------------------------------
# the shipped kernel carries no timers; a -DSIMLOD_TIMERS=2 build of the same source gives the per-phase picture
import subprocess  # noqa: E402
timed = os.path.join(ROOT, "tools", "exp", "dev_timers2.cubin")
os.makedirs(os.path.dirname(timed), exist_ok=True)
r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin", "-DSIMLOD_TIMERS=2", "-o", timed,
                    os.path.join(ROOT, "simlod_b200", "csrc", "construct.cu")], capture_output=True, text=True)
if r.returncode != 0:
    print("timers build failed:", r.stderr[-300:]); timed = None
SUBS = ["f.alloc", "f.count", "f.wait", "f.flush", "f.insert", "f.barrier", "s.work", "s.barrier", "r.items", "r.flush", "r.barrier", "f.top", "r.setup", "r.listed", "r.spilled"]
for K in sizes:
    n = K * BATCH
    dptr = sim.device_alloc(n * 16)
    sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
    sim.set_box((0, 0, 0), data.TERRAIN_EXTENT)
    for module in (None, timed):
        if module is None and False:
            continue
        sim.use_module(0, module)
        best = None
        for rep in range(3):
            sim.reset(); sim.flush_l2()
            kms, tms = sim.insert_device(dptr, n)
            st = sim.stats()
            assert st.numPoints == n and st.dbg == 0, (st.numPoints, st.dbg)
            ph = sim.memcpy_dtoh(sim.buffers().momentary + 96, 64).view(np.uint64).astype(np.float64)
            sub = sim.memcpy_dtoh(sim.buffers().momentary + 800, 128).view(np.uint64).astype(np.float64)
            ev = sim.memcpy_dtoh(sim.buffers().momentary + 976, 16).view(np.uint32).tolist()
            if best is None or kms < best[0]:
                best = (kms, tms, ph, sub, ev)
                hist = sim.memcpy_dtoh(sim.buffers().momentary + 1008, 12 * 32).view(np.uint64).reshape(12, 4)
        kms, tms, ph, sub, ev = best
        vb = sim.memcpy_dtoh(sim.buffers().momentary + 64, 32).view(np.uint64)
        print("terrain %dM [%s]: kernel %.3f ms = %.0f Mpts/s, total %.3f ms = %.0f Mpts/s | voxels fresh/rewalk %d/%d spilled %d | nodes %d"
              % (K, "shipped" if module is None else "timers=2 build", kms, n / kms / 1e3, tms, n / tms / 1e3, int(vb[0]), int(vb[1]), int(vb[2]), st.numNodes), flush=True)
        print("   events (legacy rounds, list-full warps, table-full counts, refused splits): %s" % ev, flush=True)
        if ph.sum() > 0:
            print("   us/batch %s | rounds/batch %.2f" % ({k: round(float(v) / 1e3 / K, 1) for k, v in zip(PHASES, ph) if k != "rounds(count)"}, ph[6] / K), flush=True)
            print("   block 0 timeline, us/batch:", {k: round(float(v) / 1e3 / K, 1) for k, v in zip(SUBS, sub)}, flush=True)
            for cls in range(12):
                r_, ns, li, sp = [int(x) for x in hist[cls]]
                if r_:
                    print("   rounds moving < %8d items: %5d rounds, %7.1f us each (split + re-walk), listed %8.0f + spilled %8.0f items per round, %5.1f %% of the round time"
                          % (1 << (2 * cls + 1), r_, ns / r_ / 1e3, li / r_, sp / r_, 100.0 * ns / max(1, int(hist[:, 1].sum()))), flush=True)
        if timed is None:
            break
    sim.use_module(0, None)
    if K == sizes[0]:
        # the device generator against numpy on a slice in the middle of the stream
        f0 = (n // 2) - 50_000
        host = sim.memcpy_dtoh(dptr + f0 * 16, 100_000 * 16).view(data.POINT_DTYPE)
        want = data.terrain(n, f0, 100_000, seed=7)[0]
        report("device terrain generator == numpy", [] if host.tobytes() == want.tobytes() else ["%d points differ" % int((host.view(np.uint32).reshape(-1, 4) != want.view(np.uint32).reshape(-1, 4)).any(axis=1).sum())])
    sim.device_free(dptr)
sim.close()
print("FAILS", fails)
sys.exit(1 if fails else 0)
