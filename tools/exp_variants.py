"""Developer experiment: build variant cubins of the builder (compile-time knobs of construct.cu, or any *.cubin dropped
into tools/exp/), check each against the shipped kernel (deterministic Stats + canonical octree of a full build) and
time it: whole build (kernel-only, best of 3), and — for variants built with timers — µs per batch per phase.

  python tools/exp_variants.py [batches]           # on the GPU box; nvcc is in the image
"""
import glob
import hashlib
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402  (checker: canonical forms of the two device octrees)
from simlod_b200 import SimLOD, data  # noqa: E402

BATCH = 1_000_000
# name -> extra nvcc flags for simlod_b200/csrc/construct.cu
KNOBS = {
    "timers2": ["-DSIMLOD_TIMERS=2"],
    "timers1": ["-DSIMLOD_TIMERS=1"],
    "occ3": ["-DSIMLOD_BLOCKS_PER_SM=3"],
    "occ5": ["-DSIMLOD_BLOCKS_PER_SM=5"],
    "occ3_t2": ["-DSIMLOD_BLOCKS_PER_SM=3", "-DSIMLOD_TIMERS=2"],
    "tile256": ["-DSIMLOD_TILE_POINTS=256"],
    "rwl2": ["-DSIMLOD_REWALK_L2TEST=1"],
    "tile1024": ["-DSIMLOD_TILE_POINTS=1024"],
}
only = [a for a in sys.argv[1:] if not a.isdigit()]
if only:
    KNOBS = {k: v for k, v in KNOBS.items() if k in only}
K = next((int(a) for a in sys.argv[1:] if a.isdigit()), 36)
EXP = os.path.join(ROOT, "tools", "exp")
os.makedirs(EXP, exist_ok=True)
_h = hashlib.sha256()
for _f in ("simlod_b200/csrc/construct.cu", "simlod_b200/csrc/fpmath.cuh", "include/simlod_abi.h"):
    _h.update(open(os.path.join(ROOT, _f), "rb").read())
SRC_TAG = _h.hexdigest()[:8]                  # variants are rebuilt when the kernel source changes
for name, flags in KNOBS.items():
    out = os.path.join(EXP, "knob_%s_%s.cubin" % (name, SRC_TAG))
    for stale in glob.glob(os.path.join(EXP, "knob_%s_*.cubin" % name)):
        if stale != out:
            os.remove(stale)
    if not os.path.exists(out):
        cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin"] + flags + \
              ["-o", out, os.path.join(ROOT, "simlod_b200", "csrc", "construct.cu")]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            print("build of", name, "failed:", r.stderr[-400:], flush=True)

n = K * BATCH
sim = SimLOD(1920, 1080, persistent_bytes=max(8 << 30, K * (96 << 20)))
sim.set_box((0, 0, 0), data.TERRAIN_EXTENT)
dptr = sim.device_alloc(n * 16)
sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
PHASES = ["fused", "split", "rewalk", "deferred", "final_alloc", "final_insert", "rounds(count)", "prologue"]
SUBS = ["f.alloc", "f.count", "f.wait", "f.flush", "f.insert", "f.barrier", "s.work", "s.barrier", "r.items", "r.flush", "r.barrier", "f.top", "r.setup", "r.listed", "r.spilled"]


def full_build(module):
    sim.use_module(0, module)
    best = None
    for rep in range(3):
        sim.reset(); sim.flush_l2()
        kms, tms = sim.insert_device(dptr, n)
        if best is None or kms < best[0]:
            ph = sim.memcpy_dtoh(sim.buffers().momentary + 96, 64).view(np.uint64).astype(np.float64)
            sub = sim.memcpy_dtoh(sim.buffers().momentary + 800, 128).view(np.uint64).astype(np.float64)
            best = (kms, tms, ph, sub)
    st = sim.stats()
    canon = oracle.canon_from_image(*sim.download_octree())
    return best, st, canon


(base_ms, _, _, _), base_stats, base_canon = full_build(None)
print("shipped kernel: %.3f ms for %d batches = %.0f Mpoints/s kernel-only, grid %d" % (base_ms, K, n / base_ms / 1e3, sim.launch_info()["construct_blocks"]), flush=True)
for v in sorted(glob.glob(os.path.join(EXP, "knob_*.cubin")) + glob.glob(os.path.join(EXP, "construct_*.cubin"))):
    label = os.path.basename(v)
    try:
        (ms, tms, ph, sub), st, canon = full_build(v)
        diffs = oracle.compare_canon(canon, base_canon, label) + oracle.compare_stats(st, base_stats)
        line = "%s grid %d: %.3f ms (%+.1f %%) = %.0f Mpts/s kernel-only, %.0f total; %s" % (
            label.ljust(28), sim.launch_info()["construct_blocks"], ms, 100.0 * (ms - base_ms) / base_ms, n / ms / 1e3, n / tms / 1e3,
            "identical octree" if not diffs else "DIFFERS: %s" % diffs[:2])
        print(line, flush=True)
        if ph.sum() > 0:
            print("      us/batch:", {k: round(float(x) / 1e3 / K, 1) for k, x in zip(PHASES, ph) if k != "rounds(count)"}, "rounds/batch %.2f" % (ph[6] / K), flush=True)
        if sub.sum() > 0:
            print("      block 0: ", {k: round(float(x) / 1e3 / K, 1) for k, x in zip(SUBS, sub)}, flush=True)
    except Exception as e:
        print(label, "failed:", e, flush=True)
sim.use_module(0, None)
sim.close()
