"""Render timings on a device-generated terrain octree: 6 cameras, both shading paths, ours and the reference kernel,
with our kernel's per-phase times (RCtl::phaseNanos) and cache counters. usage: render_times.py [batches=36]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from simlod_b200 import SimLOD, camera, data  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 36
VARIANTS = [a for a in sys.argv[1:] if a.endswith(".cubin")]          # extra render cubins to time beside the shipped one
n = K * 1_000_000
sim = SimLOD(1920, 1080, persistent_bytes=max(4 << 30, K * (60 << 20)))
sim.set_box((0, 0, 0), data.TERRAIN_EXTENT)
dptr = sim.device_alloc(n * 16)
sim.generate(sim.GEN_TERRAIN, dptr, n, 0, n, 7)
sim.reset()
sim.insert_device(dptr, n)
mx = data.TERRAIN_EXTENT
cams = [("autofocus+%d" % k, camera.autofocus(mx, 1920, 1080, yaw_offset=k * np.pi / 2)) for k in range(4)]
cams += [("morro_bird", camera.orbit_camera(width=1920, height=1080, **camera.MORRO_BIRD)), ("morro_close", camera.orbit_camera(width=1920, height=1080, **camera.MORRO_CLOSE))]
NAMES = ["clear|vis+cut", "-", "items", "draw", "stats+edl"]
# the shipped kernel carries no timers: a -DSIMLOD_RENDER_TIMERS=1 build of the same source gives the per-phase picture
import subprocess  # noqa: E402
timed = os.path.join(ROOT, "tools", "exp", "render_timers.cubin")
os.makedirs(os.path.dirname(timed), exist_ok=True)
r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-cubin", "-DSIMLOD_RENDER_TIMERS=1", "-o", timed,
                    os.path.join(ROOT, "simlod_b200", "csrc", "render.cu")], capture_output=True, text=True)
if r.returncode != 0:
    print("timers build failed:", r.stderr[-300:]); timed = None
for hqs in (0, 1):
    sim.set_settings(useHighQualityShading=hqs)
    tot_s = tot_ms = tot_ref = 0.0
    var_ms = {}
    for name, (view, proj) in cams:
        sim.set_camera(view, proj)
        cold = sim.render()
        ms = min(sim.render() for _ in range(5))
        s = sim.stats()
        if timed:
            sim.use_module(1, timed); sim.render(); sim.render(); sim.use_module(1, None)
        raw = sim.memcpy_dtoh(sim.buffers().renderbuffer, 96)
        c = raw[:48].view(np.uint32); ph = raw[48:88].view(np.uint64).astype(np.float64) / 1e3
        samples = s.numVisiblePoints + s.numVisibleVoxels
        ref = None
        if os.path.exists(oracle.REF_CUBINS[1]):
            sim.use_module(1, oracle.REF_CUBINS[1]); sim.render(); ref = min(sim.render() for _ in range(3)); sim.use_module(1, None)
        extra = ""
        for v in VARIANTS:
            sim.use_module(1, v); sim.render(); extra += " | %s %.4f" % (os.path.basename(v), min(sim.render() for _ in range(5))); sim.use_module(1, None)
            var_ms[v] = var_ms.get(v, 0.0) + float(extra.rsplit(" ", 1)[1])
        print("hqs %d %-12s cold %.3f warm %.4f ms (ref %s) | %d nodes %d items %.2f M samples %.1f Gs/s | cache hits/walks %d/%d | us %s" % (
            hqs, name, cold, ms, "%.4f" % ref if ref else "-", s.numVisibleNodes, int(c[0]), samples / 1e6, samples / ms / 1e6, int(c[10]), int(c[11]),
            {k: round(float(v), 1) for k, v in zip(NAMES, ph)}) + extra, flush=True)
        tot_s += samples; tot_ms += ms; tot_ref += ref or 0.0
    print("hqs %d aggregate %.1f Gsamples/s (reference kernel %.1f)" % (hqs, tot_s / tot_ms / 1e6, tot_s / tot_ref / 1e6 if tot_ref else 0.0),
          {os.path.basename(v): round(tot_s / m / 1e6, 1) for v, m in var_ms.items()}, flush=True)
sim.close()
