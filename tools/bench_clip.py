"""Clip-volume cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with insert_device)
for bench.py's six config-5 cameras (autofocus at 4 yaws, Morro bird and close) at 1920 x 1080. Per clip row and draw
path (atomicMin: the default settings; HQS) the render kernel ms summed over the six cameras, median / min / max of
--runs rounds with the L2 flushed before every frame, after a warm-up. Rows: no clip; INSIDE a box around the whole cube
(the per-sample test alone: nothing is dropped); INSIDE a 1 km^2 box; the same box OUTSIDE; INSIDE a 500 m sphere; INSIDE
a 16-plane prism. With --parent-cubin, the unclipped frame of this build's kernel_render against that cubin's, loaded as
the render program, in alternating rounds. Prints the card and its power limit.
    python tools/bench_clip.py [--batches 350] [--runs 10] [--parent-cubin render.cubin] [--out result.json]
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
W, H = 1920, 1080


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def stats3(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(min(v)), 4), "max": round(float(max(v)), 4)}


def clip_rows(extent):
    from simlod_b200 import Region
    e = np.asarray(extent, np.float64)
    c = e / 2
    prism = [[np.cos(t), np.sin(t), 0.0, 500.0 - np.cos(t) * c[0] - np.sin(t) * c[1]]
             for t in np.linspace(0, 2 * np.pi, 14, endpoint=False)]               # a 14-gon of inradius 500 m
    prism += [[0.0, 0.0, 1.0, 0.0], [0.0, 0.0, -1.0, float(e[2])]]
    return [("none", None, None),
            ("cube_inside", [Region.box(-e, 2 * e)], "inside"),
            ("km2_inside", [Region.box((c[0] - 500, c[1] - 500, -e[2]), (c[0] + 500, c[1] + 500, 2 * e[2]))], "inside"),
            ("km2_outside", [Region.box((c[0] - 500, c[1] - 500, -e[2]), (c[0] + 500, c[1] + 500, 2 * e[2]))], "outside"),
            ("sphere_inside", [Region.sphere(c, 500.0)], "inside"),
            ("planes16_inside", [Region.planes(prism)], "inside")]


def frames_ms(sim, cams):
    total = 0.0
    for view, proj in cams:
        sim.set_camera(view, proj)
        sim.flush_l2()
        total += sim.render()
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--parent-cubin")
    ap.add_argument("--out")
    a = ap.parse_args()
    from simlod_b200 import SimLOD, api, camera, data

    sim = SimLOD(W, H, persistent_bytes=a.persistent_gb << 30)
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
    cams = [camera.autofocus(data.TERRAIN_EXTENT, W, H, yaw_offset=k * np.pi / 2) for k in range(4)]
    cams += [camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD), camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE)]
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "width": W, "height": H, "runs": a.runs,
              "cameras": 6, "culled_voxel_items": None, "rows": []}
    for path, settings in (("atomicMin", {"useHighQualityShading": 0}), ("hqs", {"useHighQualityShading": 1})):
        sim.set_settings(**settings)
        for name, regions, mode in clip_rows(data.TERRAIN_EXTENT):
            sim.set_clip(regions, mode or "inside")
            frames_ms(sim, cams)                                      # warm-up
            ms = [frames_ms(sim, cams) for _ in range(a.runs)]
            row = {"path": path, "clip": name, "render_ms_6_cameras": stats3(ms)}
            print(json.dumps(row), flush=True)
            result["rows"].append(row)
        sim.set_clip(None)
    sim.set_settings(useHighQualityShading=0)
    if a.parent_cubin:
        mine, parent = [], []
        for k in range(2 * a.runs + 2):
            sim.use_module(api.PROGRAM_RENDER, a.parent_cubin if k % 2 else None)
            ms = frames_ms(sim, cams)
            if k >= 2:
                (parent if k % 2 else mine).append(ms)
        sim.use_module(api.PROGRAM_RENDER, None)
        result["kernel_render_ab"] = {"this": stats3(mine), "parent": stats3(parent)}
        print(json.dumps(result["kernel_render_ab"]), flush=True)
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
