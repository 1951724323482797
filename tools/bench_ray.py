"""Ray query cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with insert_device).
Rays: 1 k, 64 k and 1 M of each kind: camera rays through pixel centres of a 1920 x 1080 frame for two of bench.py's
config-5 cameras (autofocus and Morro close; pixels spread evenly over the frame), vertical rays from above the terrain at
uniform (x, y), and random rays through the cube (origin uniform in the cube grown by half its size on every side,
aimed at a uniform point of the cube). Depth None (the inserted points) and 5, radius --radius (5 cm). Per row, after a
warm-up, --runs runs with the L2 flushed before each: kernel ms by stage from the query's events (the export's plan +
collect; the level check + trace, which writes the destinations) as median / min / max, samples tested and records
visited per ray, rays/s over the whole kernel time, hits, and whether the repeats were byte-identical. Beside each camera
row, what a user does today for rays that happen to be pixels: render() + pick() of the same pixels (kernel ms, median
of the same number of runs, L2 flushed before each). Also the card and its power limit.

    python tools/bench_ray.py [--batches 350] [--runs 5] [--sizes 1000,65536,1048576] [--kinds camera_autofocus,...]
                              [--radius 0.05] [--out result.json]
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
SIZES = (1000, 65536, 1 << 20)
W, H = 1920, 1080
KINDS = ("camera_autofocus", "vertical", "random", "camera_morro_close")


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def stats(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(min(v)), 4), "max": round(float(max(v)), 4)}


def spread_pixels(n):
    """n pixels spread evenly over the frame, row by row."""
    ids = (np.arange(n, dtype=np.int64) * (W * H)) // n
    return np.stack([ids % W, ids // W], axis=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--sizes", default=",".join(str(v) for v in SIZES), help="ray counts, comma-separated")
    ap.add_argument("--kinds", default=",".join(KINDS))
    ap.add_argument("--radius", type=float, default=0.05)
    ap.add_argument("--out")
    a = ap.parse_args()
    sizes = [int(v) for v in a.sizes.split(",")]
    import torch
    from simlod_b200 import SimLOD, camera, data

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
    ext = np.asarray(data.TERRAIN_EXTENT, dtype=np.float64)
    size = float(ext.max())
    rng = np.random.default_rng(3)
    cams = {"camera_autofocus": camera.autofocus(data.TERRAIN_EXTENT, W, H),
            "camera_morro_close": camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE)}
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "runs": a.runs, "radius": a.radius, "rows": []}

    dev = torch.device("cuda", 0)
    m = max(sizes)
    index = torch.empty(m, dtype=torch.int64, device=dev)
    tt = torch.empty(m, dtype=torch.float32, device=dev)
    pick_index = torch.empty(m, dtype=torch.int64, device=dev)
    for nr in sizes:
        for kind in a.kinds.split(","):
            pixels = None
            if kind in cams:
                pixels = spread_pixels(nr)
                o, d = camera.pixel_rays(*cams[kind], W, H, pixels)
            elif kind == "vertical":
                o = np.zeros((nr, 3))
                o[:, :2] = rng.uniform(0, 1, (nr, 2)) * ext[:2]
                o[:, 2] = ext[2] + 100.0
                d = np.tile([[0.0, 0.0, -1.0]], (nr, 1))
            else:
                o = rng.uniform(-0.5, 1.5, (nr, 3)) * size
                d = rng.uniform(0, 1, (nr, 3)) * size - o
            r = np.zeros((nr, 8), dtype=np.float32)
            r[:, 0:3], r[:, 4:7], r[:, 7] = o, d, np.inf
            rays = torch.from_numpy(r).to(dev)
            torch.cuda.synchronize(dev)
            for depth in (None, 5):
                args = (rays.data_ptr(), nr, a.radius, depth, index.data_ptr(), tt.data_ptr(), 0, 0)
                sim.query_ray_into(*args)                                          # warm-up
                first_i, first_t = index[:nr].clone(), tt[:nr].clone()
                plan, trace, total, identical = [], [], [], True
                for _ in range(a.runs):
                    sim.flush_l2()
                    info, ms = sim.query_ray_into(*args)
                    plan.append(info.plan_ms); trace.append(info.trace_ms); total.append(ms)
                    identical &= bool(torch.equal(index[:nr], first_i) and torch.equal(tt[:nr], first_t))
                row = {"rays": nr, "kind": kind, "depth": "points" if depth is None else depth, "index_space": info.num_samples,
                       "plan_ms": stats(plan), "trace_ms": stats(trace), "total_ms": stats(total),
                       "samples_tested_per_ray": round(info.samples_tested / nr, 1),
                       "records_visited_per_ray": round(info.records_visited / nr, 2),
                       "rays_per_s": round(nr / (float(np.median(total)) / 1e3)), "hits": info.num_hits,
                       "repeats_identical": identical}
                if pixels is not None and depth is None:                          # today: render() + pick() of these pixels
                    sim.set_camera(*cams[kind])
                    sim.render()
                    sim.pick_into(pixels, pick_index.data_ptr(), 0)
                    render_ms, pick_ms = [], []
                    for _ in range(a.runs):
                        sim.flush_l2()
                        render_ms.append(sim.render())
                        sim.flush_l2()
                        pick_ms.append(sim.pick_into(pixels, pick_index.data_ptr(), 0)[1])
                    row["render_ms"], row["pick_ms"] = stats(render_ms), stats(pick_ms)
                    row["render_plus_pick_ms"] = round(float(np.median(render_ms)) + float(np.median(pick_ms)), 4)
                print(json.dumps(row), flush=True)
                result["rows"].append(row)
            del rays
    sim.close()
    print(json.dumps({"card": result["card"], "points": n, "nodes_in_octree": st.numNodes}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
