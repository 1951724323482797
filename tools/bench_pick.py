"""Pick cost on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with insert_device) for
bench.py's six config-5 cameras (autofocus at 4 yaws, Morro bird and close) at 1920 x 1080. Per camera and request (the
whole frame, and one pixel at the frame's centre) the median / min / max of --runs picks with the L2 flushed before
every run, after a warm-up: kernel ms of the whole pick and of each stage (the view's plan: flags + plan + collect; the
key pass with the frame clear; the index pass; the write), beside the render kernel and the view export (median of the
same runs) for the same camera, whether repeated picks were byte-identical, and the card and its power limit.

    python tools/bench_pick.py [--batches 350] [--runs 10] [--out result.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--out")
    a = ap.parse_args()
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
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "width": W, "height": H, "runs": a.runs, "cameras": []}

    cams = [("autofocus+%d" % k, camera.autofocus(data.TERRAIN_EXTENT, W, H, yaw_offset=k * np.pi / 2)) for k in range(4)]
    cams += [("morro_bird", camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD)),
             ("morro_close", camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE))]
    dev = torch.device("cuda", 0)
    index = torch.empty(W * H, dtype=torch.int64, device=dev)
    torch.cuda.synchronize(dev)
    for name, (view, proj) in cams:
        sim.set_camera(view, proj)
        render_ms, view_ms = [], []
        sim.render()
        for _ in range(a.runs):
            sim.flush_l2()
            render_ms.append(sim.render())
            sim.flush_l2()
            view_ms.append(sim.export_view_into(0, 0, 0, 0)[1])          # the view's plan: flags + plan + collect
        row = {"camera": name, "render_ms": stats3(render_ms), "view_plan_ms": stats3(view_ms)}
        for label, pixels in (("whole_frame", None), ("one_pixel", [[W // 2, H // 2]])):
            info, _ = sim.pick_into(pixels, index.data_ptr(), 0)           # warm-up
            first = index.clone()
            total, stages, identical = [], {"plan_ms": [], "key_ms": [], "index_ms": [], "write_ms": []}, True
            for _ in range(a.runs):
                sim.flush_l2()
                info, ms = sim.pick_into(pixels, index.data_ptr(), 0)
                total.append(ms)
                for k in stages:
                    stages[k].append(getattr(info, k))
                identical &= bool(torch.equal(index, first))
            row[label] = dict({"kernel_ms": stats3(total), "hits": info.num_hits, "repeated_picks_identical": identical},
                              **{k: stats3(v) for k, v in stages.items()})
        row["view_samples"], row["view_records"] = info.num_samples, info.num_nodes
        print(json.dumps(row), flush=True)
        result["cameras"].append(row)
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
