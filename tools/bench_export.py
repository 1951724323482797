"""Octree export throughput on the config-3 octree (350 x 1 M terrain batches generated on the device, inserted with
insert_device): the full export and the cuts at depths 3, 5 and 7, each the median of --runs runs with the L2 flushed
before every run, after a warm-up. Reports kernel time (plan + collect + gather events), Gsamples/s and achieved
bandwidth in algorithmic bytes (16 B read + 16 B written per sample, 152 B read + 64 B written per node) against the
H100 SXM data sheet's 3.35 TB/s, the host path (download_octree + canon_from_image) once, the card and its power
limit, and whether the repeated exports were byte-identical.

With --view, instead the view export (simlod_export_view) for the six config-5 cameras of bench.py at 1920 x 1080:
per camera the records, drawn nodes and samples; kernel ms of the drawn-flags kernel alone, of plan + collect (the size
query, flags included) and of the whole export, each as median / min / max; Gsamples/s and algorithmic bytes (16 B read
+ 16 B written per sample, 152 B read per node of nodes[], 64 B written per record); the render kernel's time for the
same camera; and whether repeated exports were byte-identical.

    python tools/bench_export.py [--batches 350] [--runs 10] [--view] [--out result.json]
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

PEAK_GBS = 3350.0
BATCH = 1_000_000
TERRAIN_SEED = 7


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    name, _, limit = out.partition(",")
    return {"name": name.strip(), "power_limit": limit.strip()}


def stats3(v):
    return {"median": round(float(np.median(v)), 4), "min": round(float(min(v)), 4), "max": round(float(max(v)), 4)}


def bench_views(sim, runs, num_nodes):
    """The view export for bench.py's config-5 cameras (autofocus at 4 yaws, Morro bird and close) at 1920 x 1080."""
    import torch
    from simlod_b200 import camera, data
    W, H = 1920, 1080
    cams = [("autofocus+%d" % k, camera.autofocus(data.TERRAIN_EXTENT, W, H, yaw_offset=k * np.pi / 2)) for k in range(4)]
    cams += [("morro_bird", camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD)),
             ("morro_close", camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE))]
    dev = torch.device("cuda", 0)
    out = []
    for name, (view, proj) in cams:
        sim.set_camera(view, proj)
        render_ms = []
        for _ in range(3):
            render_ms.append(sim.render())
        info, _ = sim.export_view_into(0, 0, 0, 0)
        nodes_buf = torch.empty(max(info.num_nodes, 1) * 64, dtype=torch.uint8, device=dev)
        samples_buf = torch.empty(max(info.num_samples, 1) * 16, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)
        args = (nodes_buf.data_ptr(), info.num_nodes, samples_buf.data_ptr() if info.num_samples else 0, info.num_samples)
        sim.export_view_into(*args)                                   # warm-up
        first_nodes, first_samples = nodes_buf.clone(), samples_buf.clone()
        query_ms, kernel_ms, identical = [], [], True
        for _ in range(runs):
            sim.flush_l2()
            query_ms.append(sim.export_view_into(0, 0, 0, 0)[1])      # flags + plan + collect
            sim.flush_l2()
            kernel_ms.append(sim.export_view_into(*args)[1])
            identical &= bool(torch.equal(nodes_buf, first_nodes)) and bool(torch.equal(samples_buf, first_samples))
        # the flags kernel alone: its device time in a profile of `runs` more size queries
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(runs):
                sim.flush_l2()
                sim.export_view_into(0, 0, 0, 0)
        flags_ms = [e.time_range.elapsed_us() / 1e3 for e in prof.events() if e.name == "simlod_export_view_flags"]
        drawn = int(((first_nodes.cpu().numpy()[:info.num_nodes * 64].view(api_dtype()))["flags"] & 2 != 0).sum())
        ms = float(np.median(kernel_ms))
        nbytes = 32 * info.num_samples + 152 * num_nodes + 64 * info.num_nodes
        row = {"camera": name, "records": info.num_nodes, "drawn": drawn, "samples": info.num_samples,
               "points": info.num_points, "voxels": info.num_voxels,
               "flags_ms": stats3(flags_ms) if flags_ms else "not measured", "plan_collect_ms": stats3(query_ms), "kernel_ms": stats3(kernel_ms),
               "gsamples_per_s": round(info.num_samples / ms / 1e6, 3), "algorithmic_bytes": nbytes,
               "achieved_gb_per_s": round(nbytes / ms / 1e6, 1), "share_of_3350_gb_per_s": round(nbytes / ms / 1e6 / PEAK_GBS, 4),
               "render_ms_best_of_3": round(min(render_ms), 4), "repeated_exports_identical": identical}
        print(json.dumps(row), flush=True)
        out.append(row)
        del nodes_buf, samples_buf, first_nodes, first_samples
        torch.cuda.empty_cache()
    return out


def api_dtype():
    from simlod_b200 import api
    return api.EXPORT_NODE_DTYPE


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--view", action="store_true", help="the view export for the six config-5 cameras instead")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    import oracle
    from simlod_b200 import SimLOD, data

    sim = SimLOD(1920, 1080, persistent_bytes=a.persistent_gb << 30) if a.view else SimLOD(640, 360, persistent_bytes=a.persistent_gb << 30)
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
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "heap_bytes": int(st.allocatedBytes_persistent),
              "runs": a.runs, "exports": []}
    if a.view:
        result["views"] = bench_views(sim, a.runs, st.numNodes)
        sim.close()
        print(json.dumps(result))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(result, f, indent=1)
        return

    full, _ = sim.export_octree_into(None, 0, 0, 0, 0)
    dev = torch.device("cuda", 0)
    nodes_buf = torch.empty(full.num_nodes * 64, dtype=torch.uint8, device=dev)
    samples_buf = torch.empty(full.num_samples * 16, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    for depth in (None, 3, 5, 7):
        info, plan_ms = sim.export_octree_into(depth, 0, 0, 0, 0)     # size query: plan + collect only
        args = (depth, nodes_buf.data_ptr(), info.num_nodes, samples_buf.data_ptr() if info.num_samples else 0, info.num_samples)
        sim.export_octree_into(*args)                                  # warm-up
        torch.cuda.synchronize(dev)
        first_nodes = nodes_buf[:info.num_nodes * 64].clone()
        first_samples = samples_buf[:info.num_samples * 16].clone()
        kernel_ms, wall_ms, identical = [], [], True
        for _ in range(a.runs):
            sim.flush_l2()
            t0 = time.perf_counter()
            _, ms = sim.export_octree_into(*args)
            wall_ms.append((time.perf_counter() - t0) * 1e3)
            kernel_ms.append(ms)
            identical &= bool(torch.equal(nodes_buf[:info.num_nodes * 64], first_nodes)) and \
                bool(torch.equal(samples_buf[:info.num_samples * 16], first_samples))
        del first_nodes, first_samples
        torch.cuda.empty_cache()
        ms = float(np.median(kernel_ms))
        nbytes = 32 * info.num_samples + (152 + 64) * info.num_nodes
        result["exports"].append({
            "depth": "full" if depth is None else depth, "nodes": info.num_nodes, "samples": info.num_samples,
            "points": info.num_points, "voxels": info.num_voxels,
            "kernel_ms_median": round(ms, 4), "kernel_ms_min": round(min(kernel_ms), 4), "kernel_ms_max": round(max(kernel_ms), 4),
            "plan_collect_ms": round(plan_ms, 4), "wall_ms_median": round(float(np.median(wall_ms)), 4),
            "gsamples_per_s": round(info.num_samples / ms / 1e6, 3), "algorithmic_bytes": nbytes,
            "achieved_gb_per_s": round(nbytes / ms / 1e6, 1), "share_of_3350_gb_per_s": round(nbytes / ms / 1e6 / PEAK_GBS, 4),
            "repeated_exports_identical": identical})
        print(json.dumps(result["exports"][-1]), flush=True)
    del nodes_buf, samples_buf
    torch.cuda.empty_cache()

    t0 = time.perf_counter()
    image = sim.download_octree()
    t1 = time.perf_counter()
    canon = oracle.canon_from_image(*image)
    t2 = time.perf_counter()
    result["host_path"] = {"download_octree_s": round(t1 - t0, 3), "canon_from_image_s": round(t2 - t1, 3),
                           "image_bytes": int(len(image[0]) + len(image[1])), "nodes": len(canon.records)}
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
