"""Cost of the bounding-box overlay (Uniforms::showBoundingBox) on the config-3 octree (350 x 1 M terrain batches
generated on the device, inserted with insert_device) for the six config-5 cameras of bench.py at 1920 x 1080,
minNodeSize 64: kernel_render with the overlay off and on, atomicMin and HQS, each the median / min / max of --runs
frames (CUDA events of simlod_render); the reference's kernel_render (oracle/_ref/ref_render.cubin) the same way when it
is present; per camera |D| (drawn nodes), the overlay's lines (8 + 12 |D|) and steps (from the CPU restatement of its
line list and rasteriser, tests/overlay_restatement.py), and the card and its power limit.

With --parent-cubin PATH (kernel_render built from another commit, e.g. the parent, with this build's flags), the
overlay-off frames of this build and of PATH are timed in one session, alternating, --rounds rounds of --runs frames
each, with their run-to-run spread.

    python tools/bench_overlay.py [--batches 350] [--runs 20] [--parent-cubin render.cubin] [--rounds 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def frames_ms(sim, runs):
    sim.render()                                   # warm-up (and the chunk-list cache)
    return [sim.render() for _ in range(runs)]


def drawn_lxyz(sim):
    import export_restatement as R
    import export_view_restatement as V
    st = sim.stats()
    nb = sim.memcpy_dtoh(sim.buffers().nodes, st.numNodes * 152)
    rec = np.frombuffer(np.ascontiguousarray(nb).tobytes(), dtype=R.NODE_DTYPE)
    d = V.drawn_from_flags(nb)
    return np.stack([rec[f][d].astype(np.int64) for f in ("level", "X", "Y", "Z")], axis=1)


def line_work(sim):
    """(lines, steps) of the overlay of the current frame, from the CPU restatement."""
    import overlay_restatement as O
    u = O.uniforms_from_bytes(sim.uniforms_bytes())
    s, e, c = O.line_list(u, drawn_lxyz(sim))
    pixel, _ = O.rasterize(u, s, e, c, W, H)
    return len(s), int(len(pixel))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=350)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--persistent-gb", type=int, default=16)
    ap.add_argument("--parent-cubin")
    ap.add_argument("--out")
    a = ap.parse_args()
    import oracle
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
    ref = oracle.REF_CUBINS[1] if os.path.exists(oracle.REF_CUBINS[1]) else None
    result = {"card": card(), "points": n, "nodes_in_octree": st.numNodes, "runs": a.runs, "minNodeSize": 64.0,
              "render_blocks": sim.launch_info()["render_blocks"], "cameras": []}
    cams = [("autofocus+%d" % k, camera.autofocus(data.TERRAIN_EXTENT, W, H, yaw_offset=k * np.pi / 2)) for k in range(4)]
    cams += [("morro_bird", camera.orbit_camera(width=W, height=H, **camera.MORRO_BIRD)),
             ("morro_close", camera.orbit_camera(width=W, height=H, **camera.MORRO_CLOSE))]
    sim.set_settings(minNodeSize=64.0, pointSize=1, showPoints=1)
    for name, (view, proj) in cams:
        sim.set_camera(view, proj)
        row = {"camera": name}
        for hqs in (0, 1):
            mode = "hqs" if hqs else "atomicmin"
            for overlay in (0, 1):
                sim.set_settings(useHighQualityShading=hqs, showBoundingBox=overlay)
                row["%s_overlay%s_ms" % (mode, "_on" if overlay else "_off")] = stats3(frames_ms(sim, a.runs))
            if ref:
                sim.use_module(1, ref)
                try:
                    for overlay in (0, 1):
                        sim.set_settings(useHighQualityShading=hqs, showBoundingBox=overlay)
                        row["reference_%s_overlay%s_ms" % (mode, "_on" if overlay else "_off")] = stats3(frames_ms(sim, max(3, a.runs // 4)))
                finally:
                    sim.use_module(1, None)
        sim.set_settings(useHighQualityShading=0, showBoundingBox=0)
        sim.render()
        row["drawn_nodes"] = sim.stats().numVisibleNodes
        row["lines"], row["steps_drawn"] = line_work(sim)
        row["reference_lines"] = 8 + 48 * row["drawn_nodes"]
        for mode in ("atomicmin", "hqs"):
            row["%s_overlay_cost_ms" % mode] = round(row["%s_overlay_on_ms" % mode]["median"] - row["%s_overlay_off_ms" % mode]["median"], 4)
        print(json.dumps(row), flush=True)
        result["cameras"].append(row)

    if a.parent_cubin:
        # overlay off: this build's kernel_render against the parent's, alternating rounds in one session
        sim.set_settings(showBoundingBox=0)
        cmp = {"rounds": a.rounds, "runs_per_round": a.runs, "cameras": []}
        for name, (view, proj) in cams:
            sim.set_camera(view, proj)
            entry = {"camera": name}
            for hqs in (0, 1):
                sim.set_settings(useHighQualityShading=hqs)
                this, parent = [], []
                for _ in range(a.rounds):
                    this.append(float(np.median(frames_ms(sim, a.runs))))
                    sim.use_module(1, a.parent_cubin)
                    try:
                        parent.append(float(np.median(frames_ms(sim, a.runs))))
                    finally:
                        sim.use_module(1, None)
                mode = "hqs" if hqs else "atomicmin"
                entry[mode] = {"this_ms_round_medians": stats3(this), "parent_ms_round_medians": stats3(parent),
                               "ratio_of_medians": round(float(np.median(this) / np.median(parent)), 4)}
            sim.set_settings(useHighQualityShading=0)
            print(json.dumps(entry), flush=True)
            cmp["cameras"].append(entry)
        result["overlay_off_vs_parent"] = cmp
    sim.close()
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
