"""TEST INFRASTRUCTURE — CPU restatement of simlod_pick (DESIGN.md §9.9) over the view export's records and samples,
independent of simlod_b200, on top of overlay_restatement's float helpers.

  uniforms_from_bytes(b)                  the fields of SimlodUniforms the pick reads
  node_color_id(name)                     Node::getID() % 127 with the arithmetic kernel_render compiles
  sample_keys(records, samples, u, w, h)  per sample: pixel (x, y), depth, candidate flag and key k = depth bits << 32 | c
  pick_frame(records, samples, u, w, h)   the (h, w) int64 frame of indices, -1 where no sample wins
  brute_force(records, samples, u, w, h)  the same by a plain loop over samples and covered pixels (checks pick_frame)

The device projects with 1 / w from MUFU.RCP, the restatement with a correctly rounded division, so the two agree
exactly only where w is a power of two (an orthographic camera has w = 1); elsewhere a sample can land one pixel over."""
import numpy as np

from overlay_restatement import _d2i, _row_dot

f32, f64 = np.float32, np.float64
CLEAR = (0x7F800000 << 32) | 0x00332211          # the frame's clear value: depth +inf, colour 0x00332211
HQS_LIMIT = 0x7F800000 << 32                     # with HQS a pixel is hit when the depth bits are below +inf
SPECTRAL = (0x4F3ED5, 0x436DF4, 0x61AEFD, 0x8BE0FE, 0x98F5E6, 0xA4DDAB, 0xA5C266, 0xBD8832)
M64 = (1 << 64) - 1


def uniforms_from_bytes(b):
    """The fields of SimlodUniforms (include/simlod_abi.h) that the pick reads."""
    b = bytes(b)
    fl = np.frombuffer(b[:448], dtype="<f4")
    return {"width": float(fl[0]), "height": float(fl[1]), "transform": fl[52:68].reshape(4, 4).copy(),
            "showPoints": b[449], "colorByNode": b[450], "colorByLOD": b[451], "useHighQualityShading": b[460],
            "pointSize": int(np.frombuffer(b[468:472], dtype="<i4")[0])}


def node_color_id(name):
    """Node::getID() % 127 (render.cu): digits 1-9 shifted as 32-bit ints then sign-extended, 10-18 as 64-bit values;
    unused name bytes are 0, i.e. digit -48."""
    name = bytes(name).ljust(20, b"\0")
    ident = 1 if name[0] == ord("r") else 0
    for k in range(1, 10):
        v = ((name[k] - 48) << (3 * k)) & 0xFFFFFFFF
        if v >= 1 << 31:
            v -= 1 << 32
        ident |= v & M64
    for k, sh in zip(range(10, 19), (30, 33, 36, 39, 42, 45, 48, 51, 53)):
        ident |= ((name[k] - 48) << sh) & M64
    return ident % 127


def _per_sample(records, n):
    """Level and node colour id of every sample of the export."""
    level = np.zeros(n, dtype=np.int64)
    color_id = np.zeros(n, dtype=np.int64)
    for r in records:
        a, m = int(r["sample_offset"]), int(r["num_points"]) + int(r["num_voxels"])
        level[a:a + m] = int(r["level"])
        color_id[a:a + m] = node_color_id(r["name"])
    return level, color_id


def sample_color(u, color, level, color_id):
    """sampleColor: the sample's own colour, by node (colour id * 123456789, 32 bits) or by level (SPECTRAL)."""
    if u["colorByNode"]:
        return (color_id.astype(np.uint64) * np.uint64(123456789)) & np.uint64(0xFFFFFFFF)
    if u["colorByLOD"]:
        with np.errstate(invalid="ignore"):
            idx = np.trunc((f32(8) - level.astype(f32)) * f32(1.8)).astype(np.int64)     # cvt.rzi of a float product
        return np.asarray(SPECTRAL, dtype=np.uint64)[np.clip(idx, 0, 7)]
    return np.asarray(color, dtype=np.uint64)


def sample_keys(records, samples, u, width, height):
    """(x, y, depth, candidate, key) of every sample: kernel_render's projection, its candidate test and the 64-bit key;
    `candidate` already excludes keys that cannot win a pixel (not below the clear value, or with HQS depth bits of
    +inf and above)."""
    s = np.asarray(samples)
    n = len(s)
    px, py, pz = (s[c].astype(f32) for c in ("x", "y", "z"))
    t = np.asarray(u["transform"], f32)
    with np.errstate(all="ignore"):
        w = _row_dot(t[3], px, py, pz)
        rw = (f32(1.0) / w).astype(f32)
        ndcx = (_row_dot(t[0], px, py, pz) * rw).astype(f32)
        ndcy = (_row_dot(t[1], px, py, pz) * rw).astype(f32)
        x = _d2i((ndcx.astype(f64) * 0.5 + 0.5) * f64(u["width"]))
        y = _d2i((ndcy.astype(f64) * 0.5 + 0.5) * f64(u["height"]))
    inside = (x > 1) & (x < f64(u["width"]) - 2.0) & (y > 1) & (y < f64(u["height"]) - 2.0)
    hqs = bool(u["useHighQualityShading"])
    level, color_id = _per_sample(records, n)
    key = (w.view(np.uint32).astype(np.uint64) << np.uint64(32)) | sample_color(u, s["color"], level, color_id)
    with np.errstate(invalid="ignore"):
        cand = inside & ((w > 0) if hqs else True) & (key < np.uint64(HQS_LIMIT if hqs else CLEAR))
    return x, y, w, cand, key


def pick_frame(records, samples, u, width, height):
    """The whole-frame pick: per pixel the covering candidate with the smallest (key, index), -1 for none."""
    out = np.full(width * height, -1, dtype=np.int64)
    if not u["showPoints"] or len(samples) == 0:
        return out.reshape(height, width)
    x, y, _, cand, key = sample_keys(records, samples, u, width, height)
    idx = np.nonzero(cand)[0]
    pix, keys, ids = [], [], []
    for ox in range(max(u["pointSize"], 0)):
        for oy in range(max(u["pointSize"], 0)):
            p = np.clip(x[idx] + ox, 0, width) + width * np.clip(y[idx] + oy, 0, height)
            keep = p < width * height
            pix.append(p[keep]); keys.append(key[idx][keep]); ids.append(idx[keep])
    if pix:
        pix, keys, ids = np.concatenate(pix), np.concatenate(keys), np.concatenate(ids)
        order = np.lexsort((ids, keys, pix))
        pix, ids = pix[order], ids[order]
        first = np.ones(len(pix), dtype=bool)
        first[1:] = pix[1:] != pix[:-1]
        out[pix[first]] = ids[first]
    return out.reshape(height, width)


def brute_force(records, samples, u, width, height):
    """pick_frame by a plain loop: every sample, every covered pixel, keep the smallest (key, index)."""
    best = {}
    if u["showPoints"]:
        x, y, _, cand, key = sample_keys(records, samples, u, width, height)
        for i in range(len(samples)):
            if not cand[i]:
                continue
            for ox in range(u["pointSize"]):
                for oy in range(u["pointSize"]):
                    p = min(max(int(x[i]) + ox, 0), width) + width * min(max(int(y[i]) + oy, 0), height)
                    if p < width * height and (p not in best or (int(key[i]), i) < best[p]):
                        best[p] = (int(key[i]), i)
    out = np.full(width * height, -1, dtype=np.int64)
    for p, (_, i) in best.items():
        out[p] = i
    return out.reshape(height, width)


def frame_key(records, samples, u, index):
    """What kernel_render's framebuffer holds where the pick is `index`: the picked sample's key, the clear value at -1.
    Exact on any camera: the depth is w itself, not a product with 1 / w."""
    index = np.asarray(index)
    out = np.full(index.shape, CLEAR, dtype=np.uint64)
    hit = index >= 0
    if hit.any():
        key = sample_keys(records, samples, u, int(u["width"]), int(u["height"]))[4]
        out[hit] = key[index[hit]]
    return out
