"""TEST INFRASTRUCTURE — CPU restatement of the colour stages of kernel_render that follow the splat (render.cu): the HQS
resolve and eye-dome lighting (EDL) with the RGBA8 surface, independent of simlod_b200, on pick_restatement's projection
and keys.

  covered(width, height, grid)                 pixels whose colour EDL rewrites: the first floor(tiles / grid) * grid tiles
  unsettled_samples(samples, u)                samples whose pixel could differ on the device (its 1 / w is MUFU.RCP)
  hqs_frame(records, samples, u, w, h)         the u64 frame after the HQS resolve, and the pixels an unsettled sample reaches
  past_the_frame(records, samples, u, w, h)    the word framebuffer[w * h] after the splat (the clear value unless a
                                               pointSize >= 4 sample wraps into it)
  edl(fb, phantom, grid)                       the colour words after EDL, and the channels where +-1 is allowed

The device's logarithms and exponentials are MUFU approximations, the restatement's are exact in float64; `edl` says
where that can move a channel by one (see EDL_TAU)."""
import numpy as np

import pick_restatement as P
from overlay_restatement import _d2i, _row_dot

f32, f64 = np.float32, np.float64
CLEAR = P.CLEAR
CLEAR_COLOR = CLEAR & 0xFFFFFFFF
TILE = 16


def covered(width, height, grid):
    """(height, width) mask of the pixels whose colour word the EDL pass rewrites: the first floor(tiles / grid) * grid
    16x16 tiles in row-major tile order (render.cu); partial tiles at the right and bottom edges are never covered."""
    tx, ty = width // TILE, height // TILE
    covered_tiles = (tx * ty // grid) * grid
    y, x = np.mgrid[0:height, 0:width]
    return (x // TILE < tx) & (y // TILE < ty) & ((y // TILE) * tx + x // TILE < covered_tiles)


# ---- which samples the restatement places exactly ---------------------------------------------------------------------

RCP_ULPS = 2      # rcp.approx.ftz.f32 is within 1 ulp of 1 / w by the PTX ISA; twice that is the margin taken here


def _pixel_with_rcp(samples, u, shift):
    """(x, y) of every sample with its float32 1 / w moved by `shift` ulps (render.cu project(), as sample_keys states it)."""
    s = np.asarray(samples)
    px, py, pz = (s[c].astype(f32) for c in ("x", "y", "z"))
    t = np.asarray(u["transform"], f32)
    with np.errstate(all="ignore"):
        w = _row_dot(t[3], px, py, pz)
        rw = (f32(1.0) / w).astype(f32)
        rw = (rw.view(np.int32) + np.int32(shift)).view(f32)
        ndcx = (_row_dot(t[0], px, py, pz) * rw).astype(f32)
        ndcy = (_row_dot(t[1], px, py, pz) * rw).astype(f32)
        x = _d2i((ndcx.astype(f64) * 0.5 + 0.5) * f64(u["width"]))
        y = _d2i((ndcy.astype(f64) * 0.5 + 0.5) * f64(u["height"]))
    return x, y


def unsettled_samples(samples, u, x=None, y=None):
    """Per sample: True when recomputing its pixel with 1 / w moved by +-RCP_ULPS ulps changes it (and with it the inside
    test, a function of the pixel). A power-of-two w is settled: MUFU.RCP is exact there. `x`, `y`: the samples' pixels
    as sample_keys gives them (computed here when None)."""
    if x is None:
        x, y = _pixel_with_rcp(samples, u, 0)
    w = _row_dot(np.asarray(u["transform"], f32)[3], *(np.asarray(samples)[c].astype(f32) for c in ("x", "y", "z")))
    out = np.zeros(len(x), dtype=bool)
    for shift in (-RCP_ULPS, RCP_ULPS):
        xs, ys = _pixel_with_rcp(samples, u, shift)
        out |= (xs != x) | (ys != y)
    mant = w.view(np.uint32) & np.uint32(0x007FFFFF)
    exp = (w.view(np.uint32) >> np.uint32(23)) & np.uint32(0xFF)
    pow2 = (mant == 0) & (exp != 0) & (exp != 0xFF)
    return out & ~pow2


def _footprint(x, y, ps, width, height):
    """Pixel indices of the pointSize^2 footprint of each (x, y), (ps*ps, n): the clamp to width / height is inclusive
    (render.cu), so x + ox >= width lands on the next row's first pixel and y + oy >= height at index >= width * height."""
    out = []
    for ox in range(ps):
        for oy in range(ps):
            out.append(np.clip(x + ox, 0, width) + width * np.clip(y + oy, 0, height))
    return np.array(out, dtype=np.int64).reshape(ps * ps, len(x))


# ---- HQS ----------------------------------------------------------------------------------------------------------------

def hqs_frame(records, samples, u, width, height):
    """The u64 framebuffer after the HQS passes and resolve (render.cu), and the (N,) mask of pixels an unsettled sample
    could reach (its colour and depth there are not restated exactly).

    Candidates are samples inside the frame with w > 0. Pass 1 keeps each pixel's least depth; pass 2 sums the channels
    of the samples with depth < float32(least * 1.01f) (one rounded float32 multiply); the resolve writes
    depth << 32 | 0xff000000 | (sum / n & 0xff) per channel, and a pixel no sample reaches keeps the clear value.
    Footprint pixels at index >= width * height change no pixel of the frame: there the depth target overlaps the
    colour sums (or the pad before them), and the resolve only covers the frame."""
    n = width * height
    fb = np.full(n, CLEAR, dtype=np.uint64)
    loose = np.zeros(n, dtype=bool)
    if not u["showPoints"] or len(samples) == 0:
        return fb, loose
    x, y, w, _, key = P.sample_keys(records, samples, u, width, height)
    inside = (x > 1) & (x < f64(u["width"]) - 2.0) & (y > 1) & (y < f64(u["height"]) - 2.0)
    with np.errstate(invalid="ignore"):
        positive = w > 0
    ps = max(int(u["pointSize"]), 0)
    # the pixels an unsettled sample could reach: its footprint from the pixel of 1 / w moved either way
    shaky = unsettled_samples(samples, u, x, y) & positive
    if shaky.any():
        idx = np.nonzero(shaky)[0]
        for shift in (-RCP_ULPS, 0, RCP_ULPS):
            xs, ys = _pixel_with_rcp(np.asarray(samples)[idx], u, shift)
            ok = (xs > 1) & (xs < width - 2) & (ys > 1) & (ys < height - 2)
            p = _footprint(xs[ok], ys[ok], ps, width, height).reshape(-1)
            loose[p[p < n]] = True
    cand = np.nonzero(inside & positive)[0]
    if len(cand) == 0 or ps == 0:
        return fb, loose
    pix = _footprint(x[cand], y[cand], ps, width, height).reshape(-1)
    depth = np.tile(w[cand], ps * ps)
    color = np.tile(key[cand] & np.uint64(0xFFFFFFFF), ps * ps)
    keep = pix < n
    pix, depth, color = pix[keep], depth[keep], color[keep]
    order = np.argsort((pix.astype(np.uint64) << np.uint64(32)) | depth.view(np.uint32).astype(np.uint64))   # positive depths order as their bits
    pix, depth, color = pix[order], depth[order], color[order]
    start = np.ones(len(pix), dtype=bool)
    start[1:] = pix[1:] != pix[:-1]
    first = np.nonzero(start)[0]
    least = depth[first]                                            # sorted by depth within a pixel
    window = (least * f32(1.01)).astype(f32)
    group = np.cumsum(start) - 1
    within = depth < window[group]
    sums = np.zeros((len(first), 4), dtype=np.int64)
    for c in range(3):
        sums[:, c] = np.bincount(group[within], weights=((color[within] >> np.uint64(8 * c)) & np.uint64(0xFF)).astype(f64),
                                 minlength=len(first)).astype(np.int64)
    sums[:, 3] = np.bincount(group[within], minlength=len(first))
    word = np.full(len(first), 0xFF000000, dtype=np.uint64)
    for c in range(3):
        word |= ((sums[:, c] // sums[:, 3]) & 0xFF).astype(np.uint64) << np.uint64(8 * c)
    fb[pix[first]] = (least.view(np.uint32).astype(np.uint64) << np.uint64(32)) | word
    return fb, loose


def past_the_frame(records, samples, u, width, height):
    """framebuffer[width * height] after the frame's splat: kernel_render clears it with the clear value, and without HQS a
    sample whose pointSize >= 4 footprint wraps from the last row's right edge into it atomicMins it there."""
    if not u["showPoints"] or u["useHighQualityShading"] or len(samples) == 0:
        return CLEAR
    x, y, _, cand, key = P.sample_keys(records, samples, u, width, height)
    idx = np.nonzero(cand)[0]
    pix = _footprint(x[idx], y[idx], max(int(u["pointSize"]), 0), width, height)
    hit = (pix == width * height).any(axis=0)
    return int(min(CLEAR, int(key[idx][hit].min()))) if hit.any() else CLEAR


# ---- eye-dome lighting --------------------------------------------------------------------------------------------------

# Constants as kernel_render's EDL uses them: sum / 50 as sum * 0.02f, then (double) * 300.0 * (double)0.4f, then
# ex2(e * -1.4426950216293334961f) for __expf(-e).
K_RESPONSE = f64(f32(0.02))
K_STRENGTH = f64(f32(0.4))
K_LOG2E = f64(f32(-1.4426950216293334961))
# shade = 2^(K * sum) with K = 0.02 * 300 * 0.4 * -log2(e), so d(shade) / d(sum) = -2.4 shade (to float32 rounding)
K_SUM = K_RESPONSE * 300.0 * K_STRENGTH * K_LOG2E
NEIGHBOURS = 4

# EDL_TAU: how far the device's shade * c can lie from the restatement's. ASSUMED from the error bounds the PTX ISA states
# for the approximations kernel_render uses, not measured:
#   lg2.approx.ftz.f32  absolute error <= 2^-22.6 on the logarithm of the mantissa; the float32 result then rounds, which
#                       adds <= 2^-24 |log2 d|. Per logarithm: e_L(d) <= 2^-22 + 2^-24 |log2 d|.
#   ex2.approx.ftz.f32  relative error <= 2 ulp, <= 2^-22.
# One neighbour term max(lg2(d) - lg2(n), 0) is 1-Lipschitz in the difference, so it is off by at most
# e_L(d) + e_L(n) + 2^-24 |lg2(d) - lg2(n)| (the float32 subtraction); terms with an infinite or NaN logarithm
# (depth 0, subnormal, +inf or negative) are the same on both sides. The float32 sum rounds after each of the 4 adds:
# 4 * 2^-24 * sum. With E_S the sum of these, the exponent x = K * sum (K = -3.4625) is off by |K| E_S plus three float32
# roundings (response, e, the product), 3 * 2^-24 |x|; shade = 2^x is then off relatively by ln 2 times that, plus 2^-22
# for ex2 itself, and shade * c by another 2^-24 for the float32 product. We allow twice the first-order sum of these
# (for the second-order terms and the float64 evaluation here), per pixel and channel: v = shade * c may come out one
# lower or higher on the device only where v lies within tau = 2 * v * (...) of an integer.
# Exact by construction: sum == 0 (every neighbour as deep or deeper, or empty: shade is 1 on both sides; this
# takes MUFU.LG2 to be monotone, so that d <= n gives lg2(d) <= lg2(n)), sum == +inf (shade 0) and c == 0.
EDL_TAU_FACTOR = 2.0


def _log2_ftz(d):
    """log2 of float32 depths in float64, with lg2.approx.ftz's input flush: subnormals are 0 (-> -inf)."""
    d = np.asarray(d, f32)
    sub = (d.view(np.uint32) & np.uint32(0x7F800000)) == 0
    with np.errstate(all="ignore"):
        return np.where(sub, -np.inf, np.log2(np.abs(d).astype(f64)) * np.where(d < 0, np.nan, 1.0))


def edl(fb, phantom, grid):
    """Eye-dome lighting of a (height, width) u64 frame (depth bits << 32 | colour) whose framebuffer[width * height] is
    `phantom`, with a render grid of `grid` blocks (render.cu). Returns (colour words (height, width) uint32, loose
    (height, width, 3) bool: the R, G, B channels where the device may differ by one).

    On covered pixels: sum over the neighbours at +width, +1, -width, -1 (index clamped to [0, width * height]: the top
    row reads pixel 0, the first and last columns wrap into the neighbouring row, the last row reads `phantom`) of
    max(log2 d - log2 n, 0), where inf - inf and NaN contribute 0 and a +inf term makes the shade 0; shade =
    2^(K * sum); each channel trunc(shade * c), alpha 0xff. Uncovered pixels keep their colour word."""
    fb = np.asarray(fb, dtype=np.uint64)
    height, width = fb.shape
    n = width * height
    words = np.concatenate([fb.reshape(-1), np.array([phantom], dtype=np.uint64)])
    depth = (words >> np.uint64(32)).astype(np.uint32).view(f32)
    color = (fb.reshape(-1) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    lg = _log2_ftz(depth)
    i = np.arange(n, dtype=np.int64)
    lp = lg[:n]
    total = np.zeros(n, dtype=f64)
    err = np.zeros(n, dtype=f64)
    with np.errstate(all="ignore"):
        for off in (width, 1, -width, -1):
            ln = lg[np.clip(i + off, 0, n)]
            diff = lp - ln
            total = total + np.fmax(diff, 0.0)                      # fmax: a NaN difference adds 0
            finite = np.isfinite(lp) & np.isfinite(ln)
            e_l = 2.0 ** -22 * 2 + 2.0 ** -24 * (np.abs(lp) + np.abs(ln) + np.abs(diff))
            err = err + np.where(finite, e_l, 0.0)
        err = err + NEIGHBOURS * 2.0 ** -24 * np.where(np.isfinite(total), total, 0.0)
        x = total * K_SUM
        shade = np.exp2(x)
        rel = np.log(2.0) * (-K_SUM * err + 3 * 2.0 ** -24 * np.abs(x)) + 2.0 ** -22 + 2.0 ** -24
    out = np.zeros(n, dtype=np.uint32)
    loose = np.zeros((n, 3), dtype=bool)
    soft = np.isfinite(total) & (total > 0)
    for c in range(3):
        ch = ((color >> np.uint32(8 * c)) & np.uint32(0xFF)).astype(f64)
        with np.errstate(all="ignore"):
            v = shade * ch
            got = np.floor(v)
            tau = EDL_TAU_FACTOR * v * rel                          # NaN where sum is +inf: not loose
            near = np.minimum(v - got, got + 1.0 - v) <= tau
        loose[:, c] = soft & (ch > 0) & near
        out |= got.astype(np.uint32) << np.uint32(8 * c)
    out |= np.uint32(0xFF000000)
    cov = covered(width, height, grid).reshape(-1)
    out = np.where(cov, out, color)
    loose &= cov[:, None]
    return out.reshape(height, width), loose.reshape(height, width, 3)


def mismatch(got, want, loose):
    """(height, width) mask of pixels where the colour words `got` differ from `want` by more than `loose` allows: any
    alpha difference, a channel off by more than one, or off by one where it is not loose."""
    got = np.asarray(got, dtype=np.uint32)
    want = np.asarray(want, dtype=np.uint32)
    bad = (got >> np.uint32(24)) != (want >> np.uint32(24))
    for c in range(3):
        g = ((got >> np.uint32(8 * c)) & np.uint32(0xFF)).astype(np.int64)
        w = ((want >> np.uint32(8 * c)) & np.uint32(0xFF)).astype(np.int64)
        d = np.abs(g - w)
        bad |= (d > 1) | ((d == 1) & ~loose[..., c])
    return bad
