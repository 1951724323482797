"""CPU-only: the restatement of kernel_render's colour stages after the splat (frame_restatement: HQS resolve, eye-dome
lighting, the word past the frame) against plain per-pixel loops on small hand-made frames. The device frame is pinned to
this restatement in test_frame_gpu.py."""
import math

import numpy as np
import pytest

import frame_restatement as Fr
import pick_restatement as P
from simlod_b200 import api

F = np.float32
INF_BITS = 0x7F800000
BG = Fr.CLEAR                                   # background: depth +inf, colour 0x00332211
SIZES = [(64, 48), (80, 32)]
GRIDS = [1, 3, 7]


def word(depth, color):
    return (int(np.array(depth, F).view(np.uint32)) << 32) | int(color)


def frame(width, height):
    return np.full((height, width), BG, dtype=np.uint64)


# ---- plain statements -------------------------------------------------------------------------------------------------

def plain_covered(width, height, grid):
    tx, ty = width // 16, height // 16
    out = np.zeros((height, width), dtype=bool)
    for t in range((tx * ty) // grid * grid):
        x0, y0 = (t % tx) * 16, (t // tx) * 16
        out[y0:y0 + 16, x0:x0 + 16] = True
    return out


def plain_log2(bits):
    d = float(np.array(bits, np.uint32).view(F))
    if bits & 0x7F800000 == 0:
        return -math.inf                                  # 0 and subnormals: the input is flushed
    if d < 0 or math.isnan(d):
        return math.nan
    return math.log2(d)


def plain_edl(fb, phantom, grid):
    """Per pixel, as render.cu's EDL reads: neighbours +width, +1, -width, -1 clamped to [0, N], N being `phantom`."""
    height, width = fb.shape
    flat = [int(v) for v in fb.reshape(-1)] + [int(phantom)]
    cov = plain_covered(width, height, grid).reshape(-1)
    n = width * height
    out = np.zeros(n, dtype=np.uint32)
    for i in range(n):
        color = flat[i] & 0xFFFFFFFF
        if not cov[i]:
            out[i] = color
            continue
        lp = plain_log2(flat[i] >> 32)
        s = 0.0
        for off in (width, 1, -width, -1):
            diff = lp - plain_log2(flat[min(max(i + off, 0), n)] >> 32)
            if diff > 0:                                          # NaN (inf - inf) and -inf add nothing
                s += diff
        shade = 0.0 if s == math.inf else math.exp(-(s * float(F(0.02))) * 300.0 * float(F(0.4)))
        rgb = [int(shade * ((color >> (8 * c)) & 0xFF)) for c in range(3)]
        out[i] = rgb[0] | rgb[1] << 8 | rgb[2] << 16 | 0xFF000000
    return out.reshape(height, width)


def check_edl(fb, phantom, grid):
    want, loose = Fr.edl(fb, phantom, grid)
    plain = plain_edl(fb, phantom, grid)
    bad = Fr.mismatch(want, plain, loose)
    assert not bad.any(), "%d pixels differ from the plain loop, first at %s" % (int(bad.sum()), np.argwhere(bad)[:3].tolist())
    return want, loose


# ---- coverage ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("grid", GRIDS + [5, 13])
@pytest.mark.parametrize("size", SIZES + [(48, 32), (40, 24)])
def test_covered_is_the_first_whole_tiles(size, grid):
    w, h = size
    got = Fr.covered(w, h, grid)
    assert got.shape == (h, w) and np.array_equal(got, plain_covered(w, h, grid))


def test_the_sizes_cover_full_partial_none_and_the_last_row():
    cov = {(s, g): Fr.covered(*s, g) for s in SIZES + [(48, 32)] for g in GRIDS}
    assert cov[((64, 48), 1)].all() and cov[((64, 48), 3)].all()
    assert cov[((64, 48), 7)].any() and not cov[((64, 48), 7)][-1].any()
    assert not cov[((48, 32), 7)].any()
    assert cov[((80, 32), 3)][-1].any() and not cov[((80, 32), 3)][-1].all()
    assert cov[((80, 32), 7)][-1].any()


# ---- eye-dome lighting ------------------------------------------------------------------------------------------------

def random_frame(width, height, seed):
    """Background, drawn pixels over a range of depths, equal neighbours, depth 0 and a subnormal depth."""
    rng = np.random.default_rng(seed)
    n = width * height
    depth = np.where(rng.random(n) < 0.3, np.inf, rng.uniform(1.0, 60.0, n) * 2.0 ** rng.integers(-8, 12, n)).astype(F)
    depth[rng.integers(0, n, n // 8)] = F(37.5)                  # runs of equal depths
    depth[rng.integers(0, n, 3)] = F(0.0)
    depth[rng.integers(0, n, 2)] = np.array([1], np.uint32).view(F)[0]
    color = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    color[rng.random(n) < 0.1] &= np.uint64(0xFFFFFF00)          # some zero channels
    fb = (depth.view(np.uint32).astype(np.uint64) << np.uint64(32)) | color
    return fb.reshape(height, width)


PHANTOMS = {"clear": BG, "depth0": 0, "0xCD": 0xCDCDCDCDCDCDCDCD, "drawn": word(3.0, 0x00102030)}


@pytest.mark.parametrize("phantom", list(PHANTOMS))
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("size", SIZES)
def test_edl_equals_a_plain_loop(size, grid, phantom):
    fb = random_frame(*size, seed=size[0] + grid)
    want, loose = check_edl(fb, PHANTOMS[phantom], grid)
    cov = Fr.covered(*size, grid)
    assert (want[cov] >> np.uint32(24) == 0xFF).all()
    assert np.array_equal(want[~cov], (fb[~cov] & np.uint64(0xFFFFFFFF)).astype(np.uint32))     # alpha included
    assert loose.mean() < 0.01                                    # the +-1 band is narrow


def test_isolated_pixel_background_and_depth_zero():
    fb = frame(64, 48)
    fb[10, 10] = word(5.0, 0x00405060)
    fb[30, 40] = word(0.0, 0x00A0B0C0)                           # depth +0.0 as a winning key
    want, loose = check_edl(fb, BG, 1)
    assert want[10, 10] == 0xFF405060 and want[30, 40] == 0xFFA0B0C0
    for y, x in ((11, 10), (10, 11), (9, 10), (10, 9), (31, 40), (30, 41), (29, 40), (30, 39)):
        assert want[y, x] == 0xFF000000, (y, x)                   # a +inf term: shade 0
    assert want[20, 20] == 0xFF332211 and want[0, 0] == 0xFF332211   # background among background
    assert not loose.any()
    fb[30, 41] = word(2.0, 0x00FFFFFF)                           # next to depth 0: log2 0 = -inf, its term is +inf
    assert check_edl(fb, BG, 1)[0][30, 41] == 0xFF000000


def test_top_row_reads_pixel_zero():
    fb = frame(64, 48)
    fb[0, 5] = word(8.0, 0x00C8C8C8)
    fb[1, 5] = word(9.0, 0)
    fb[0, 4] = fb[0, 6] = word(9.0, 0)
    far, _ = check_edl(fb, BG, 1)
    assert far[0, 5] == 0xFFC8C8C8                               # pixel 0 is background: its term is -inf
    fb[0, 0] = word(4.0, 0)
    near, loose = check_edl(fb, BG, 1)
    shade = math.exp(-1.0 * float(F(0.02)) * 300 * float(F(0.4)))    # log2 8 - log2 4 = 1
    assert near[0, 5] == 0xFF000000 | int(shade * 200) * 0x010101 and not loose[0, 5].any()


def test_first_and_last_columns_wrap():
    w, h = 80, 32
    fb = frame(w, h)
    fb[4, w - 1] = word(16.0, 0x00646464)
    fb[5, 0] = word(16.0, 0x00646464)
    fb[3, w - 1] = fb[5, w - 1] = fb[4, w - 2] = fb[4, 0] = word(16.0, 0)
    fb[5, 1] = fb[6, 0] = fb[4, 0] = word(16.0, 0)
    want, _ = check_edl(fb, BG, 1)
    assert want[4, w - 1] == 0xFF646464 and want[5, 0] == 0xFF646464
    fb[5, 0] = word(8.0, 0x00646464)                              # the +1 neighbour of (w-1, 4) is (0, 5)
    want, _ = check_edl(fb, BG, 1)
    assert want[4, w - 1] == 0xFF000000 | int(math.exp(-1.0 * float(F(0.02)) * 300 * float(F(0.4))) * 100) * 0x010101
    assert want[5, 0] == 0xFF646464                               # its -1 neighbour (w-1, 4) is deeper


@pytest.mark.parametrize("grid", [1, 3, 7])
def test_the_word_below_the_last_row(grid):
    w, h = 80, 32
    fb = frame(w, h)
    fb[h - 1, 3] = word(2.0, 0x00808080)
    fb[h - 2, 3] = fb[h - 1, 2] = fb[h - 1, 4] = word(2.0, 0)
    cov = Fr.covered(w, h, grid)
    assert cov[h - 1, 3] and cov[h - 1, 20]                      # the last row is covered at these grids
    empty, _ = check_edl(fb, BG, grid)
    assert empty[h - 1, 3] == 0xFF808080 and empty[h - 1, 20] == 0xFF332211
    zero, _ = check_edl(fb, 0, grid)                              # fresh zeroed memory below: black
    assert zero[h - 1, 3] == 0xFF000000 and zero[h - 1, 20] == 0xFF000000
    cd, _ = check_edl(fb, 0xCDCDCDCDCDCDCDCD, grid)               # a negative depth: its NaN logarithm adds nothing
    assert np.array_equal(cd, empty)
    drawn, _ = check_edl(fb, PHANTOMS["drawn"], grid)             # a sample that wrapped into the word
    assert drawn[h - 1, 20] == 0xFF000000 and drawn[h - 1, 3] == 0xFF808080
    assert np.array_equal(zero[:h - 1], empty[:h - 1])            # only the last row reads it


# ---- HQS --------------------------------------------------------------------------------------------------------------

W, H = 64, 48
# w = z, ndc = (x, y) / z: samples on the axis x = y = 0 land on the centre pixel (32, 24) whatever 1 / w is
AXIS = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 1, 0]]


def uniforms(transform, width=W, height=H, **kw):
    u = api.Uniforms()
    u.width, u.height, u.showPoints, u.pointSize, u.useHighQualityShading = float(width), float(height), 1, 1, 1
    u.transform = api.mat4_to_struct(np.asarray(transform, dtype=np.float32))
    for k, v in kw.items():
        setattr(u, k, v)
    return P.uniforms_from_bytes(bytes(bytearray(u)))


def view(samples):
    pts = api.make_points(np.array([s[:3] for s in samples], dtype=F).reshape(-1, 3), [int(s[3]) for s in samples])
    rec = np.zeros(1, dtype=api.EXPORT_NODE_DTYPE)
    rec["level"], rec["name"], rec["num_points"] = 1, b"r3", len(pts)
    return rec, pts


def plain_hqs(rec, pts, u, width, height):
    """The two HQS passes and the resolve, sample by sample and pixel by pixel."""
    x, y, w, _, key = P.sample_keys(rec, pts, u, width, height)
    n = width * height
    foot = []
    for i in range(len(pts)):
        if not (x[i] > 1 and x[i] < width - 2 and y[i] > 1 and y[i] < height - 2 and w[i] > 0):
            continue
        for ox in range(u["pointSize"]):
            for oy in range(u["pointSize"]):
                p = min(max(int(x[i]) + ox, 0), width) + width * min(max(int(y[i]) + oy, 0), height)
                if p < n:
                    foot.append((p, F(w[i]), int(key[i]) & 0xFFFFFFFF))
    least = {}
    for p, d, _ in foot:
        least[p] = min(least.get(p, F(np.inf)), d)
    sums = {}
    for p, d, c in foot:
        if d < F(least[p] * F(1.01)):
            s = sums.setdefault(p, [0, 0, 0, 0])
            for k in range(3):
                s[k] += (c >> (8 * k)) & 0xFF
            s[3] += 1
    out = np.full(n, BG, dtype=np.uint64)
    for p, s in sums.items():
        c = sum(((s[k] // s[3]) & 0xFF) << (8 * k) for k in range(3)) | 0xFF000000
        out[p] = word(least[p], c)
    return out


def check_hqs(samples, u, width=W, height=H):
    rec, pts = view(samples)
    got, loose = Fr.hqs_frame(rec, pts, u, width, height)
    want = plain_hqs(rec, pts, u, width, height)
    assert np.array_equal(got, want), "%d pixels differ" % int((got != want).sum())
    return got.reshape(height, width), loose.reshape(height, width)


def test_hqs_ties_and_the_window_at_exact_depths():
    d = F(100.0)
    t = F(d * F(1.01))                                            # the window's bound: depth < t
    below, above = np.nextafter(t, F(0)), np.nextafter(t, F(np.inf))
    samples = [(0.0, 0.0, d, 0x00000010), (0.0, 0.0, d, 0x00000020),                 # a tie at the least depth
               (0.0, 0.0, below, 0x00000090),                                           # one ulp inside the window
               (0.0, 0.0, t, 0x00FFFFFF), (0.0, 0.0, above, 0x00FFFFFF)]              # on and past the bound: out
    got, loose = check_hqs(samples, uniforms(AXIS))
    assert got[24, 32] == word(d, 0xFF000000 | (0x10 + 0x20 + 0x90) // 3) and not loose.any()
    assert (got != BG).sum() == 1
    got, _ = check_hqs(samples[2:], uniforms(AXIS))                # the least depth is now `below`: t is inside
    assert got[24, 32] == word(below, 0xFFAAAA00 | (0x90 + 0xFF + 0xFF) // 3)
    # the sums divide per channel and keep the low byte
    got, _ = check_hqs([(0.0, 0.0, d, 0x00FF0001), (0.0, 0.0, d, 0x00FF0002), (0.0, 0.0, d, 0x00000002)], uniforms(AXIS))
    assert got[24, 32] == word(d, 0xFFAA0001)


@pytest.mark.parametrize("ps", [4, 5])
def test_point_size_wraps_into_the_next_row_and_past_the_frame(ps):
    ortho = [[2.0 / W, 0, 0, -1], [0, 2.0 / H, 0, -1], [0, 0, 1, 0], [0, 0, 0, 1]]        # w = 1: pixel (x, y) for x, y
    samples = [(W - 3.0 + 0.25, 10.25, 0.0, 0x00404040),       # the last inside column: x + ox reaches width
               (10.25, H - 3.0 + 0.25, 0.0, 0x00808080),       # the last inside row: y + oy reaches height
               (W - 3.0 + 0.25, H - 3.0 + 0.25, 0.0, 0x00C0C0C0)]
    u = uniforms(ortho, pointSize=ps)
    rec, pts = view(samples)
    x, y = P.sample_keys(rec, pts, u, W, H)[:2]
    assert list(x) == [W - 3, 10, W - 3] and list(y) == [10, H - 3, H - 3]
    got, loose = check_hqs(samples, u)
    assert not loose.any()
    assert got[11, 0] != BG and got[11 + ps, 0] == BG             # x + ox == width: the next row's first pixel
    assert got[H - 1, 10] != BG
    # without HQS the same footprint atomicMins the word past the frame (index width * height)
    u = uniforms(ortho, pointSize=ps, useHighQualityShading=0)
    key = P.sample_keys(rec, pts, u, W, H)[4]
    assert Fr.past_the_frame(rec, pts, u, W, H) == int(key[2])
    assert Fr.past_the_frame(rec, pts, uniforms(ortho, pointSize=3, useHighQualityShading=0), W, H) == BG
    assert Fr.past_the_frame(rec, pts, uniforms(ortho, pointSize=ps), W, H) == BG


def test_random_hqs_frames_equal_the_plain_loop():
    rng = np.random.default_rng(3)
    persp = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 2, 0]]
    n = 400
    xyz = np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-1.2, 1.2, n), rng.choice([0.5, 0.502, 0.503, 1.0, -1.0], n)], 1)
    samples = [(float(a), float(b), float(c), int(col)) for (a, b, c), col in zip(xyz, rng.integers(0, 1 << 24, n))]
    for ps in (1, 2, 3, 5):
        check_hqs(samples, uniforms(persp, pointSize=ps))


# ---- which samples are placed exactly ---------------------------------------------------------------------------------

def test_unsettled_samples():
    # w = z: 1 / 3 is not exact, and x = 0.75 at w = 3 lands on the pixel boundary (0.25 * 0.5 + 0.5) * 64 = 40
    persp = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 1, 0]]
    samples = [(0.75, 0.1, 3.0, 0), (0.7, 0.1, 3.0, 0), (1.0, 0.1, 4.0, 0), (0.0, 0.0, 3.0, 0)]
    rec, pts = view(samples)
    u = uniforms(persp, useHighQualityShading=0)
    x, y = P.sample_keys(rec, pts, u, W, H)[:2]
    assert x[0] == 40 and x[2] == 40
    assert list(Fr.unsettled_samples(pts, u)) == [True, False, False, False]    # w = 4 is a power of two: exact
    assert np.array_equal(Fr._pixel_with_rcp(pts, u, 0)[0], x)
    _, loose = check_hqs(samples, uniforms(persp))
    assert loose[24 + 0, 39:41].all() and loose.sum() == 2
