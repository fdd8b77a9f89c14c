"""The colour preparation's RGB instantiations on the GPU, pixel by pixel: plstvo_debug_color_planes returns both planes the
FLD branch's colour sessions compute in one launch (color_convert_kernel<C, true> without maps, color_remap_kernel<C, false,
true> with shared maps, color_remap_kernel<C, true, true> with a per-pair table), and this file holds the COLOR_RGB2GRAY
plane to oracle/fld.py and the COLOR_BGR2GRAY plane to oracle/color.py / tests/golden/color.npz and, byte for byte, to
plstvo_rectify_batch (the RGB = false instantiations) on the same images.  Bit-exact everywhere: the arithmetic is integer.

Where these kernels could go wrong alone: the last partial 16-pixel group of a batch (the bottom-right pixels of its last
right image), the last partial quad of each image when W * H % 4 != 0, the byte-wise stores where an image starts off a
4-byte boundary, the table's entries without maps, and the grid slices past 65535 images.  Needs neither cv2 nor the
reference sources."""
import ctypes as C

import numpy as np
import pytest

from oracle import color as OC
from oracle import fld as OF
from test_color_host import G, all_triples, assert_golden, case_image, case_maps
from test_gpu_track_images import sm_count
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine

pytestmark = pytest.mark.gpu


def random_maps(rng, W, H):
    """CV_16SC2 + CV_16UC1 maps whose taps reach two pixels beyond every edge (x in [-2, W + 1], y in [-2, H + 1]) and whose
    map2 words use all 16 bits (the kernels and OpenCV read the low 10)"""
    m1 = np.stack([rng.integers(-2, W + 2, (H, W)), rng.integers(-2, H + 2, (H, W))], -1).astype(np.int16)
    m2 = rng.integers(0, 1 << 16, (H, W)).astype(np.uint16)
    return m1, m2


def stacked_oracle(imgs, maps):
    """(BGR2GRAY, RGB2GRAY) of cvtColor(remap(img)) for each of the images [n, H, W, C], maps[k] = image k's (map1, map2) or
    None (cvtColor alone), through oracle/color.py and oracle/fld.py on one image: the images one above the other with 3 zero
    rows before each and after the last, each one's maps moved down to its rows.  The maps reach at most 2 rows beyond an
    image (random_maps), so every tap outside an image reads a zero row, BORDER_CONSTANT's 0, and never another image."""
    n, H, W, Ch = imgs.shape
    P = 3
    band = H + P
    tall = np.zeros((n * band + P, W, Ch), np.uint8)
    m1 = np.zeros((n * band + P, W, 2), np.int64)
    m2 = np.zeros((n * band + P, W), np.uint16)
    grey = OC.bgr_to_gray(imgs)
    rgb = OF.rgb_to_gray(imgs)
    mapped = [k for k in range(n) if maps[k] is not None]
    if not mapped:
        return grey, rgb
    for k in mapped:
        r0 = k * band + P
        tall[r0:r0 + H] = imgs[k]
        m1[r0:r0 + H] = maps[k][0]
        m1[r0:r0 + H, :, 1] += r0
        m2[r0:r0 + H] = maps[k][1]
    g_tall, r_tall = OC.remap_gray(tall, m1, m2), OF.remap_gray_rgb(tall, m1, m2)
    for k in mapped:
        r0 = k * band + P
        grey[k], rgb[k] = g_tall[r0:r0 + H], r_tall[r0:r0 + H]
    return grey, rgb


def assert_planes(got, want, what):
    """got / want: (grey, rgb), each [2, B, H, W]; the first differing pixel named"""
    for name, g, w in (("BGR2GRAY", got[0], want[0]), ("RGB2GRAY", got[1], want[1])):
        bad = np.argwhere(g != w)
        assert len(bad) == 0, (f"{what}: {name} plane differs at {len(bad)} pixels, first [side, pair, y, x] = {bad[0].tolist()}: "
                               f"{int(g[tuple(bad[0])])} != {int(w[tuple(bad[0])])}")


def rectify_batch_planes(e, rect, il, ir):
    """plstvo_rectify_batch's grey images as [2, B, H, W]"""
    ol, orr = e.rectify_batch(rect, il, ir)
    return np.stack([ol, orr])


# ---- 1. every BGR triple, with no maps and through a table of map-less entries ----
@pytest.mark.parametrize("form", ["convert", "table"])
@pytest.mark.parametrize("channels", [3, 4])
def test_every_triple(engine, channels, form):
    """All 2^24 triples as one 4096 x 4096 image on the left, its rows reversed on the right, so a side swap shows"""
    img = all_triples(channels, seed=41 + channels)
    il, ir = img[None], img[::-1][None].copy()
    rect = engine.rectifier_create_color(4096, 4096, channels)
    grey, rgb = engine.debug_color_planes(rect, il, ir, [rect] if form == "table" else None)
    want_g, want_r = OC.bgr_to_gray(img), OF.rgb_to_gray(img)
    assert_planes((grey, rgb), (np.stack([want_g, want_g[::-1]])[:, None], np.stack([want_r, want_r[::-1]])[:, None]), form)
    np.testing.assert_array_equal(grey, rectify_batch_planes(engine, rect, il, ir))
    assert engine.rectify_kernel_times() > 0
    engine.rectifier_destroy(rect)


# ---- 2. every golden case, batched, with the rectifier's maps and through a table holding them ----
@pytest.mark.parametrize("size", ["1", "37", "sms+5"])
def test_every_golden_case(engine, size):
    B = {"1": 1, "37": 37}.get(size, sm_count() + 5)
    for c in G["cases"]:
        w, h = (int(v) for v in G[f"{c}_size"])
        channels = int(G[f"{c}_channels"])
        m1, m2 = case_maps(c)
        rect = engine.rectifier_create_color(w, h, channels, *(() if m1 is None else (m1, m2)))
        if B == 1:
            il, ir = case_image(c)[None], case_image(c)[None]
        else:   # the golden image first on the left and last on the right, seeded noise images between
            rng = np.random.default_rng(B + 3 * len(c))
            il = rng.integers(0, 256, (B, h, w, channels), dtype=np.uint8)
            ir = rng.integers(0, 256, (B, h, w, channels), dtype=np.uint8)
            il[0] = ir[-1] = case_image(c)
        grey, rgb = engine.debug_color_planes(rect, il, ir)
        assert_golden(c, grey[0, 0])
        assert_golden(c, grey[1, -1])
        np.testing.assert_array_equal(grey, rectify_batch_planes(engine, rect, il, ir), err_msg=c)
        # the RGB plane on the golden images, the middle pair, and pairs 0 .. 3, whose images start at every offset mod 4
        # where W * H is odd (test 3 holds every image of many more sizes, on maps of its own)
        for b in sorted({0, 1, 2, 3, B // 2, B - 1} & set(range(B))):
            for side, img in ((0, il[b]), (1, ir[b])):
                np.testing.assert_array_equal(rgb[side, b], OF.remap_gray_rgb(img, m1, m2), err_msg=f"{c} side {side} pair {b}")
        # the same rectifier in every entry of a table: color_remap_kernel<C, true, true>, its !m1 branch for the plain cases
        tab = engine.debug_color_planes(rect, il, ir, [rect] * B)
        np.testing.assert_array_equal(tab[0], grey, err_msg=c)
        np.testing.assert_array_equal(tab[1], rgb, err_msg=c)
        engine.rectifier_destroy(rect)


def test_both_sides_own_maps(engine):
    """The EuRoC rig's two sides in one rectifier, 3 and 4 channels: each side's golden through its own maps, and a table of
    that rectifier"""
    for channels in (3, 4):
        cl, cr = f"c{channels}_euroc_l", f"c{channels}_euroc_r"
        (m1l, m2l), (m1r, m2r) = case_maps(cl), case_maps(cr)
        rect = engine.rectifier_create_color(752, 480, channels, m1l, m2l, m1r, m2r)
        il, ir = case_image(cl)[None], case_image(cr)[None]
        want = (np.stack([OC.remap_gray(il[0], m1l, m2l), OC.remap_gray(ir[0], m1r, m2r)])[:, None],
                np.stack([OF.remap_gray_rgb(il[0], m1l, m2l), OF.remap_gray_rgb(ir[0], m1r, m2r)])[:, None])
        for rects in (None, [rect]):
            grey, rgb = engine.debug_color_planes(rect, il, ir, rects)
            assert_golden(cl, grey[0, 0])
            assert_golden(cr, grey[1, 0])
            assert_planes((grey, rgb), want, f"{channels} channels, table {rects is not None}")
        engine.rectifier_destroy(rect)


# ---- 3. tails and alignment: every W * H % 4, image starts at every offset mod 16, batch totals at every even one ----
# W * H % 4: 1 (1x1, 5x1, 3x3, 45x1), 2 (2x1, 6x3, 7x2), 3 (3x1, 7x1, 7x5, 13x11), 0 (4x1, 8x2)
TAIL_SIZES = [(1, 1), (2, 1), (3, 1), (4, 1), (5, 1), (7, 1), (3, 3), (7, 2), (6, 3), (8, 2), (7, 5), (13, 11), (45, 1)]
# n = 2 B W H pixels in all, so n % 16 is even; B = 1 .. 8 gives every even remainder for odd W * H, and with odd W * H the
# images of B >= 8 pairs start at every offset mod 16
TAIL_B = [1, 2, 3, 4, 5, 6, 7, 8, 9, 37]


@pytest.mark.parametrize("form", ["convert", "maps", "table"])
@pytest.mark.parametrize("channels", [3, 4])
def test_tails_and_alignment(engine, channels, form):
    rng = np.random.default_rng(700 + 10 * channels + len(form))
    remainders = set()
    for W, H in TAIL_SIZES:
        maps_a = random_maps(rng, W, H) + random_maps(rng, W, H)   # left, right
        maps_b = random_maps(rng, W, H) + random_maps(rng, W, H)
        plain = engine.rectifier_create_color(W, H, channels)
        with_a = engine.rectifier_create_color(W, H, channels, *maps_a)
        with_b = engine.rectifier_create_color(W, H, channels, *maps_b)
        maps_of = {id(plain): None, id(with_a): maps_a, id(with_b): maps_b}
        for B in TAIL_B:
            remainders.add(2 * B * W * H % 16)
            il = rng.integers(0, 256, (B, H, W, channels), dtype=np.uint8)
            ir = rng.integers(0, 256, (B, H, W, channels), dtype=np.uint8)
            if form == "table":   # entries with maps, NULL entries and map-less ones, in an order that moves with B
                cycle = [with_a, None, plain, with_b, with_b, None, with_a, plain]
                rects = [cycle[(b + B) % len(cycle)] for b in range(B)]
                rect = plain
            else:
                rects = None
                rect = plain if form == "convert" else with_a
            got = engine.debug_color_planes(rect, il, ir, rects)
            # the rectifier that prepares each pair: a NULL entry converts only, as the map-less one does
            used = [plain if r is None else r for r in (rects or [rect] * B)]
            per = [maps_of[id(r)] for r in used]
            gl, rl = stacked_oracle(il, [None if m is None else m[:2] for m in per])
            gr, rr = stacked_oracle(ir, [None if m is None else m[2:] for m in per])
            assert_planes(got, (np.stack([gl, gr]), np.stack([rl, rr])), f"{form} {W}x{H}x{channels} B={B}")
            # the grey plane against plstvo_rectify_batch, each rectifier's pairs through it
            for r in (plain, with_a, with_b):
                idx = [b for b, u in enumerate(used) if u is r]
                if idx:
                    np.testing.assert_array_equal(got[0][:, idx], rectify_batch_planes(engine, r, il[idx], ir[idx]),
                                                  err_msg=f"{form} {W}x{H}x{channels} B={B}")
        for r in (plain, with_a, with_b):
            engine.rectifier_destroy(r)
    assert remainders == set(range(0, 16, 2)), remainders


# ---- 4. more than 65535 images: the launches' grid slices ----
@pytest.mark.parametrize("form", ["maps", "table"])
@pytest.mark.parametrize("W", [1, 3])
def test_more_than_65535_images(engine, W, form):
    B, H, channels = 33000, 1, 3   # 66000 images: two grid slices of the remap launch
    rng = np.random.default_rng(90 + W + len(form))
    maps_a = random_maps(rng, W, H) + random_maps(rng, W, H)
    maps_b = random_maps(rng, W, H) + random_maps(rng, W, H)
    plain = engine.rectifier_create_color(W, H, channels)
    with_a = engine.rectifier_create_color(W, H, channels, *maps_a)
    with_b = engine.rectifier_create_color(W, H, channels, *maps_b)
    il = rng.integers(0, 256, (B, H, W, channels), dtype=np.uint8)
    ir = rng.integers(0, 256, (B, H, W, channels), dtype=np.uint8)
    if form == "table":
        cycle = [with_a, plain, None, with_b, with_a]
        rects = [cycle[b % len(cycle)] for b in range(B)]
        per = [{id(with_a): maps_a, id(with_b): maps_b}.get(id(r)) for r in rects]
        got = engine.debug_color_planes(plain, il, ir, rects)
    else:
        rects, per = None, [maps_a] * B
        got = engine.debug_color_planes(with_a, il, ir)
        np.testing.assert_array_equal(got[0], rectify_batch_planes(engine, with_a, il, ir))
    gl, rl = stacked_oracle(il, [None if m is None else m[:2] for m in per])
    gr, rr = stacked_oracle(ir, [None if m is None else m[2:] for m in per])
    assert_planes(got, (np.stack([gl, gr]), np.stack([rl, rr])), f"{form} {W}x{H} B={B}")
    for r in (plain, with_a, with_b):
        engine.rectifier_destroy(r)


# ---- 5. errors ----
def test_errors_leave_the_context_usable():
    e = Engine()
    W, H = 13, 11
    rng = np.random.default_rng(17)
    maps = random_maps(rng, W, H) + random_maps(rng, W, H)
    rect = e.rectifier_create_color(W, H, 4, *maps)
    plain = e.rectifier_create_color(W, H, 4)
    il = rng.integers(0, 256, (5, H, W, 4), dtype=np.uint8)
    ir = rng.integers(0, 256, (5, H, W, 4), dtype=np.uint8)
    table = [plain, None, rect, rect, None]
    want = e.debug_color_planes(rect, il, ir, table)
    other = Engine()
    foreign = other.rectifier_create_color(W, H, 4)
    grey_rect = e.rectifier_create(*maps)
    three = e.rectifier_create_color(W, H, 3)
    wider = e.rectifier_create_color(W + 1, H, 4)
    taller = e.rectifier_create_color(W, H + 1, 4)
    u8 = T.c_uint8_p
    out_g, out_r = np.zeros((2, 5, H, W), np.uint8), np.zeros((2, 5, H, W), np.uint8)
    pl, pr, pg, prgb = (a.ctypes.data_as(u8) for a in (il, ir, out_g, out_r))
    null = C.cast(None, u8)

    def call(r=rect, rects=table, B=5, a=pl, b=pr, c=pg, d=prgb):
        rarr = None if rects is None else (C.c_void_p * len(rects))(*[None if x is None else x.handle for x in rects])
        rc = e.lib.plstvo_debug_color_planes(e.ctx, None if r is None else r.handle, rarr, B, a, b, c, d)
        return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()

    def still_usable():
        got = e.debug_color_planes(rect, il, ir, table)
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])

    assert e.lib.plstvo_debug_color_planes(None, rect.handle, None, 5, pl, pr, pg, prgb) == -1
    cases = [
        (dict(r=None), "null argument"),
        (dict(a=null), "null argument"),
        (dict(b=null), "null argument"),
        (dict(c=null), "null argument"),
        (dict(d=null), "null argument"),
        (dict(B=0), "B must be at least 1"),
        (dict(B=-3), "B must be at least 1"),
        (dict(r=grey_rect, rects=None), "a grey rectifier has no RGB plane"),
        (dict(r=foreign, rects=None), "the rectifier belongs to another context"),
        (dict(rects=[plain, None, foreign, rect, None]), "a table rectifier belongs to another context"),
        (dict(rects=[plain, None, rect, wider, None]), "a table rectifier's size differs from rect's"),
        (dict(rects=[taller, None, rect, rect, None]), "a table rectifier's size differs from rect's"),
        (dict(rects=[plain, None, rect, rect, three]), "a table rectifier's channels differ from rect's"),
        (dict(rects=[plain, grey_rect, rect, rect, None]), "a table rectifier's channels differ from rect's"),
    ]
    for kw, msg in cases:
        out_g[...] = 7
        rc, got = call(**kw)
        assert rc == -1 and msg in got, (kw, rc, got)
        assert (out_g == 7).all(), kw   # nothing written on a refused call
        still_usable()
    with pytest.raises(ValueError, match="channels"):
        e.debug_color_planes(rect, il[..., :3], ir[..., :3])
    still_usable()
    other.close()
    e.close()
