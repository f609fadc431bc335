"""CPU: the video formats of ht_yuv_image beyond NV12 / I420 (NV21, I422, I444, YUYV, UYVY, P010, BGRA, BGR24, RGB24)
and the BT.2020 colour (DESIGN.md 2, "YUV video").

  * the two BT.2020 rows are round(256 x the real non-constant-luminance matrix), within 1 level of the real-valued
    conversion over all 2^24 triples, and the library's per-pixel code, the C restatement tests/format_oracle.c and a
    numpy restatement agree on all of them;
  * format_oracle.c equals an independent numpy restatement on random frames of every format, 1x1 to 1280x720, with
    tight, padded and odd pitches, P010 samples around every rounding edge;
  * identities through the library's host-compiled draw tie every new format to NV12 / I420 / RGBA;
  * the draw (ht_selftest_feed_yuv) equals hto_draw_image of format_oracle's frame bit for bit, for every format and
    colour, 1:1, down- and up-scaled, with planes on and off 2-, 4- and 16-byte boundaries;
  * every new rejection, the ABI constants, and a spill-free k_feed_draw_yuv."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_yuv_host import oracle_draw

NEW = ["nv21", "i422", "i444", "yuyv", "uyvy", "p010", "bgra", "bgr24", "rgb24"]
RGB = {"bgra", "bgr24", "rgb24"}
YUV_COLORS = ["bt601", "bt709", "bt601-full", "bt709-full", "bt2020", "bt2020-full"]
# y0, cy, rv, gu, gv, bu
TABLE = {"bt601": (16, 298, 409, 100, 208, 516), "bt709": (16, 298, 459, 55, 136, 541),
         "bt601-full": (0, 256, 359, 88, 183, 454), "bt709-full": (0, 256, 403, 48, 120, 475),
         "bt2020": (16, 298, 430, 48, 167, 548), "bt2020-full": (0, 256, 377, 42, 146, 482)}


def colors_of(fmt):
    return ["bt601"] if fmt in RGB else YUV_COLORS


@pytest.fixture(scope="session")
def fo(tmp_path_factory):
    """tests/format_oracle.c built into a temporary directory"""
    so = tmp_path_factory.mktemp("format_oracle") / "libformat_oracle.so"
    subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", str(so), str(Path(__file__).with_name("format_oracle.c"))])
    L = C.CDLL(str(so))
    L.hto_format_to_rgba.argtypes = [C.c_void_p * 3, C.c_int * 3, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.hto_format_to_rgba.restype = None
    return L


# ---- frames: (fmt, w, h, planes), each plane a 2-D uint8 view of its bytes (P010: 2 bytes per sample) ----------------

def plane_shapes(fmt, w, h):
    """(rows, tight pitch in bytes) of each plane (the table at ht_yuv_image)"""
    cw, ch = (w + 1) // 2, (h + 1) // 2
    return {"nv12": [(h, w), (ch, 2 * cw)], "nv21": [(h, w), (ch, 2 * cw)], "i420": [(h, w), (ch, cw), (ch, cw)],
            "i422": [(h, w), (h, cw), (h, cw)], "i444": [(h, w), (h, w), (h, w)], "yuyv": [(h, 4 * cw)],
            "uyvy": [(h, 4 * cw)], "p010": [(h, 2 * w), (ch, 4 * cw)], "bgra": [(h, 4 * w)], "bgr24": [(h, 3 * w)],
            "rgb24": [(h, 3 * w)]}[fmt]


def place(a, offset=0, extra=0, fill=0x5A):
    """2-D uint8 `a` copied into a fresh buffer whose row 0 starts `offset` bytes past a 64-byte boundary, rows of
    a.shape[1] + extra bytes -> the view"""
    rows, cols = a.shape
    pitch = cols + extra
    buf = np.full(rows * pitch + 128 + offset, fill, np.uint8)
    start = (-buf.ctypes.data) % 64 + offset
    view = np.lib.stride_tricks.as_strided(buf[start:], shape=(rows, cols), strides=(pitch, 1))
    view[...] = a
    return view


P010_EDGES = np.array([0x0000, 0x007F, 0x0080, 0x00FF, 0x0100, 0x017F, 0x0180, 0x7F7F, 0x7F80, 0xFE7F, 0xFE80, 0xFEFF,
                       0xFF00, 0xFF7F, 0xFF80, 0xFFC0, 0xFFFF, 64 << 6, 940 << 6, 512 << 6, (64 << 6) | 0x3F], np.uint16)


def random_plane(rng, fmt, rows, cols):
    if fmt != "p010":
        return rng.integers(0, 256, (rows, cols), dtype=np.uint8)
    s = rng.integers(0, 1 << 16, (rows, cols // 2), dtype=np.uint16)
    mask = rng.random(s.shape) < 0.3
    s[mask] = rng.choice(P010_EDGES, int(mask.sum()))
    return np.ascontiguousarray(s.astype("<u2")).view(np.uint8)


def random_frame(rng, fmt, w, h, offsets=(0, 0, 0), extras=(0, 0, 0)):
    return fmt, w, h, tuple(place(random_plane(rng, fmt, r, c), offsets[i], extras[i])
                            for i, (r, c) in enumerate(plane_shapes(fmt, w, h)))


def image(frame, color):
    fmt, w, h, planes = frame
    ptrs = [p.ctypes.data for p in planes] + [None] * (3 - len(planes))
    pitches = [p.strides[0] for p in planes] + [0] * (3 - len(planes))
    return _lib.YuvImage((C.c_void_p * 3)(*ptrs), (C.c_int32 * 3)(*pitches), w, h, _lib.YUV_FORMATS[fmt],
                         _lib.YUV_COLORS[color])


def oracle_convert(fo, frame, color):
    fmt, w, h, planes = frame
    ptrs = (C.c_void_p * 3)(*([p.ctypes.data for p in planes] + [None] * (3 - len(planes))))
    pitches = (C.c_int * 3)(*([p.strides[0] for p in planes] + [0] * (3 - len(planes))))
    out = np.zeros((h, w, 4), np.uint8)
    fo.hto_format_to_rgba(ptrs, pitches, w, h, _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color], out.ctypes.data)
    return out


def selftest_draw(st, frame, color, dw, dh):
    st.ht_selftest_feed_yuv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    img = image(frame, color)
    canvas = np.zeros((dh, dw, 4), np.uint8)
    assert st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, dw, dh) == 0
    return canvas


# ---- numpy restatement ----------------------------------------------------------------------------------------------

def np_triples(color, Y, U, V):
    y0, cy, rv, gu, gv, bu = TABLE[color]
    c, d, e = cy * (Y - y0), U - 128, V - 128
    out = np.empty(np.broadcast(Y, U, V).shape + (4,), np.uint8)
    out[..., 0] = np.clip((c + rv * e + 128) >> 8, 0, 255)
    out[..., 1] = np.clip((c - gu * d - gv * e + 128) >> 8, 0, 255)
    out[..., 2] = np.clip((c + bu * d + 128) >> 8, 0, 255)
    out[..., 3] = 255
    return out


def np_convert(frame, color):
    fmt, w, h, P = frame
    P = [p.astype(np.int64) for p in P]
    y, x = np.arange(h)[:, None], np.arange(w)[None, :]
    hx, hy = x >> 1, y >> 1

    def r16(p, row, i):                  # sample i of a P010 row, reduced
        return np.minimum(255, ((p[row, 2 * i] | p[row, 2 * i + 1] << 8) + 128) >> 8)

    if fmt in RGB:
        n = 4 if fmt == "bgra" else 3
        px = [P[0][y, n * x + k] for k in range(n)]
        r, g, b = (px[2], px[1], px[0]) if fmt != "rgb24" else (px[0], px[1], px[2])
        a = px[3] if fmt == "bgra" else np.full((h, w), 255)
        return np.stack([np.broadcast_to(c, (h, w)) for c in (r, g, b, a)], -1).astype(np.uint8)
    if fmt == "nv12":
        Y, U, V = P[0][y, x], P[1][hy, 2 * hx], P[1][hy, 2 * hx + 1]
    elif fmt == "nv21":
        Y, V, U = P[0][y, x], P[1][hy, 2 * hx], P[1][hy, 2 * hx + 1]
    elif fmt == "i420":
        Y, U, V = P[0][y, x], P[1][hy, hx], P[2][hy, hx]
    elif fmt == "i422":
        Y, U, V = P[0][y, x], P[1][y, hx], P[2][y, hx]
    elif fmt == "i444":
        Y, U, V = P[0][y, x], P[1][y, x], P[2][y, x]
    elif fmt == "yuyv":
        Y, U, V = P[0][y, 2 * x], P[0][y, 4 * hx + 1], P[0][y, 4 * hx + 3]
    elif fmt == "uyvy":
        Y, U, V = P[0][y, 2 * x + 1], P[0][y, 4 * hx], P[0][y, 4 * hx + 2]
    else:
        Y, U, V = r16(P[0], y, x), r16(P[1], hy, 2 * hx), r16(P[1], hy, 2 * hx + 1)
    return np_triples(color, Y, U, V)


# ---- 1. BT.2020 -----------------------------------------------------------------------------------------------------

def real_bt2020(full):
    kr, kb = 0.2627, 0.0593
    kg = 1 - kr - kb
    ys, cs = (1.0, 1.0) if full else (255 / 219, 255 / 224)
    return ys, 2 * (1 - kr) * cs, 2 * (1 - kb) * kb / kg * cs, 2 * (1 - kr) * kr / kg * cs, 2 * (1 - kb) * cs


@pytest.mark.parametrize("color", ["bt2020", "bt2020-full"])
def test_bt2020_rows_are_the_rounded_real_matrix(color):
    y0, *ints = TABLE[color]
    assert (y0 == 0) == color.endswith("-full")
    assert ints == [int(np.floor(256 * c + 0.5)) for c in real_bt2020(color.endswith("-full"))]
    # every intermediate of the int32 path stays below 2^18
    cy, rv, gu, gv, bu = ints
    assert cy * 255 + max(rv, bu, gu + gv) * 128 < 1 << 18


@pytest.mark.parametrize("color", ["bt2020", "bt2020-full"])
def test_bt2020_every_triple_library_oracle_numpy_and_within_one_level(st, fo, color):
    """I444 frames of constant luma, chroma sample (x, y) = (U, V): all 2^24 triples through the library's draw, the C
    restatement and numpy, each within 1 level of the real-valued conversion"""
    ys, rv, gu, gv, bu = real_bt2020(color.endswith("-full"))
    y0 = TABLE[color][0]
    U = np.arange(256, dtype=np.int64)[None, :]
    V = np.arange(256, dtype=np.int64)[:, None]
    Up = np.tile(np.arange(256, dtype=np.uint8)[None, :], (256, 1))
    worst = 0
    for Y in range(256):
        f = ("i444", 256, 256, (np.full((256, 256), Y, np.uint8), Up, np.ascontiguousarray(Up.T)))
        want = np_triples(color, np.int64(Y), U, V)
        assert np.array_equal(selftest_draw(st, f, color, 256, 256), want), (color, Y)
        assert np.array_equal(oracle_convert(fo, f, color), want), (color, Y)
        c = ys * (Y - y0)
        real = np.stack([c + rv * (V - 128) + 0 * U, c - gu * (U - 128) - gv * (V - 128), c + bu * (U - 128) + 0 * V], -1)
        real = np.clip(np.floor(real + 0.5), 0, 255)
        worst = max(worst, int(np.abs(want[..., :3].astype(np.int64) - real).max()))
    assert worst == 1, worst


# ---- 2. the C restatement against numpy -----------------------------------------------------------------------------

SIZES = [(1, 1), (1, 7), (2, 2), (3, 5), (7, 3), (33, 17), (641, 481), (1280, 720)]


@pytest.mark.parametrize("fmt", NEW + ["nv12", "i420"])
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_format_oracle_equals_numpy(fo, fmt, size):
    w, h = size
    rng = np.random.default_rng(w * 7919 + h + 31 * len(fmt))
    even = fmt == "p010"
    layouts = [((0, 0, 0), (0, 0, 0)), ((0, 0, 0), (6, 2, 4)) if even else ((1, 3, 5), (3, 1, 5)),
               ((2, 2, 2), (18, 2, 8)) if even else ((3, 1, 2), (17, 9, 1))]
    for i, color in enumerate(colors_of(fmt)):
        offsets, extras = layouts[i % 3]
        f = random_frame(rng, fmt, w, h, offsets, extras)
        assert np.array_equal(oracle_convert(fo, f, color), np_convert(f, color)), (fmt, size, color)


def test_p010_reduction_edges(fo):
    """r(s) = min(255, (s + 128) >> 8): 0x..7F rounds down, 0x..80 up, 0xFF80 and above clamp; 10-bit nominal levels"""
    s = np.array([0x007F, 0x0080, 0x107F, 0x1080, 0xFF7F, 0xFF80, 0xFFFF, 64 << 6, 940 << 6, 512 << 6], np.uint16)
    want = [0, 1, 16, 17, 255, 255, 255, 16, 235, 128]
    w = len(s)
    uv = np.full(2 * ((w + 1) // 2), 512 << 6, np.uint16)
    f = ("p010", w, 1, (s[None].astype("<u2").view(np.uint8), uv[None].astype("<u2").view(np.uint8)))
    got = oracle_convert(fo, f, "bt601-full")                          # full range, neutral chroma: R = G = B = Y
    assert got[0, :, 0].tolist() == want


# ---- 3. identities through the library's draw -----------------------------------------------------------------------

def rgba_draw(st, rgba, dw, dh):
    """the library's RGBA resampler (k_ingest's per-pixel code) over one frame"""
    st.ht_selftest_ingest.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    h, w = rgba.shape[:2]
    src = np.ascontiguousarray(rgba)
    out = np.zeros((1, dh, dw, 4), np.uint8)
    assert st.ht_selftest_ingest(src.ctypes.data, 1, w, h, out.ctypes.data, dw, dh) == 0
    return out[0]


IDRAWS = [((64, 48), (64, 48)), ((33, 17), (33, 17)), ((641, 481), (160, 120)), ((33, 17), (100, 60))]


@pytest.mark.parametrize("draw", IDRAWS, ids=[f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in IDRAWS])
def test_identities_with_nv12_i420_and_rgba(st, draw):
    (w, h), (dw, dh) = draw
    rng = np.random.default_rng(w * 3 + dw)
    for color in YUV_COLORS:
        d = lambda f: selftest_draw(st, f, color, dw, dh)            # noqa: E731
        # NV21 = NV12 with the chroma bytes swapped
        _, _, _, (Y, UV) = random_frame(rng, "nv12", w, h)
        VU = UV.copy()
        VU[:, 0::2], VU[:, 1::2] = UV[:, 1::2], UV[:, 0::2]
        assert np.array_equal(d(("nv21", w, h, (Y, VU))), d(("nv12", w, h, (Y, UV)))), color
        # YUYV = UYVY with the bytes of each pair swapped = I422 of the de-interleaved planes
        _, _, _, (P,) = random_frame(rng, "yuyv", w, h)
        Q = P.copy()
        Q[:, 0::2], Q[:, 1::2] = P[:, 1::2], P[:, 0::2]
        yuyv = d(("yuyv", w, h, (P,)))
        assert np.array_equal(yuyv, d(("uyvy", w, h, (Q,)))), color
        i422 = (np.ascontiguousarray(P[:, 0::2][:, :w]), np.ascontiguousarray(P[:, 1::4]), np.ascontiguousarray(P[:, 3::4]))
        assert np.array_equal(yuyv, d(("i422", w, h, i422))), color
        # I444 with chroma constant on 2x2 blocks = I420 of the subsampled chroma
        _, _, _, (Y, U, V) = random_frame(rng, "i420", w, h)
        up = lambda c: np.ascontiguousarray(np.repeat(np.repeat(c, 2, 0), 2, 1)[:h, :w])   # noqa: E731
        i420 = d(("i420", w, h, (Y, U, V)))
        assert np.array_equal(d(("i444", w, h, (Y, up(U), up(V)))), i420), color
        # I422 whose chroma rows repeat in pairs = I420
        rows = lambda c: np.ascontiguousarray(np.repeat(c, 2, 0)[:h])  # noqa: E731
        assert np.array_equal(d(("i422", w, h, (Y, rows(U), rows(V)))), i420), color
        # P010 = NV12 of r(s)
        _, _, _, (Yb, UVb) = random_frame(rng, "p010", w, h)
        red = lambda b: np.minimum(255, (b.view("<u2").astype(np.int64) + 128) >> 8).astype(np.uint8)  # noqa: E731
        assert np.array_equal(d(("p010", w, h, (np.ascontiguousarray(Yb), np.ascontiguousarray(UVb)))),
                              d(("nv12", w, h, (red(np.ascontiguousarray(Yb)), red(np.ascontiguousarray(UVb)))))), color
    # BGRA = RGBA with bytes 0 and 2 swapped; BGR24 / RGB24 = RGBA with A = 255
    rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    bgra = rgba[..., [2, 1, 0, 3]].reshape(h, 4 * w)
    assert np.array_equal(selftest_draw(st, ("bgra", w, h, (np.ascontiguousarray(bgra),)), "bt601", dw, dh),
                          rgba_draw(st, rgba, dw, dh))
    opaque = rgba.copy()
    opaque[..., 3] = 255
    bgr = np.ascontiguousarray(rgba[..., [2, 1, 0]].reshape(h, 3 * w))
    rgb = np.ascontiguousarray(rgba[..., :3].reshape(h, 3 * w))
    want = rgba_draw(st, opaque, dw, dh)
    assert np.array_equal(selftest_draw(st, ("bgr24", w, h, (bgr,)), "bt601", dw, dh), want)
    assert np.array_equal(selftest_draw(st, ("rgb24", w, h, (rgb,)), "bt601", dw, dh), want)


# ---- 4. the draw against the oracle ---------------------------------------------------------------------------------

DRAWS = [((1280, 720), (1280, 720)), ((640, 480), (640, 480)), ((641, 481), (641, 481)), ((33, 17), (33, 17)),
         ((36, 8), (36, 8)), ((1280, 720), (320, 240)), ((641, 481), (160, 120)), ((33, 17), (200, 150))]


@pytest.mark.parametrize("fmt", NEW)
@pytest.mark.parametrize("draw", DRAWS, ids=[f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in DRAWS])
def test_draw_is_the_resampler_over_the_oracle_frame(st, fo, fmt, draw):
    (w, h), (dw, dh) = draw
    rng = np.random.default_rng(w + 13 * dw + 7 * len(fmt))
    colors = colors_of(fmt)
    i0 = DRAWS.index(draw)
    # planes on 16-byte boundaries, and off them by 2, 4 and 1 bytes (P010: 2 and 6, odd multiples of 2)
    layouts = ([(0, 0), (2, 4), (6, 2), (16, 10)] if fmt == "p010" else [(0, 0), (2, 3), (4, 5), (1, 1)])
    for j, (off, extra) in enumerate(layouts):
        color = colors[(i0 + j) % len(colors)]
        f = random_frame(rng, fmt, w, h, (off, off, off), (extra, 2 * extra, extra))
        want = oracle_draw(oracle_convert(fo, f, color), dw, dh)
        assert np.array_equal(selftest_draw(st, f, color, dw, dh), want), (fmt, draw, color, off)


@pytest.mark.parametrize("fmt", [f for f in NEW if f not in RGB] + ["nv12", "i420"])
def test_every_colour_every_format(st, fo, fmt):
    rng = np.random.default_rng(len(fmt))
    for color in YUV_COLORS:
        for (w, h), (dw, dh) in (((64, 36), (64, 36)), ((65, 37), (40, 30))):
            f = random_frame(rng, fmt, w, h)
            want = oracle_draw(oracle_convert(fo, f, color), dw, dh)
            assert np.array_equal(selftest_draw(st, f, color, dw, dh), want), (fmt, color, w)


# ---- 5. rejections and the ABI --------------------------------------------------------------------------------------

def test_selftest_rejects_every_new_bad_record(st):
    st.ht_selftest_feed_yuv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    rng = np.random.default_rng(2)
    canvas = np.zeros((4, 8, 4), np.uint8)
    spare = np.zeros(64, np.uint8)
    rc = lambda img: st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, 8, 4)   # noqa: E731
    n = 0
    for fmt in NEW:
        f = random_frame(rng, fmt, 8, 4)
        used = len(f[3])
        for color in ([1, 2, 3, 8, 10, 4, 9, 11, -1] if fmt in RGB else [4, 5, 6, 7, 9, 11, 12, 16, -1]):
            img = image(f, "bt601")
            img.color = color
            assert rc(img) == _lib.HT_ERR_ARG, (fmt, color)
            n += 1
        for p in range(3):
            img = image(f, "bt601")
            if p < used:
                img.planes[p] = None                                    # a required plane missing
                assert rc(img) == _lib.HT_ERR_ARG, (fmt, p)
                img = image(f, "bt601")
                img.pitch[p] = plane_shapes(fmt, 8, 4)[p][1] - 1        # below the tight pitch
                assert rc(img) == _lib.HT_ERR_ARG, (fmt, p)
            else:
                img.planes[p] = spare.ctypes.data                       # a plane the format does not use
                assert rc(img) == _lib.HT_ERR_ARG, (fmt, p)
            n += 1
        if fmt == "p010":
            for p in range(2):
                img = image(f, "bt601")
                img.planes[p] = img.planes[p] + 1                       # an odd plane pointer
                assert rc(img) == _lib.HT_ERR_ARG, p
                img = image(f, "bt601")
                img.pitch[p] = plane_shapes(fmt, 8, 4)[p][1] + 1        # an odd pitch
                assert rc(img) == _lib.HT_ERR_ARG, p
    f = random_frame(rng, "nv12", 8, 4)
    for format_ in (2, 3, 15, 22, 31, 35, -1):
        img = image(f, "bt601")
        img.format = format_
        assert rc(img) == _lib.HT_ERR_ARG, format_
    assert n > 0 and not canvas.any()


def test_formats_abi():
    L = _lib.lib()
    assert C.sizeof(_lib.YuvImage) == 56 and C.sizeof(_lib.YuvFrame) == 80
    assert _lib.YUV_FORMATS == {"nv12": 0, "i420": 1, "nv21": 16, "i422": 17, "i444": 18, "yuyv": 19, "uyvy": 20,
                                "p010": 21, "bgra": 32, "bgr24": 33, "rgb24": 34}
    assert _lib.YUV_COLORS == {"bt601": 0, "bt709": 1, "bt601-full": 2, "bt709-full": 3, "bt2020": 8, "bt2020-full": 10}
    header = (Path(__file__).resolve().parent.parent / "include" / "headtrackr_b200.h").read_text()
    for name, value in list(_lib.YUV_FORMATS.items()) + [("bt2020", 8)]:
        assert re.search(rf"#define HT_YUV_{name.upper()} {value}\b", header), name
    assert L.ht_version() == (1 << 16) | 3


def test_feed_draw_yuv_does_not_spill(tmp_path):
    """ptxas -v of the library as build() compiles it: k_feed_draw_yuv and its out-of-line CTA for the formats other
    than NV12 / I420 (feed_draw_fmt) keep everything in registers, within the 48 that give five 256-thread CTAs per SM"""
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    m = re.search(r"Function properties for \S*k_feed_draw_yuv\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*Used (\d+) registers", out)
    assert m, out[-2000:]
    assert (m.group(2), m.group(3)) == ("0", "0") and int(m.group(4)) <= 48, m.group(0)
    f = re.search(r"Function properties for \S*feed_draw_fmt\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", out)
    assert f, out[-2000:]
    assert (f.group(2), f.group(3)) == ("0", "0"), f.group(0)
