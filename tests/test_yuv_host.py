"""CPU: the YUV 4:2:0 -> RGBA8 conversion of ht_tracker_feed_yuv / ht_ingest_yuv (DESIGN.md 2, "YUV video").

  * the four coefficient rows are round(256 x the real BT.601 / BT.709 matrices, limited and full range), and the
    library's per-pixel code, the C restatement tests/yuv_oracle.c (hto_yuv_to_rgba) and a numpy restatement agree on
    all 2^24 (Y, U, V) triples of each, each row within 1 level of the real-valued conversion rounded half up;
  * hto_yuv_to_rgba equals the numpy restatement on random NV12 and I420 planes of odd and even sizes with padded,
    odd pitches;
  * k_feed_draw_yuv's per-record code, compiled for the host, draws exactly hto_draw_image of hto_yuv_to_rgba's frame
    (the composition the GPU tests rely on): 1:1, down- and up-scales, NV12 and I420, aligned and unaligned planes."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)

COLORS = ("bt601", "bt709", "bt601-full", "bt709-full")
# y0, cy, rv, gu, gv, bu
TABLE = {"bt601": (16, 298, 409, 100, 208, 516), "bt709": (16, 298, 459, 55, 136, 541),
         "bt601-full": (0, 256, 359, 88, 183, 454), "bt709-full": (0, 256, 403, 48, 120, 475)}
KRKB = {"bt601": (0.299, 0.114), "bt709": (0.2126, 0.0722)}
SIZES = [(1, 1), (1, 7), (3, 5), (2, 2), (641, 481), (1280, 720)]     # (width, height)


@pytest.fixture(scope="session")
def yo(tmp_path_factory):
    """tests/yuv_oracle.c built into a temporary directory"""
    from pathlib import Path
    so = tmp_path_factory.mktemp("yuv_oracle") / "libyuv_oracle.so"
    subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-o", str(so), str(Path(__file__).with_name("yuv_oracle.c"))])
    L = C.CDLL(str(so))
    L.hto_yuv_to_rgba.argtypes = [C.c_void_p * 3, C.c_int * 3, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.hto_yuv_to_rgba.restype = None
    return L


def real_coefficients(color):
    """(y scale, rv, gu, gv, bu) of the real-valued matrix"""
    kr, kb = KRKB[color.split("-")[0]]
    full = color.endswith("-full")
    ys, cs = (1.0, 1.0) if full else (255 / 219, 255 / 224)
    kg = 1 - kr - kb
    return ys, 2 * (1 - kr) * cs, 2 * (1 - kb) * kb / kg * cs, 2 * (1 - kr) * kr / kg * cs, 2 * (1 - kb) * cs


def np_triples(color, Y, U, V):
    """the defined conversion of int64 arrays Y, U, V -> (..., 4) uint8"""
    y0, cy, rv, gu, gv, bu = TABLE[color]
    c, d, e = cy * (Y - y0), U - 128, V - 128
    out = np.empty(np.broadcast(Y, U, V).shape + (4,), np.uint8)
    out[..., 0] = np.clip((c + rv * e + 128) >> 8, 0, 255)
    out[..., 1] = np.clip((c - gu * d - gv * e + 128) >> 8, 0, 255)
    out[..., 2] = np.clip((c + bu * d + 128) >> 8, 0, 255)
    out[..., 3] = 255
    return out


def chroma_planes(frame, fmt):
    """(U, V) sample arrays of a frame's chroma planes (views)"""
    if fmt == "nv12":
        return frame[1][:, 0::2], frame[1][:, 1::2]
    return frame[1], frame[2]


def np_convert(frame, fmt, color):
    """numpy restatement: nearest chroma (x >> 1, y >> 1), then np_triples"""
    Y = frame[0].astype(np.int64)
    h, w = Y.shape
    U, V = chroma_planes(frame, fmt)
    rows, cols = np.arange(h)[:, None] >> 1, np.arange(w)[None, :] >> 1
    return np_triples(color, Y, U.astype(np.int64)[rows, cols], V.astype(np.int64)[rows, cols])


def padded_plane(a, extra, fill=0x5A):
    """a row-padded view of 2-D `a`: rows of a.shape[1] + extra bytes"""
    buf = np.full((a.shape[0], a.shape[1] + extra), fill, np.uint8)
    buf[:, :a.shape[1]] = a
    return buf[:, :a.shape[1]]


def random_frame(rng, w, h, fmt, pad=(0, 0, 0)):
    """random planes of a w x h frame, plane i row-padded by pad[i] bytes"""
    cw, ch = (w + 1) // 2, (h + 1) // 2
    shapes = [(h, w), (ch, 2 * cw)] if fmt == "nv12" else [(h, w), (ch, cw), (ch, cw)]
    return tuple(padded_plane(rng.integers(0, 256, s, dtype=np.uint8), pad[i]) for i, s in enumerate(shapes))


def yuv_image(frame, fmt, color):
    """an ht_yuv_image over a frame's host planes (the frame must outlive it)"""
    ptrs = [p.ctypes.data for p in frame] + [None] * (3 - len(frame))
    pitches = [p.strides[0] for p in frame] + [0] * (3 - len(frame))
    return _lib.YuvImage((C.c_void_p * 3)(*ptrs), (C.c_int32 * 3)(*pitches), frame[0].shape[1], frame[0].shape[0],
                         _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color])


def oracle_convert(yo, frame, fmt, color):
    """hto_yuv_to_rgba -> (h, w, 4) uint8"""
    h, w = frame[0].shape
    ptrs = (C.c_void_p * 3)(*([p.ctypes.data for p in frame] + [None] * (3 - len(frame))))
    pitches = (C.c_int * 3)(*([p.strides[0] for p in frame] + [0] * (3 - len(frame))))
    out = np.zeros((h, w, 4), np.uint8)
    yo.hto_yuv_to_rgba(ptrs, pitches, w, h, _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color], out.ctypes.data)
    return out


def oracle_draw(rgba, dw, dh):
    """hto_draw_image of an RGBA frame onto dw x dh, channel by channel"""
    sh, sw = rgba.shape[:2]
    out = np.zeros((dh, dw, 4), np.uint8)
    for c in range(4):
        out[..., c] = oracle.draw_image(np.ascontiguousarray(rgba[..., c]), 0, 0, sw, sh, dw, dh, dw, dh)
    return out


def selftest_draw(st, frame, fmt, color, dw, dh):
    st.ht_selftest_feed_yuv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    img = yuv_image(frame, fmt, color)
    canvas = np.zeros((dh, dw, 4), np.uint8)
    assert st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, dw, dh) == 0
    return canvas


def all_triples_frame(Y):
    """an I420 512 x 512 frame of constant luma Y whose chroma sample (cx, cy) is (U, V) = (cx, cy): every (U, V) pair"""
    U = np.tile(np.arange(256, dtype=np.uint8)[None, :], (256, 1))
    return (np.full((512, 512), Y, np.uint8), U, np.ascontiguousarray(U.T))


# ---- the coefficients -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("color", COLORS)
def test_coefficients_are_the_rounded_real_matrices(color):
    ys, rv, gu, gv, bu = real_coefficients(color)
    y0, cy, irv, igu, igv, ibu = TABLE[color]
    assert (y0 == 0) == color.endswith("-full")
    assert [cy, irv, igu, igv, ibu] == [int(np.floor(256 * c + 0.5)) for c in (ys, rv, gu, gv, bu)]


@pytest.mark.parametrize("color", COLORS)
def test_every_triple_library_oracle_numpy_and_within_one_level(st, yo, color):
    """256 frames of constant luma, each holding all 65536 (U, V) pairs: the library's per-pixel code (host build), the
    C restatement and numpy agree on all 2^24 triples, and each is within 1 level of the real-valued conversion"""
    ys, rv, gu, gv, bu = real_coefficients(color)
    y0 = TABLE[color][0]
    U = np.arange(256, dtype=np.int64)[None, :]
    V = np.arange(256, dtype=np.int64)[:, None]
    worst = 0
    for Y in range(256):
        f = all_triples_frame(Y)
        want = np_triples(color, np.int64(Y), U, V)                      # [V][U]
        lib = selftest_draw(st, f, "i420", color, 512, 512)[0::2, 0::2]  # chroma sample (U, V) = (x >> 1, y >> 1)
        assert np.array_equal(lib, want), (color, Y)
        assert np.array_equal(oracle_convert(yo, f, "i420", color)[1::2, 1::2], want), (color, Y)
        c = ys * (Y - y0)
        real = np.stack([c + rv * (V - 128) + 0 * U, c - gu * (U - 128) - gv * (V - 128), c + bu * (U - 128) + 0 * V], -1)
        real = np.clip(np.floor(real + 0.5), 0, 255)
        worst = max(worst, int(np.abs(want[..., :3].astype(np.int64) - real).max()))
    assert worst == 1, worst             # within one level, and the rounding does show


# ---- the C restatement against numpy --------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", ["nv12", "i420"])
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_oracle_equals_numpy(yo, fmt, size):
    w, h = size
    rng = np.random.default_rng(w * 7919 + h)
    for i, color in enumerate(COLORS):
        pad = [(0, 0, 0), (3, 1, 5), (17, 2, 1), (1, 9, 3)][i]             # tight, and odd pitches
        f = random_frame(rng, w, h, fmt, pad)
        assert np.array_equal(oracle_convert(yo, f, fmt, color), np_convert(f, fmt, color)), (fmt, size, color)


# ---- the device draw's per-record code ------------------------------------------------------------------------------

DRAWS = [((1280, 720), (1280, 720)), ((640, 480), (640, 480)), ((641, 481), (641, 481)), ((33, 17), (33, 17)),
         ((1280, 720), (320, 240)), ((641, 481), (160, 120)), ((33, 17), (200, 150))]


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
@pytest.mark.parametrize("draw", DRAWS, ids=[f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in DRAWS])
def test_draw_is_the_resampler_over_the_converted_frame(st, yo, fmt, draw):
    (w, h), (dw, dh) = draw
    rng = np.random.default_rng(w + 13 * dw)
    for color, pad, offset in (("bt601", (0, 0, 0), 0), ("bt709-full", (3, 5, 1), 1), ("bt709", (4, 8, 8), 2),
                               ("bt601-full", (1, 2, 3), 3)):
        f = random_frame(rng, w, h, fmt, pad)
        if offset:                        # planes starting off a 4-byte boundary: the byte-load paths
            f = tuple(padded_plane(np.pad(p, ((0, 0), (offset, 0))), 3)[:, offset:] for p in f)
        want = oracle_draw(oracle_convert(yo, f, fmt, color), dw, dh)
        assert np.array_equal(selftest_draw(st, f, fmt, color, dw, dh), want), (fmt, draw, color, offset)


def test_selftest_rejects_what_the_library_rejects(st):
    st.ht_selftest_feed_yuv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    f = random_frame(np.random.default_rng(1), 8, 4, "nv12")
    canvas = np.zeros((4, 8, 4), np.uint8)
    for field, value in (("format", 2), ("color", 4), ("width", 0)):
        img = yuv_image(f, "nv12", "bt601")
        setattr(img, field, value)
        rc = st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, 8, 4)
        assert rc == (_lib.HT_ERR_SIZE if field == "width" else _lib.HT_ERR_ARG), field
    img = yuv_image(f, "nv12", "bt601")
    img.pitch[1] = 7                                                     # below 2 * ceil(8 / 2)
    assert st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, 8, 4) == _lib.HT_ERR_ARG
    img = yuv_image(f, "nv12", "bt601")
    img.planes[2] = f[1].ctypes.data                                     # a third plane for NV12
    assert st.ht_selftest_feed_yuv(C.addressof(img), canvas.ctypes.data, 8, 4) == _lib.HT_ERR_ARG
    assert not canvas.any()


def test_yuv_abi():
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_feed_yuv") and hasattr(L, "ht_ingest_yuv")
    assert C.sizeof(_lib.YuvImage) == 56 and C.sizeof(_lib.YuvFrame) == 80
    assert (_lib.YuvImage.pitch.offset, _lib.YuvImage.width.offset, _lib.YuvImage.height.offset,
            _lib.YuvImage.format.offset, _lib.YuvImage.color.offset) == (24, 36, 40, 44, 48)
    assert (_lib.YuvFrame.stream.offset, _lib.YuvFrame.canvas_w.offset, _lib.YuvFrame.canvas_h.offset,
            _lib.YuvFrame.now_ms.offset) == (56, 60, 64, 72)
    assert L.ht_version() == (1 << 16) | 3
