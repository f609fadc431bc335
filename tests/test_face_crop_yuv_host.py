"""CPU: YUV face crops (DESIGN.md 2, "Face crops", item 5) through the host build of k_face_crop's per-crop code
(ht_selftest_face_crop_yuv) and of the conversion (ht_selftest_rgba_to_yuv420), against the independent C restatement
tests/crop_yuv_oracle.c and numpy:

  * the coefficient table is the one the derivation rule gives from the real BT.601 / BT.709 matrices (in numpy and in
    the restatement), and over all 2^24 RGB triples the library, the restatement and numpy agree; every row hits its
    sum, stays within one level of the real conversion rounded half up (and reaches it), greys give U = V = 128, the
    limited range stays nominal, and the round trip through yuv_to_rgba's rows is within 3 levels (limited) / 2 (full);
  * a block's chroma is the box mean of its four pixels, the same in all three;
  * the host-built YUV crop equals the restatement's conversion of the host-built RGBA crop, bit for bit, over the face
    crop corpus (golden CS boxes, random rotated boxes with NaN angles, scales 0.25 to 16, every orientation x mirror x
    source rectangle, every input format and colour), with odd pitches and plane offsets whose padding stays;
  * the new bodies do not spill, and the ABI exports the setter."""
import ctypes as C
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_face_crop_host import HALF_PI, event, golden_cs_boxes, lib_crop_rgba, lib_crop_yuv, smooth_frame
from test_formats_host import NEW, colors_of, fo, image, random_frame  # noqa: F401
from test_views_host import view_of

COLORS = ["bt601", "bt709", "bt601-full", "bt709-full"]
TABLE = {  # y0, (yr, yg, yb), (ur, ug, ub), (vr, vg, vb), as DESIGN.md and include/headtrackr_b200.h state them
    "bt601": (16, (66, 129, 25), (-38, -74, 112), (112, -94, -18)),
    "bt709": (16, (47, 157, 16), (-26, -86, 112), (112, -102, -10)),
    "bt601-full": (0, (77, 150, 29), (-43, -85, 128), (128, -107, -21)),
    "bt709-full": (0, (54, 183, 19), (-29, -99, 128), (128, -116, -12)),
}
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def yo(tmp_path_factory):
    """tests/crop_yuv_oracle.c built into a temporary directory"""
    lib = tmp_path_factory.mktemp("crop_yuv_oracle") / "libcrop_yuv_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("crop_yuv_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hcyo_rows.argtypes = [C.c_int, C.c_void_p]
    L.hcyo_rows.restype = None
    L.hcyo_blocks.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    L.hcyo_blocks.restype = None
    L.hcyo_convert.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                               C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    L.hcyo_convert.restype = None
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_face_crop.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_crop_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_crop_yuv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_rgba_to_yuv420.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    st.ht_selftest_rgba_to_yuv420.restype = None
    return st


# ---- the conversion ---------------------------------------------------------------------------------------------------

def derive(color):
    """the table row by the derivation rule, from the real matrix"""
    kr, kb = (0.2126, 0.0722) if "709" in color else (0.299, 0.114)
    kg, full = 1 - kr - kb, color.endswith("full")
    ys, cs = (1.0, 1.0) if full else (219 / 255, 224 / 255)
    real = [np.array([kr, kg, kb]) * ys, np.array([-kr / (1 - kb) / 2, -kg / (1 - kb) / 2, 0.5]) * cs,
            np.array([0.5, -kg / (1 - kr) / 2, -kb / (1 - kr) / 2]) * cs]
    rows = []
    for r, target, keep in zip(real, (256 if full else 220, 0, 0), (None, 2, 0)):
        q = np.floor(256 * r + 0.5).astype(int)
        while q.sum() != target:
            step = 1 if q.sum() < target else -1
            err = [(abs(256 * r[i] - q[i]), i) for i in range(3) if i != keep and np.sign(256 * r[i] - q[i]) == step]
            q[max(err)[1]] += step
        rows.append(tuple(int(v) for v in q))
    return (0 if full else 16,) + tuple(rows), real


def np_convert(color, R, G, B, SR=None, SG=None, SB=None):
    """numpy restatement: Y per pixel, U / V from block sums (default: a uniform block, sums 4x)"""
    y0, ky, ku, kv = TABLE[color]
    SR, SG, SB = (4 * R if SR is None else SR), (4 * G if SG is None else SG), (4 * B if SB is None else SB)
    Y = y0 + ((ky[0] * R + ky[1] * G + ky[2] * B + 128) >> 8)
    U = np.clip(128 + ((ku[0] * SR + ku[1] * SG + ku[2] * SB + 512) >> 10), 0, 255)
    V = np.clip(128 + ((kv[0] * SR + kv[1] * SG + kv[2] * SB + 512) >> 10), 0, 255)
    return Y, U, V


def yuv_to_rgb_np(color, Y, U, V):
    """yuv_to_rgba's rows (ht_detect.cuh) for BT.601 / BT.709"""
    full, bt709 = color.endswith("full"), "709" in color
    y0, cy = (0, 256) if full else (16, 298)
    rv, gu, gv, bu = {(False, False): (409, 100, 208, 516), (False, True): (459, 55, 136, 541),
                      (True, False): (359, 88, 183, 454), (True, True): (403, 48, 120, 475)}[(full, bt709)]
    c, d, e = cy * (Y - y0), U - 128, V - 128
    return [np.clip((x + 128) >> 8, 0, 255) for x in (c + rv * e, c - gu * d - gv * e, c + bu * d)]


def all_triples():
    i = np.arange(1 << 24, dtype=np.int64)
    return i & 255, (i >> 8) & 255, i >> 16


def blocks_call(fn, color, blocks):
    """fn (the library's or the restatement's) over (n, 4) uint32 blocks -> (n, 6) uint8"""
    out = np.empty((len(blocks), 6), np.uint8)
    fn(_lib.YUV_COLORS[color], np.ascontiguousarray(blocks, np.uint32).ctypes.data, len(blocks), out.ctypes.data)
    return out


@pytest.mark.parametrize("color", COLORS)
def test_table_is_the_derived_one(yo, color):
    rows, _ = derive(color)
    assert rows == TABLE[color]
    k = (C.c_int * 10)()
    yo.hcyo_rows(_lib.YUV_COLORS[color], k)
    assert tuple(k) == (rows[0],) + rows[1] + rows[2] + rows[3]


@pytest.mark.parametrize("color", COLORS)
def test_all_triples(lib, yo, color):
    y0, ky, ku, kv = TABLE[color]
    full = color.endswith("full")
    assert sum(ky) == (256 if full else 220) and sum(ku) == sum(kv) == 0 and ku[2] == kv[0] == (128 if full else 112)
    R, G, B = all_triples()
    Y, U, V = np_convert(color, R, G, B)
    for start in range(0, 1 << 24, 1 << 22):      # the library and the restatement on uniform 2 x 2 blocks
        s = slice(start, start + (1 << 22))
        px = (R[s] | G[s] << 8 | B[s] << 16 | 255 << 24).astype(np.uint32)
        blocks = np.repeat(px[:, None], 4, axis=1)
        want = np.stack([Y[s]] * 4 + [U[s], V[s]], 1).astype(np.uint8)
        assert np.array_equal(blocks_call(lib.ht_selftest_rgba_to_yuv420, color, blocks), want), start
        assert np.array_equal(blocks_call(yo.hcyo_blocks, color, blocks), want), start
    _, real = derive(color)
    for got, row, off in ((Y, real[0], y0), (U, real[1], 128), (V, real[2], 128)):
        exact = np.floor(off + row[0] * R + row[1] * G + row[2] * B + 0.5)
        err = np.abs(got - np.clip(exact, 0, 255))
        assert err.max() == 1, color
    if full:                                         # pure blue needs the clamp
        assert np_convert(color, 0, 0, 255)[1] == 255 and 128 + ((ku[2] * 4 * 255 + 512) >> 10) == 256
    else:
        assert Y.min() == 16 and Y.max() == 235 and U.min() >= 16 and U.max() <= 240 and V.min() >= 16 and V.max() <= 240
    grey = R == G
    grey &= G == B
    assert (U[grey] == 128).all() and (V[grey] == 128).all()
    back = yuv_to_rgb_np(color, Y, U, V)
    worst = max(int(np.abs(b - c).max()) for b, c in zip(back, (R, G, B)))
    assert worst == (2 if full else 3), worst
    gworst = max(int(np.abs(b[grey] - R[grey]).max()) for b in back)
    assert gworst == (0 if full else 1), gworst


@pytest.mark.parametrize("color", COLORS)
def test_block_chroma_is_the_box_mean(lib, yo, color):
    rng = np.random.default_rng(len(color))
    px = rng.integers(0, 1 << 32, (1 << 18, 4), dtype=np.uint64).astype(np.uint32)
    px[:1000] = px[:1000, :1]                            # some uniform blocks among them
    got = blocks_call(lib.ht_selftest_rgba_to_yuv420, color, px)
    assert np.array_equal(got, blocks_call(yo.hcyo_blocks, color, px))
    ch = [(px.astype(np.int64) >> (8 * c)) & 255 for c in range(3)]
    Y, U, V = np_convert(color, *ch, *[c.sum(1) for c in ch])
    assert np.array_equal(got[:, :4], Y) and np.array_equal(got[:, 4], U) and np.array_equal(got[:, 5], V)


# ---- crops ------------------------------------------------------------------------------------------------------------

def yuv_layout(fmt, Sw, Sh, pads=(0, 0, 0), offs=(0, 0, 0)):
    """plane (offset, pitch, rows, row bytes) in one sentinel buffer, each plane `offs` bytes after the previous one"""
    rows = [(Sh, Sw), (Sh // 2, Sw)] if fmt == "nv12" else [(Sh, Sw), (Sh // 2, Sw // 2), (Sh // 2, Sw // 2)]
    out, at = [], 0
    for (n, b), pad, off in zip(rows, pads, offs):
        at += off
        out.append((at, b + pad, n, b))
        at += (b + pad) * n
    return out, at + 16


def yuv_crop(lib, e, cw, ch, src, fmt, color, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0, in_color=None, pads=(0, 0, 0),
             offs=(0, 0, 0), tight=False):
    """the host build's YUV crop, of an RGBA8 frame (in_color None) or of a frame of any format -> (rc, buffer)"""
    planes, size = yuv_layout(fmt, Sw, Sh, pads, offs)
    buf = np.full(size, SENTINEL, np.uint8)
    base = buf.ctypes.data
    crop = _lib.FaceCropYuv((C.c_void_p * 3)(*([base + p[0] for p in planes] + [None] * (3 - len(planes)))),
                            (C.c_int32 * 3)(*([0 if tight else p[1] for p in planes] + [0] * (3 - len(planes)))),
                            Sw, Sh, _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color], 0, scale)
    view = view_of(o, rect)
    if in_color is None:
        h, w = src.shape[:2]
        frame = np.ascontiguousarray(src)
        f = _lib.VideoFrame(frame.ctypes.data, 0, w, h, 4 * w, 0.0)
        rc = lib.ht_selftest_face_crop_yuv(C.addressof(e), cw, ch, None, C.addressof(f), C.addressof(view), C.addressof(crop))
    else:
        img = image(src, in_color)
        rc = lib.ht_selftest_face_crop_yuv(C.addressof(e), cw, ch, C.addressof(img), None, C.addressof(view), C.addressof(crop))
    return rc, buf


def convert_into(yo, rgba_buf, rgba_pitch, fmt, color, Sw, Sh, pads=(0, 0, 0), offs=(0, 0, 0)):
    """the restatement's conversion of an RGBA crop buffer into a sentinel buffer of yuv_layout"""
    planes, size = yuv_layout(fmt, Sw, Sh, pads, offs)
    buf = np.full(size, SENTINEL, np.uint8)
    base = buf.ctypes.data
    p = planes + [(0, 0, 0, 0)] * (3 - len(planes))
    yo.hcyo_convert(_lib.YUV_COLORS[color], fmt == "nv12", rgba_buf.ctypes.data, Sw, Sh, rgba_pitch, base + p[0][0],
                    p[0][1], base + p[1][0], p[1][1], base + p[2][0] if fmt == "i420" else None, p[2][1])
    return buf


def check(lib, yo, e, cw, ch, frame, fmt, color, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0, **kw):
    """YUV crop of an RGBA8 frame == the restatement's conversion of the RGBA crop; -> rc"""
    rc, got = yuv_crop(lib, e, cw, ch, frame, fmt, color, o, rect, Sw, Sh, scale, **kw)
    a = lib_crop_rgba(lib, e, cw, ch, frame, o, rect, Sw, Sh, scale)
    assert rc == a[0], (e.x, e.y, e.width, e.height, e.angle, o, rect, Sw, Sh, scale)
    want = convert_into(yo, a[1], a[2], fmt, color, Sw, Sh, kw.get("pads", (0, 0, 0)), kw.get("offs", (0, 0, 0)))
    if not rc:
        want[:] = SENTINEL
    assert np.array_equal(got, want), (e.x, e.y, e.width, e.height, e.angle, o, rect, Sw, Sh, scale, fmt, color)
    return rc


def test_golden_boxes(lib, yo):
    frame = smooth_frame(160, 120, seed=4)
    made = 0
    for i, (x, y, w, h, a) in enumerate(golden_cs_boxes()):
        fmt, color = ("nv12", "i420")[i % 2], COLORS[i % 4]
        made += check(lib, yo, event(2, x, y, w, h, a), 160, 120, frame, fmt, color, Sw=32, Sh=24, scale=1.25)
    assert made > 20


def test_random_rotated_boxes_scales_views(lib, yo):
    rng = np.random.default_rng(23)
    frame = rng.integers(0, 256, (60, 80, 4), dtype=np.uint8)
    angles = [HALF_PI, math.nan, 0.0, -HALF_PI] + list(rng.uniform(-math.pi, math.pi, 6))
    scales = [0.25, 0.6, 1.0, 2.5, 16.0]
    sizes = [(24, 20), (2, 2), (48, 16), (10, 34)]
    n = 0
    for i, a in enumerate(angles):
        scale, (Sw, Sh) = scales[i % len(scales)], sizes[i % len(sizes)]
        e = event(2, float(rng.uniform(10, 150)), float(rng.uniform(10, 110)), float(rng.integers(4, 60)),
                  float(rng.integers(4, 60)), a)
        for o in range(8):
            W, H = (60, 80) if o & 1 else (80, 60)
            for rect in ((0, 0, 0, 0), (W // 5, H // 7, W - W // 3, H - H // 4)):
                n += check(lib, yo, e, 160, 120, frame, ("nv12", "i420")[(i + o) % 2], COLORS[(i + o) % 4], o, rect,
                           Sw, Sh, scale)
    assert n == len(angles) * 16


@pytest.mark.parametrize("fmt_in", ["nv12", "i420"] + NEW)
def test_every_input_format_and_colour(lib, yo, fo, fmt_in):  # noqa: F811
    """a YUV crop of a frame of any format is the conversion of that frame's RGBA crop (itself pinned against the
    crop of the converted RGBA8 frame by tests/test_face_crop_host.py)"""
    rng = np.random.default_rng(len(fmt_in) * 7 + 1)
    for k, color_in in enumerate(colors_of(fmt_in)):
        frame = random_frame(rng, fmt_in, 67, 45, offsets=(2, 6, 4) if fmt_in == "p010" else (1, 3, 2))
        for o, rect in ((0, (0, 0, 0, 0)), (5, (2, 1, 30, 60))):
            e = event(2, float(rng.uniform(10, 70)), float(rng.uniform(10, 50)), float(rng.integers(6, 40)),
                      float(rng.integers(6, 40)), float(rng.uniform(0, math.pi)))
            for fmt in ("nv12", "i420"):
                color = COLORS[(k + o) % 4]
                rc, got = yuv_crop(lib, e, 80, 60, frame, fmt, color, o, rect, 22, 18, 1.2, in_color=color_in)
                a = lib_crop_yuv(lib, e, 80, 60, frame, color_in, o, rect, 22, 18, 1.2)
                assert rc == a[0] == 1
                assert np.array_equal(got, convert_into(yo, a[1], a[2], fmt, color, 22, 18)), (fmt_in, color_in, o, fmt)


def test_odd_pitches_offsets_and_tight_pitches(lib, yo):
    frame = smooth_frame(160, 120, seed=8)
    e = event(2, 70.0, 55.0, 40.0, 50.0, 1.1)
    for fmt in ("nv12", "i420"):
        for pads, offs in (((1, 3, 5), (1, 7, 3)), ((7, 1, 2), (3, 1, 1)), ((0, 0, 0), (0, 0, 0))):
            for color in COLORS:
                assert check(lib, yo, e, 160, 120, frame, fmt, color, Sw=30, Sh=26, pads=pads, offs=offs) == 1
        rc, tight = yuv_crop(lib, e, 160, 120, frame, fmt, "bt709", Sw=30, Sh=26, tight=True)
        assert rc == 1 and np.array_equal(tight, yuv_crop(lib, e, 160, 120, frame, fmt, "bt709", Sw=30, Sh=26)[1])


def test_transparent_pixels_convert_as_black(lib, yo):
    """a box that leaves the video: its transparent pixels (0, 0, 0, 0) become black, and the restatement agrees"""
    frame = np.full((120, 160, 4), 200, np.uint8)
    e = event(2, -30.0, -30.0, 40.0, 40.0, HALF_PI)
    for color in COLORS:
        rc, got = yuv_crop(lib, e, 160, 120, frame, "i420", color, Sw=16, Sh=16)
        assert rc == 1 and check(lib, yo, e, 160, 120, frame, "i420", color, Sw=16, Sh=16)
        assert got[0] == (0 if color.endswith("full") else 16) and got[16 * 16] == 128


def test_records_that_keep_no_face_write_nothing(lib, yo):
    frame = smooth_frame(160, 120)
    for e in (event(1, 50, 50, 30, 30, 0.0), event(2, 50, 50, 0, 30, HALF_PI), event(2, math.nan, 50, 30, 30, HALF_PI)):
        rc, got = yuv_crop(lib, e, 160, 120, frame, "nv12", "bt601", Sw=16, Sh=16)
        assert rc == 0 and (got == SENTINEL).all()


# ---- the kernel and the ABI -------------------------------------------------------------------------------------------

def test_yuv_bodies_do_not_spill(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    names = ["k_face_crop"] + [f"face_crop_yuv_tileILi{k}ELb{b}" for k in range(3) for b in range(2)]
    for name in names:
        m = re.search(r"Function properties for \S*" + name + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", out)
        assert m, (name, out[-2000:])
        assert m.group(2) == m.group(3) == "0", m.group(0)


def test_abi():
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_set_face_crop_yuv") and "ht_tracker_set_face_crop_yuv" in _lib.EXPORTS
    assert L.ht_tracker_set_face_crop_yuv(None, 0, 1, (_lib.FaceCropYuv * 1)()) == _lib.HT_ERR_ARG
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "int ht_tracker_set_face_crop_yuv(ht_ctx *ctx, int first, int n, const ht_face_crop_yuv *crops);" in header
    assert "} ht_face_crop_yuv;       /* 64 bytes */" in header
    offs = {f: getattr(_lib.FaceCropYuv, f).offset for f in ("planes", "pitch", "width", "height", "format", "color",
                                                             "pad_", "scale")}
    assert offs == dict(planes=0, pitch=24, width=36, height=40, format=44, color=48, pad_=52, scale=56)
