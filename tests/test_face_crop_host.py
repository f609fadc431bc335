"""CPU: face crops (DESIGN.md 2, "Face crops") through ht_face_crop_map and the host build of k_face_crop's per-crop
code (ht_selftest_face_crop / ht_selftest_face_crop_rgba), against the independent C restatement tests/crop_oracle.c:

  * the map equals the restatement bit for bit: the CS boxes of reference_js_debug.json and reference_js_main.json,
    random rotated boxes (+-pi/2 and NaN angles included), scales 0.25 to 16, both aspect directions, 1x1 and
    2048-wide crops, every orientation x mirror x source rectangle, canvas up- and downscales;
  * views.crop_to_video puts the crop's centre on views.cs_to_video's centre;
  * the crop equals the restatement bit for bit, a numpy float64 brute force of the continuous definition within one
    level, and a copy of the box on the 1:1 pin;
  * composition: a turned or mirrored video through its view crops exactly like the upright video, a source rectangle
    exactly like the same pixels cut out as a frame, and every format and colour exactly like its converted RGBA8
    frame (tests/format_oracle.c);
  * taps that leave the video or the rectangle read transparent black exactly where they leave; records that keep no
    face write nothing; padded pitches keep their padding;
  * a spill-free k_face_crop, the exported symbols, and ht_face_crop_map's rejections."""
import ctypes as C
import json
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib, views
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_formats_host import NEW, colors_of, fo, image, oracle_convert, random_frame  # noqa: F401
from test_views_host import orient_np, view_of

GOLDEN = Path(__file__).resolve().parent / "golden"
HALF_PI = 1.5707963267948966


@pytest.fixture(scope="module")
def so(tmp_path_factory):
    """tests/crop_oracle.c built into a temporary directory, without contraction"""
    lib = tmp_path_factory.mktemp("crop_oracle") / "libcrop_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("crop_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hco_map.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                          C.c_double, C.c_void_p, C.c_void_p]
    L.hco_crop.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.hco_crop.restype = None
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_face_crop.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_crop_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return st


def event(det, x, y, w, h, angle, conf=1.0):
    e = _lib.TrackerEvent()
    e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle = det, conf, x, y, w, h, angle
    return e


def rect_of(o, w, h, rect):
    W, H = (h, w) if o & 1 else (w, h)
    return tuple(rect) if any(rect) else (0, 0, W, H)


def lib_map(e, cw, ch, w, h, o, rect, Sw, Sh, scale):
    out = (C.c_int64 * 6)()
    crop, view = _lib.FaceCrop(None, Sw, Sh, 0, 0, scale), view_of(o, rect)
    rc = _lib.lib().ht_face_crop_map(C.addressof(e), cw, ch, w, h, C.addressof(view), C.addressof(crop), out)
    return rc, tuple(out)


def oracle_map(so, e, cw, ch, w, h, o, rect, Sw, Sh, scale):
    rec = (C.c_double * 6)(e.detection, e.x, e.y, e.width, e.height, e.angle)
    mr, mv = (C.c_int64 * 6)(), (C.c_int64 * 6)()
    rc = so.hco_map(rec, cw, ch, w, h, o, (C.c_int * 4)(*rect_of(o, w, h, rect)), Sw, Sh, scale, mr, mv)
    return rc, tuple(mr), tuple(mv)


def check_map(so, e, cw, ch, w, h, o=0, rect=(0, 0, 0, 0), Sw=112, Sh=112, scale=1.0):
    got = lib_map(e, cw, ch, w, h, o, rect, Sw, Sh, scale)
    rc, _, mv = oracle_map(so, e, cw, ch, w, h, o, rect, Sw, Sh, scale)
    assert got == (rc, mv if rc else (0,) * 6), (e.x, e.y, e.width, e.height, e.angle, cw, ch, w, h, o, rect, Sw, Sh, scale)
    return rc


def crop_buf(Sw, Sh, pad=0, fill=0xA5):
    pitch = 4 * Sw + pad
    return np.full(Sh * pitch, fill, np.uint8), pitch


def as_image(buf, Sw, Sh, pitch):
    return buf.reshape(Sh, pitch)[:, :4 * Sw].reshape(Sh, Sw, 4)


def lib_crop_rgba(lib, e, cw, ch, frame, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0, pad=0, stored_pad=0):
    """the host build's crop of an RGBA8 frame (h, w, 4) -> (rc, crop buffer, pitch)"""
    h, w = frame.shape[:2]
    src = np.zeros((h, w + stored_pad, 4), np.uint8)
    src[:, :w] = frame
    f = _lib.VideoFrame(src.ctypes.data, 0, w, h, 4 * (w + stored_pad), 0.0)
    buf, pitch = crop_buf(Sw, Sh, pad)
    crop, view = _lib.FaceCrop(buf.ctypes.data, Sw, Sh, pitch, 0, scale), view_of(o, rect)
    rc = lib.ht_selftest_face_crop_rgba(C.addressof(e), cw, ch, C.addressof(f), C.addressof(view), C.addressof(crop))
    return rc, buf, pitch


def lib_crop_yuv(lib, e, cw, ch, frame, color, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0):
    img = image(frame, color)
    buf, pitch = crop_buf(Sw, Sh)
    crop, view = _lib.FaceCrop(buf.ctypes.data, Sw, Sh, pitch, 0, scale), view_of(o, rect)
    rc = lib.ht_selftest_face_crop(C.addressof(e), cw, ch, C.addressof(img), C.addressof(view), C.addressof(crop))
    return rc, buf, pitch


def oracle_crop(so, e, cw, ch, frame, o=0, rect=(0, 0, 0, 0), Sw=24, Sh=20, scale=1.0, pad=0):
    """the restatement's crop: the rectangle cut out of the numpy-oriented frame, sampled through its own map"""
    h, w = frame.shape[:2]
    sx, sy, sw, sh = rect_of(o, w, h, rect)
    R = np.ascontiguousarray(orient_np(frame, o)[sy:sy + sh, sx:sx + sw])
    rc, mr, _ = oracle_map(so, e, cw, ch, w, h, o, rect, Sw, Sh, scale)
    buf, pitch = crop_buf(Sw, Sh, pad)
    if rc:
        so.hco_crop(R.ctypes.data, sw, sh, (C.c_int64 * 6)(*mr), buf.ctypes.data, Sw, Sh, pitch)
    return rc, buf, pitch


def check_crop(lib, so, e, cw, ch, frame, **kw):
    a = lib_crop_rgba(lib, e, cw, ch, frame, **kw)
    b = oracle_crop(so, e, cw, ch, frame, **{k: v for k, v in kw.items() if k != "stored_pad"})
    assert a[0] == b[0] and np.array_equal(a[1], b[1]), (e.x, e.y, e.width, e.height, e.angle, cw, ch, kw)
    return a


# ---- the map ----------------------------------------------------------------------------------------------------------

def golden_cs_boxes():
    """(x, y, w, h, angle) of every green stroke of the debug golden and every CS facetrackingEvent of the main one"""
    out = []
    for case in json.loads((GOLDEN / "reference_js_debug.json").read_text())["cases"]:
        for s in case["steps"]:
            tx = ty = th = None
            for c in s["calls"]:
                if c[0] == "translate":
                    tx, ty = c[1], c[2]
                elif c[0] == "rotate":
                    th = c[1]
                elif c[0] == "strokeRect" and c[1] == "#00CC00":
                    out.append((tx, ty, float(c[4]), float(c[5]), th + HALF_PI))
    for case in json.loads((GOLDEN / "reference_js_main.json").read_text())["cases"]:
        for s in case["steps"]:
            for ev in s.get("events", []):
                if ev.get("type") == "facetrackingEvent" and ev.get("detection") == "CS":
                    out.append((ev["x"], ev["y"], ev["width"], ev["height"], ev["angle"]))
    return out


def test_map_golden_boxes(so):
    boxes = golden_cs_boxes()
    assert len(boxes) > 20 and any(math.isnan(b[4]) for b in boxes) and any(abs(b[4] - HALF_PI) > 1e-3 for b in boxes
                                                                             if not math.isnan(b[4]))
    made = 0
    for i, (x, y, w, h, a) in enumerate(boxes):
        e = event(2, x, y, w, h, a)
        made += check_map(so, e, 160, 120, 160, 120)                                      # ht_tracker_step, 1:1
        made += check_map(so, e, 160, 120, 1280, 720, Sw=112, Sh=112, scale=1.25)          # feed, upscaled video
        made += check_map(so, e, 160, 120, 720, 1280, o=1 + (i % 7), Sw=64, Sh=96)          # a turned video
    assert made == 3 * sum(w > 0 and h > 0 for _, _, w, h, _ in boxes)


def test_map_random_boxes_scales_aspects_views(so):
    rng = np.random.default_rng(7)
    angles = [HALF_PI, -HALF_PI, math.pi, 0.0, math.nan, 1e-12, HALF_PI + 1e-9] + list(rng.uniform(-math.pi, math.pi, 9))
    scales = [0.25, 0.5, 1.0, 1.7, 4.0, 16.0]
    sizes = [(112, 112), (224, 224), (64, 128), (160, 90), (1, 1), (2048, 16), (2048, 2048), (3, 2048)]
    videos = [(640, 480), (1280, 720), (320, 240), (37, 53)]
    canvases = [(320, 240), (160, 120), (1280, 960), (41, 29)]
    n = 0
    for i, a in enumerate(angles):
        for j, scale in enumerate(scales):
            Sw, Sh = sizes[(i + j) % len(sizes)]
            w, h = videos[(i * 3 + j) % len(videos)]
            cw, ch = canvases[(i + 2 * j) % len(canvases)]
            bw, bh = float(rng.integers(1, 90)), float(rng.integers(1, 90))
            x, y = float(rng.uniform(-20, cw + 20)), float(rng.uniform(-20, ch + 20))
            for o in range(8):
                W, H = (h, w) if o & 1 else (w, h)
                for rect in ((0, 0, 0, 0), (W // 5, H // 7, W - W // 3, H - H // 4), (W - 1, 0, 1, H)):
                    n += check_map(so, event(2, x, y, bw, bh, a), cw, ch, w, h, o, rect, Sw, Sh, scale)
    assert n == len(angles) * len(scales) * 24


def test_map_aspect_growth_and_centre(so):
    """the shorter side grows to S_w : S_h about the box's centre; the crop's centre is the stroked box's centre"""
    e = event(2, 100.0, 80.0, 40.0, 60.0, HALF_PI)
    for Sw, Sh in ((40, 60), (80, 60), (40, 120), (1, 1), (2048, 2)):
        rc, (U0, V0, Ui, Vi, Uj, Vj) = lib_map(e, 320, 240, 320, 240, 0, (0, 0, 0, 0), Sw, Sh, 1.0)
        assert rc == 1 and Vi == 0 and Uj == 0 and Ui * Sw >= 40 * 65536 - Sw and Vj * Sh >= 60 * 65536 - Sh
        assert min(abs(Ui * Sw - 40 * 65536), abs(Vj * Sh - 60 * 65536)) <= max(Sw, Sh)   # one side is the box's
        assert abs((U0 + (Sw - 1) / 2 * Ui) / 65536 + 0.5 - 100.0) <= Sw / 65536
        assert abs((V0 + (Sh - 1) / 2 * Vj) / 65536 + 0.5 - 80.0) <= Sh / 65536


def test_crop_to_video_centre(so):
    """views.crop_to_video maps the crop's centre onto cs_to_video's centre: to 1e-9 where the map is exact (even
    boxes, quarter-turn angles, dyadic scales), within the 1/65536-px quantisation of origin and steps otherwise"""
    rng = np.random.default_rng(3)
    for k in range(200):
        o, exact = k % 8, k % 3 == 0
        W, H = (640, 480) if exact else (1280, 720)                   # the oriented frame; exact: dyadic scales
        w, h = (H, W) if o & 1 else (W, H)
        view = {"rotate": 90 * (o & 3), "mirror": bool(o & 4), "crop": None if k % 4 else (W // 4, H // 4, W // 2, H // 2)}
        bw, bh = (2.0 * rng.integers(4, 40), 2.0 * rng.integers(4, 40)) if exact else (float(rng.integers(3, 80)),) * 2
        a = HALF_PI if exact else float(rng.uniform(0, math.pi))
        x, y = (float(rng.integers(0, 320)), float(rng.integers(0, 240))) if exact else (rng.uniform(0, 320), rng.uniform(0, 240))
        Sw, Sh = ((128, 128) if k % 5 else (64, 128)) if exact else ((112, 112) if k % 5 else (96, 128))
        rec = dict(detection="CS", x=x, y=y, width=bw, height=bh, angle=a)
        A = views.crop_to_video(view, w, h, 320, 240, rec, Sw, Sh, 2.0 if exact else 1.3)
        got = (A[0][0] * Sw / 2 + A[0][1] * Sh / 2 + A[0][2], A[1][0] * Sw / 2 + A[1][1] * Sh / 2 + A[1][2])
        # the stroked box's local centre: (ToInt32(-w/2) + w/2, ToInt32(-h/2) + h/2), 0 for even sizes
        lx, ly = math.trunc(-bw / 2) + bw / 2, math.trunc(-bh / 2) + bh / 2
        s, c = math.sin(a - HALF_PI), math.cos(a - HALF_PI)
        want = views.cs_to_video(view, w, h, 320, 240, x + c * lx - s * ly, y + s * lx + c * ly, bw, bh, a)[:2]
        tol = 1e-9 if exact else (1 + (Sw + Sh) / 2) / 65536 * 1.01
        assert abs(got[0] - want[0]) <= tol and abs(got[1] - want[1]) <= tol, (k, got, want)
    assert views.crop_to_video(None, 320, 240, 320, 240, dict(detection="VJ", x=1, y=2, width=30, height=30, angle=0),
                               112, 112) is None


# ---- pixels -----------------------------------------------------------------------------------------------------------

def smooth_frame(w, h, seed=0, alpha=255):
    """an RGBA8 frame whose channels change by at most ~40 levels per pixel, so a brute force in float64 bounds the
    fixed-point map's and 8-bit weights' error by one level"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.empty((h, w, 4), np.uint8)
    for c in range(3):
        fx, fy, ph = rng.uniform(0.02, 0.12), rng.uniform(0.02, 0.12), rng.uniform(0, 6)
        out[..., c] = np.clip(np.round(127.5 + 120 * np.sin(fx * x + ph) * np.cos(fy * y)), 0, 255)
    out[..., 3] = alpha
    return out


def brute_force(e, cw, ch, frame, Sw, Sh, scale):
    """the continuous definition in float64: real sin / cos, real map, real bilinear weights, transparent outside"""
    h, w = frame.shape[:2]
    a = 0.0 if math.isnan(e.angle) else e.angle - HALF_PI
    s, c = math.sin(a), math.cos(a)
    rx, ry = math.trunc(-(e.width / 2)), math.trunc(-(e.height / 2))
    cx, cy = rx + e.width / 2, ry + e.height / 2
    hw, hh = e.width * scale / 2, e.height * scale / 2
    if hw * Sh < hh * Sw:
        hw = hh * Sw / Sh
    else:
        hh = hw * Sh / Sw
    j, i = np.mgrid[0:Sh, 0:Sw].astype(np.float64)
    lx, ly = cx - hw + (i + 0.5) * 2 * hw / Sw, cy - hh + (j + 0.5) * 2 * hh / Sh
    u = (e.x + c * lx - s * ly) * w / cw - 0.5
    v = (e.y + s * lx + c * ly) * h / ch - 0.5
    x0, y0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    fx, fy = u - x0, v - y0
    out = np.zeros((Sh, Sw, 4))
    for dx, dy, wt in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
        X, Y = x0 + dx, y0 + dy
        ok = (X >= 0) & (Y >= 0) & (X < w) & (Y < h)
        out += np.where(ok[..., None], frame[np.clip(Y, 0, h - 1), np.clip(X, 0, w - 1)], 0) * wt[..., None]
    return out


@pytest.mark.parametrize("canvas", [(160, 120), (320, 240), (640, 480)], ids=["up", "1to1", "down"])
def test_crop_equals_restatement_and_brute_force(lib, so, canvas):
    cw, ch = canvas
    frame = smooth_frame(320, 240, seed=cw)
    rng = np.random.default_rng(cw)
    n = 0
    for k in range(24):
        a = [HALF_PI, math.nan, 0.0, math.pi][k] if k < 4 else float(rng.uniform(0, math.pi))
        bw, bh = float(rng.integers(8, cw // 3)), float(rng.integers(8, ch // 3))
        x, y = float(rng.uniform(cw / 3, 2 * cw / 3)), float(rng.uniform(ch / 3, 2 * ch / 3))
        Sw, Sh = [(24, 20), (7, 13), (1, 1), (33, 17), (48, 48), (16, 40)][k % 6]
        scale = [1.0, 0.5, 0.25, 1.5][k % 4]
        e = event(2, x, y, bw, bh, a)
        rc, buf, pitch = check_crop(lib, so, e, cw, ch, frame, Sw=Sw, Sh=Sh, scale=scale, pad=4 * (k % 3))
        assert rc == 1
        got = as_image(buf, Sw, Sh, pitch).astype(np.float64)
        # where the crop leaves the video, alpha steps from 255 to 0 within a pixel: the bound holds on smooth content
        _, mr, _ = oracle_map(so, e, cw, ch, 320, 240, 0, (0, 0, 0, 0), Sw, Sh, scale)
        inside, _ = taps_inside(mr, 320, 240, Sw, Sh)
        assert np.abs(got - brute_force(e, cw, ch, frame, Sw, Sh, scale))[inside].max(initial=0) <= 1.0, k
        n += int(inside.sum())
    assert n > 0.9 * 24 * 24 * 20


@pytest.mark.parametrize("w,h", [(40, 30), (41, 31), (1, 1), (2, 7)])
def test_one_to_one_copy_pin(lib, so, w, h):
    """an unrotated box, scale 1, a crop of the box's own size, on a 1:1 canvas: the box's canvas pixels"""
    rng = np.random.default_rng(w)
    frame = rng.integers(0, 256, (120, 160, 4), dtype=np.uint8)
    for x, y in ((80.0, 60.0), (30.0, 90.0), (150.0, 5.0)):
        rc, buf, pitch = check_crop(lib, so, event(2, x, y, float(w), float(h), HALF_PI), 160, 120, frame, Sw=w, Sh=h)
        rx, ry = int(x) + math.trunc(-w / 2), int(y) + math.trunc(-h / 2)
        want = np.zeros((h, w, 4), np.uint8)
        ys, xs = slice(max(ry, 0), min(ry + h, 120)), slice(max(rx, 0), min(rx + w, 160))
        want[ys.start - ry:ys.stop - ry, xs.start - rx:xs.stop - rx] = frame[ys, xs]
        assert rc == 1 and np.array_equal(as_image(buf, w, h, pitch), want), (x, y)


def stored(upright, o):
    """the video that orientation o turns into `upright`"""
    a = np.fliplr(upright) if o & 4 else upright
    return np.ascontiguousarray(np.rot90(a, o & 3))


def test_turned_video_through_its_view_equals_the_upright_crop(lib, so):
    rng = np.random.default_rng(11)
    V = rng.integers(0, 256, (72, 96, 4), dtype=np.uint8)          # upright 96 x 72
    for k in range(12):
        e = event(2, float(rng.uniform(0, 192)), float(rng.uniform(0, 144)), float(rng.integers(4, 60)),
                  float(rng.integers(4, 60)), float(rng.uniform(0, math.pi)) if k else math.nan)
        Sw, Sh, scale = [(24, 20), (31, 9), (5, 40)][k % 3] + ([1.0, 2.5, 0.75][k % 3],)
        for rect in ((0, 0, 0, 0), (10, 6, 61, 50)):
            want = lib_crop_rgba(lib, e, 192, 144, V, 0, rect, Sw, Sh, scale)
            for o in range(8):
                S = stored(V, o)
                assert np.array_equal(orient_np(S, o), V)
                got = check_crop(lib, so, e, 192, 144, S, o=o, rect=rect, Sw=Sw, Sh=Sh, scale=scale, stored_pad=o % 2)
                assert got[0] == want[0] and np.array_equal(got[1], want[1]), (k, rect, o)
            if any(rect):    # a source rectangle crops exactly like its pixels cut out as a frame of their own
                sx, sy, sw, sh = rect
                cut = lib_crop_rgba(lib, e, 192, 144, np.ascontiguousarray(V[sy:sy + sh, sx:sx + sw]), 0, (0, 0, 0, 0),
                                    Sw, Sh, scale)
                assert np.array_equal(cut[1], want[1])


@pytest.mark.parametrize("fmt", ["nv12", "i420"] + NEW)
def test_every_format_equals_the_crop_of_its_rgba_frame(lib, fo, fmt):  # noqa: F811
    rng = np.random.default_rng(len(fmt) * 13 + 5)
    for color in colors_of(fmt):
        frame = random_frame(rng, fmt, 67, 45, offsets=(2, 6, 4) if fmt == "p010" else (1, 3, 2))
        rgba = oracle_convert(fo, frame, color)
        for o, rect in ((0, (0, 0, 0, 0)), (1, (3, 5, 40, 50)), (6, (0, 0, 0, 0)), (5, (2, 1, 30, 60))):
            e = event(2, float(rng.uniform(10, 70)), float(rng.uniform(10, 50)), float(rng.integers(6, 40)),
                      float(rng.integers(6, 40)), float(rng.uniform(0, math.pi)))
            a = lib_crop_yuv(lib, e, 80, 60, frame, color, o, rect, 23, 19, 1.2)
            b = lib_crop_rgba(lib, e, 80, 60, rgba, o, rect, 23, 19, 1.2)
            assert a[0] == b[0] == 1 and np.array_equal(a[1], b[1]), (fmt, color, o, rect)


# ---- edges ------------------------------------------------------------------------------------------------------------

def taps_inside(m, sw, sh, Sw, Sh):
    """per crop pixel: (every tap with weight > 0 inside the sw x sh rectangle, none of them inside)"""
    U0, V0, Ui, Vi, Uj, Vj = m
    j, i = np.mgrid[0:Sh, 0:Sw].astype(np.int64)
    U, V = U0 + i * Ui + j * Uj, V0 + i * Vi + j * Vj
    x0, y0, fx, fy = U >> 16, V >> 16, (U >> 8) & 255, (V >> 8) & 255
    every, none = np.ones((Sh, Sw), bool), np.ones((Sh, Sw), bool)
    for dx, dy, wt in ((0, 0, (256 - fx) * (256 - fy)), (1, 0, fx * (256 - fy)), (0, 1, (256 - fx) * fy), (1, 1, fx * fy)):
        inside = (x0 + dx >= 0) & (y0 + dy >= 0) & (x0 + dx < sw) & (y0 + dy < sh)
        every &= inside | (wt == 0)
        none &= ~inside | (wt == 0)
    return every, none


def test_boxes_leaving_the_video_fade_to_transparent(lib, so):
    rng = np.random.default_rng(5)
    frame = rng.integers(0, 256, (120, 160, 4), dtype=np.uint8)
    frame[..., 3] = 255
    cases = [(-10.0, 60.0, 40.0, 40.0, HALF_PI), (150.0, 110.0, 50.0, 30.0, 1.0), (80.0, 60.0, 100.0, 100.0, 0.3),
             (-200.0, -200.0, 20.0, 20.0, 2.0), (0.0, 0.0, 10.0, 10.0, HALF_PI), (160.0, 60.0, 30.0, 60.0, math.nan)]
    seen_partial = 0
    for k, (x, y, bw, bh, a) in enumerate(cases):
        for o, rect in ((0, (0, 0, 0, 0)), (0, (20, 10, 100, 90)), (3, (5, 30, 100, 110))):
            e = event(2, x, y, bw, bh, a)
            rc, buf, pitch = check_crop(lib, so, e, 160, 120, frame, o=o, rect=rect, Sw=32, Sh=24, scale=1.5)
            assert rc == 1
            img = as_image(buf, 32, 24, pitch)
            _, mr, _ = oracle_map(so, e, 160, 120, 160, 120, o, rect, 32, 24, 1.5)
            sx, sy, sw, sh = rect_of(o, 160, 120, rect)
            every, none = taps_inside(mr, sw, sh, 32, 24)
            assert (img[every][:, 3] == 255).all() and (img[none] == 0).all()
            assert (img[~every & ~none][:, 3] < 255).all()
            seen_partial += int((~every & ~none).any())
    assert seen_partial >= 6


def test_records_that_keep_no_face_write_nothing(lib, so):
    frame = np.random.default_rng(2).integers(0, 256, (120, 160, 4), dtype=np.uint8)
    for e in (event(1, 50, 50, 30, 30, 0.0), event(2, 50, 50, 0, 30, HALF_PI), event(2, 50, 50, 30, 0, HALF_PI),
              event(2, 50, 50, 0, 0, HALF_PI), event(0, 50, 50, 30, 30, HALF_PI), event(3, 50, 50, 30, 30, HALF_PI),
              event(2, math.nan, 50, 30, 30, HALF_PI), event(2, 50, 50, math.inf, 30, HALF_PI),
              event(2, 70000.0, 50, 30, 30, HALF_PI), event(2, 50, 50, -30, 30, HALF_PI)):
        rc, buf, _ = check_crop(lib, so, e, 160, 120, frame, Sw=16, Sh=16, pad=8)
        assert rc == 0 and (buf == 0xA5).all()
        assert lib_map(e, 160, 120, 160, 120, 0, (0, 0, 0, 0), 16, 16, 1.0) == (0, (0,) * 6)


def test_padded_pitches_keep_their_padding(lib, so):
    frame = np.random.default_rng(9).integers(0, 256, (120, 160, 4), dtype=np.uint8)
    for pad in (4, 12, 64):
        rc, buf, pitch = check_crop(lib, so, event(2, 80, 60, 40, 50, 1.2), 160, 120, frame, Sw=20, Sh=30, pad=pad)
        rows = buf.reshape(30, pitch)
        assert rc == 1 and (rows[:, 80:] == 0xA5).all() and not (rows[:, :80] == 0xA5).all()


# ---- the kernel and the ABI -------------------------------------------------------------------------------------------

def test_face_crop_does_not_spill(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    found = 0
    for name in ("k_face_crop", "face_crop_tileILi0", "face_crop_tileILi1", "face_crop_tileILi2"):
        m = re.search(r"Function properties for \S*" + name + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads", out)
        assert m, (name, out[-2000:])
        assert m.group(2) == m.group(3) == "0", m.group(0)
        found += 1
    assert found == 4


def test_abi_symbols_and_map_rejections():
    L = _lib.lib()
    for s in ("ht_tracker_set_face_crop", "ht_face_crop_map"):
        assert hasattr(L, s) and s in _lib.EXPORTS
    assert L.ht_tracker_set_face_crop(None, 0, 1, (_lib.FaceCrop * 1)()) == _lib.HT_ERR_ARG
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "int ht_tracker_set_face_crop(ht_ctx *ctx, int first, int n, const ht_face_crop *crops);" in header
    assert "} ht_face_crop;           /* 32 bytes */" in header
    e = event(2, 80, 60, 40, 40, HALF_PI)
    out = (C.c_int64 * 6)()
    whole = view_of(0)

    def call(ev=e, cw=160, ch=120, w=160, h=120, view=whole, Sw=16, Sh=16, scale=1.0, o=out):
        crop = _lib.FaceCrop(None, Sw, Sh, 0, 0, scale)
        return L.ht_face_crop_map(C.addressof(ev) if ev is not None else None, cw, ch, w, h,
                                  C.addressof(view) if view is not None else None, C.addressof(crop), o)
    assert call() == 1 and call(view=None) == 1
    assert call(ev=None) == call(o=None) == _lib.HT_ERR_ARG
    for bad in (dict(cw=0), dict(ch=16385), dict(w=0), dict(h=20000), dict(Sw=0), dict(Sh=2049)):
        assert call(**bad) == _lib.HT_ERR_SIZE, bad
    for scale in (0.0, -1.0, 16.5, math.nan, math.inf):
        assert call(scale=scale) == _lib.HT_ERR_ARG, scale
    assert call(scale=16.0) == 1
    for v in (view_of(8), view_of(0, (0, 0, 161, 120)), view_of(0, (0, 0, 0, 0), (1, 0, 0)), view_of(1, (0, 0, 160, 120))):
        assert call(view=v) == _lib.HT_ERR_ARG
