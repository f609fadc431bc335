"""CPU: a stream's framing (DESIGN.md 2, "Face crops", item 7) through the host build of framing_step
(ht_selftest_framing_step), headtrackr_b200.framing and the independent C restatement tests/framing_oracle.c:

  * the three agree bit for bit, box after box, over the CS sequences of every golden and over random sequences with
    snaps, canvas-size changes, boundary values of alpha and dead_zone, and errors exactly at the band and at w / 2;
  * alpha 1 and dead zone 0 give the tracked crop bit for bit on calcAngles-off records;
  * targets inside the dead zone never move the box; a constant target is approached monotonically and ends within
    the band;
  * on reference_js_main.json's "default" case the framed centre stays put while the raw centre moves on every tick;
  * ht_face_crop_map_framed and the host-built framed crop equal the restatement's map and crop_oracle.c's sampling;
  * the fifth span kind of the overlap rule, the ABI's sizes and offsets, its rejections, and a spill-free
    k_face_crop at no more than 64 registers."""
import ctypes as C
import itertools
import json
import math
import random
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib, framing, views
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_face_crop_host import golden_cs_boxes, lib_crop_rgba, smooth_frame
from test_output_overlap_host import brute as brute_spans
from test_output_overlap_host import random_stream, spans
from test_views_host import orient_np, view_of

GOLDEN = Path(__file__).resolve().parent / "golden"
HALF_PI = 1.5707963267948966
FRAMING = 4                                  # the overlap rule's kind of a framed box


@pytest.fixture(scope="module")
def fo(tmp_path_factory):
    """tests/framing_oracle.c built into a temporary directory, without contraction"""
    lib = tmp_path_factory.mktemp("framing_oracle") / "libframing_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("framing_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hfo_step.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_int]
    L.hfo_map.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                          C.c_double, C.c_void_p, C.c_void_p]
    L.hco_crop.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.hco_crop.restype = None
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_framing_step.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_int]
    st.ht_selftest_face_crop_framed_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_face_crop_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_tick_writes_framed.argtypes = [C.c_int] + [C.c_void_p] * 7
    return st


def event(det, x, y, w, h, angle):
    e = _lib.TrackerEvent()
    e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle = det, 1.0, x, y, w, h, angle
    return e


def rec(det, x, y, w, h, angle):
    return dict(detection=det, x=x, y=y, width=w, height=h, angle=angle)


class Three:
    """one framing run three ways: the library's host build, framing.py and the C restatement"""

    def __init__(self, lib, fo, alpha, dead_zone):
        self.lib, self.fo, self.alpha, self.dz = lib, fo, alpha, dead_zone
        self.lb, self.py, self.ob = _lib.FramedBox(), framing.new_box(), (C.c_char * 48)()

    def step(self, r, cw, ch):
        e = event(r["detection"], r["x"], r["y"], r["width"], r["height"], r["angle"])
        a = self.lib.ht_selftest_framing_step(C.addressof(self.lb), self.alpha, self.dz, C.addressof(e), cw, ch)
        b = framing.framing_step(self.py, r, cw, ch, self.alpha, self.dz)
        c = self.fo.hfo_step(self.ob, self.alpha, self.dz,
                             (C.c_double * 6)(r["detection"], r["x"], r["y"], r["width"], r["height"], r["angle"]), cw, ch)
        assert a == int(b) == c, (r, a, b, c)
        lb = bytes(self.lb)
        assert lb == framing.box_to_bytes(self.py) == bytes(self.ob), (r, framing.box_from_bytes(lb), self.py)
        return a

    @property
    def box(self):
        return dict(self.py)


def golden_sequences():
    """every golden's ordered tracker-record-like dicts with an angle (the CS events, per case), and the debug golden's
    green strokes as CS records"""
    seqs = []

    def walk(v, out):
        if isinstance(v, dict):
            if {"x", "y", "width", "height", "angle"} <= v.keys() and v.get("detection") in ("CS", "VJ", 1, 2):
                d = v["detection"]
                out.append(rec({"VJ": 1, "CS": 2}.get(d, d), *(float(v[k]) for k in ("x", "y", "width", "height", "angle"))))
            for x in v.values():
                walk(x, out)
        elif isinstance(v, list):
            for x in v:
                walk(x, out)
    for p in sorted(GOLDEN.glob("*.json")):
        doc = json.loads(p.read_text())
        for case in doc.get("cases", [doc]) if isinstance(doc, dict) else [doc]:
            out = []
            walk(case, out)
            if any(r["detection"] == 2 for r in out):
                seqs.append((p.name, out))
    seqs.append(("debug strokes", [rec(2, x, y, w, h, a) for x, y, w, h, a in golden_cs_boxes()]))
    return seqs


# ---- the update -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("alpha,dead_zone", [(0.25, 0.1), (1.0, 0.0), (1.0, 0.5), (1e-9, 0.0), (0.7, 0.5), (0.5, 0.25)])
def test_golden_sequences_agree(lib, fo, alpha, dead_zone):
    seqs = golden_sequences()
    assert len(seqs) >= 3 and sum(len(s) for _, s in seqs) > 100
    ticks = 0
    for name, seq in seqs:
        t = Three(lib, fo, alpha, dead_zone)
        for r in seq:
            ticks += t.step(r, 320, 240)
    assert ticks > 80


def test_random_sequences_agree(lib, fo):
    rng = np.random.default_rng(18)
    kinds = dict(snap=0, glide=0, still=0, band=0, half=0, canvas=0, other=0)
    for run in range(300):
        alpha = [1.0, 0.25, 1e-300, 2.0 ** -52, float(rng.uniform(0.01, 1.0)), 0.5][run % 6]
        dz = [0.0, 0.5, 0.1, 0.125, float(rng.uniform(0, 0.5)), 0.25][(run // 6) % 6]
        t = Three(lib, fo, alpha, dz)
        canvas = (320, 240)
        x, y, w, h = 160.0, 120.0, 32.0, 32.0
        for k in range(40):
            u = rng.random()
            b = t.box
            if u < 0.05:
                canvas = [(320, 240), (160, 120), (640, 480), (320, 180)][int(rng.integers(0, 4))]
                kinds["canvas"] += 1
            if u < 0.1:                                                 # something that is not a crop tick
                r = [rec(1, x, y, w, h, 0.0), rec(2, x, y, 0.0, h, HALF_PI), rec(3, x, y, w, h, HALF_PI),
                     rec(2, 70000.0, y, w, h, HALF_PI), rec(2, x, y, -w, h, HALF_PI)][int(rng.integers(0, 5))]
                kinds["other"] += 1
            elif u < 0.2 and b["valid"]:                               # an error exactly at the band (dyadic values)
                r = rec(2, b["cx"] + dz * b["width"], b["cy"] - dz * b["height"], b["width"], b["height"], HALF_PI)
                kinds["band"] += 1
            elif u < 0.3 and b["valid"]:                               # exactly at w / 2, and just past it
                sgn = 1.0 if rng.random() < 0.5 else -1.0
                r = rec(2, b["cx"] + sgn * b["width"] / 2 + (0.0 if rng.random() < 0.5 else 1e-9), b["cy"],
                        b["width"], b["height"], HALF_PI)
                kinds["half"] += 1
            else:
                if rng.random() < 0.1:                                  # a jump: lost and refound elsewhere
                    x, y = float(rng.uniform(0, canvas[0])), float(rng.uniform(0, canvas[1]))
                step = float(rng.choice([0.5, 1.0, 2.0, 4.0]))
                x += float(rng.integers(-3, 4)) * step
                y += float(rng.integers(-3, 4)) * step
                w = float(max(4, w + 4 * int(rng.integers(-1, 2)))) if rng.random() < 0.7 else float(rng.uniform(3, 90))
                h = w if rng.random() < 0.8 else float(rng.integers(3, 90))
                a = HALF_PI if rng.random() < 0.6 else (math.nan if rng.random() < 0.1 else float(rng.uniform(0, math.pi)))
                r = rec(2, x, y, w, h, a)
            before = t.box
            if t.step(r, *canvas):
                after = t.box
                moved = before["valid"] and (after["cx"], after["cy"], after["width"], after["height"]) != \
                    (before["cx"], before["cy"], before["width"], before["height"])
                snapped = after["width"] == r["width"] and after["height"] == r["height"] and not before["valid"]
                kinds["snap" if snapped else "glide" if moved else "still"] += 1
    assert min(kinds.values()) > 20, kinds


def test_alpha_one_dead_zone_zero_is_the_tracked_crop(lib):
    """calcAngles-off records (angle pi/2, sizes in steps of 4, integer centres): the framed box is the record's box and
    the framed map and crop are the tracked ones, bit for bit"""
    rng = np.random.default_rng(4)
    frame = smooth_frame(320, 240, seed=4)
    box = _lib.FramedBox()
    n = 0
    for k in range(60):
        x, y = float(rng.integers(-10, 330)), float(rng.integers(-10, 250))
        w, h = 4.0 * rng.integers(1, 20), 4.0 * rng.integers(1, 20)
        e = event(2, x, y, w, h, HALF_PI)
        assert lib.ht_selftest_framing_step(C.addressof(box), 1.0, 0.0, C.addressof(e), 320, 240) == 1
        assert (box.cx, box.cy, box.width, box.height) == (x, y, w, h)
        Sw, Sh, scale = [(112, 112), (64, 96), (33, 17)][k % 3] + ([1.0, 1.5, 0.75][k % 3],)
        for vw, vh, o in ((320, 240, 0), (1280, 720, 0), (720, 1280, 1)):
            tracked = views.crop_map(None if o == 0 else {"rotate": 90}, vw, vh, 320, 240,
                                     dict(detection="CS", x=x, y=y, width=w, height=h, angle=HALF_PI), Sw, Sh, scale)
            framed = views.crop_map(None if o == 0 else {"rotate": 90}, vw, vh, 320, 240, box, Sw, Sh, scale)
            assert framed == tracked, (k, vw, vh)
        a = lib_crop_rgba(lib, e, 320, 240, frame, Sw=Sw, Sh=Sh, scale=scale)
        b = framed_crop(lib, box, 320, 240, frame, Sw, Sh, scale)
        assert a[0] == b[0] == 1 and np.array_equal(a[1], b[1])
        n += 1
    assert n == 60


def test_targets_inside_the_dead_zone_never_move_the_box(lib, fo):
    rng = np.random.default_rng(9)
    for dz in (0.1, 0.25, 0.5):
        t = Three(lib, fo, 0.3, dz)
        t.step(rec(2, 100.0, 80.0, 40.0, 48.0, HALF_PI), 320, 240)
        b0 = t.box
        for k in range(200):
            bx, by = dz * b0["width"], dz * b0["height"]
            r = rec(2, b0["cx"] + float(rng.uniform(-bx, bx)), b0["cy"] + float(rng.uniform(-by, by)),
                    b0["width"] + float(rng.uniform(-bx, bx)), b0["height"] + float(rng.uniform(-by, by)), HALF_PI)
            r["x"] -= math.trunc(-(r["width"] / 2)) + r["width"] * 0.5      # the target's centre stays at r's x, y
            r["y"] -= math.trunc(-(r["height"] / 2)) + r["height"] * 0.5
            tx, ty, tw, th = framing.target(r)
            if abs(tx - b0["cx"]) > bx or abs(ty - b0["cy"]) > by or abs(tw - b0["width"]) > bx or abs(th - b0["height"]) > by:
                continue
            assert t.step(r, 320, 240) == 1
            b = t.box
            assert (b["cx"], b["cy"], b["width"], b["height"]) == (b0["cx"], b0["cy"], b0["width"], b0["height"])
        assert t.box["updates"] > 150


def test_a_constant_target_is_approached_monotonically(lib, fo):
    for alpha, dz in ((0.25, 0.1), (0.05, 0.02), (0.5, 0.3), (1.0, 0.1)):
        t = Three(lib, fo, alpha, dz)
        t.step(rec(2, 100.0, 100.0, 40.0, 40.0, HALF_PI), 320, 240)
        goal = rec(2, 115.0, 88.0, 60.0, 24.0, HALF_PI)         # inside the box: a glide, not a snap
        tx, ty, tw, th = framing.target(goal)
        prev = t.box
        for k in range(1000):
            t.step(goal, 320, 240)
            b = t.box
            for key, tv in (("cx", tx), ("cy", ty), ("width", tw), ("height", th)):
                assert abs(tv - b[key]) <= abs(tv - prev[key]), (alpha, dz, key, k)
                assert (tv - b[key]) * (tv - prev[key]) >= 0, (alpha, dz, key, k)       # never overshoots
            prev = b
        assert b["valid"] and b["updates"] == 1001
        for key, tv, s in (("cx", tx, "width"), ("cy", ty, "height"), ("width", tw, "width"), ("height", th, "height")):
            assert abs(tv - b[key]) <= dz * b[s] * (1 + 1e-9) + 1e-9, (alpha, dz, key)


def test_main_golden_default_holds_the_centre_still():
    case = next(c for c in json.loads((GOLDEN / "reference_js_main.json").read_text())["cases"] if c["name"] == "default")
    box = framing.new_box()
    raw, framed, sizes = [], [], []
    for s in case["steps"]:
        for ev in s.get("events", []):
            if ev.get("type") != "facetrackingEvent":
                continue
            r = dict(ev, detection=ev["detection"])
            if framing.framing_step(box, r, 320, 240, 0.25, 0.1):
                raw.append(framing.target(r)[:2])
                framed.append((box["cx"], box["cy"]))
                sizes.append((box["width"], box["height"]))
    assert len(framed) == 22 and set(framed) == {(130.0, 49.0)}
    moves = [abs(a[0] - b[0]) + abs(a[1] - b[1]) for a, b in zip(raw[1:11], raw[2:12])]
    assert len(moves) == 10 and all(1 <= m <= 4 for m in moves), moves        # the raw centre moves on every tick
    assert sizes[0] == (32.0, 32.0) and round(sizes[-1][0], 2) == 32.73 and sizes[-1][0] == sizes[-1][1]
    assert all(b >= a for a, b in zip(sizes, sizes[1:]))


# ---- the map and the crop ---------------------------------------------------------------------------------------------

def rect_of(o, w, h, rect):
    W, H = (h, w) if o & 1 else (w, h)
    return tuple(rect) if any(rect) else (0, 0, W, H)


def framed_crop(lib, box, cw, ch, frame, Sw, Sh, scale, o=0, rect=(0, 0, 0, 0)):
    h, w = frame.shape[:2]
    src = np.ascontiguousarray(frame)
    f = _lib.VideoFrame(src.ctypes.data, 0, w, h, 4 * w, 0.0)
    buf = np.full(Sh * 4 * Sw, 0xA5, np.uint8)
    crop = _lib.FaceCrop(buf.ctypes.data, Sw, Sh, 4 * Sw, 0, scale)
    view = view_of(o, rect)
    rc = lib.ht_selftest_face_crop_framed_rgba(C.addressof(box), cw, ch, C.addressof(f), C.addressof(view),
                                               C.addressof(crop))
    return rc, buf


def random_box(rng, cw, ch):
    return _lib.FramedBox(float(rng.uniform(-20, cw + 20)), float(rng.uniform(-20, ch + 20)), float(rng.uniform(2, 90)),
                          float(rng.uniform(2, 90)), cw, ch, int(rng.integers(1, 100)), 1)


def test_map_framed_equals_the_restatement(fo):
    rng = np.random.default_rng(21)
    L = _lib.lib()
    n = 0
    for k in range(120):
        cw, ch = [(320, 240), (160, 120), (41, 29)][k % 3]
        w, h = [(640, 480), (1280, 720), (37, 53)][(k // 3) % 3]
        box = random_box(rng, cw, ch)
        Sw, Sh = [(112, 112), (64, 128), (1, 1), (2048, 16)][k % 4]
        scale = [0.25, 1.0, 1.7, 16.0][(k // 4) % 4]
        for o in range(8):
            W, H = (h, w) if o & 1 else (w, h)
            for rect in ((0, 0, 0, 0), (W // 5, H // 7, W - W // 3, H - H // 4)):
                out = (C.c_int64 * 6)()
                crop, view = _lib.FaceCrop(None, Sw, Sh, 0, 0, scale), view_of(o, rect)
                rc = L.ht_face_crop_map_framed(C.addressof(box), cw, ch, w, h, C.addressof(view), C.addressof(crop), out)
                mr, mv = (C.c_int64 * 6)(), (C.c_int64 * 6)()
                want = fo.hfo_map(C.addressof(box), cw, ch, w, h, o, (C.c_int * 4)(*rect_of(o, w, h, rect)), Sw, Sh,
                                  scale, mr, mv)
                assert (rc, tuple(out)) == (want, tuple(mv)) and rc == 1, (k, o, rect)
                n += 1
    assert n == 120 * 16


def test_framed_crop_equals_the_restatement(lib, fo):
    rng = np.random.default_rng(12)
    frame = smooth_frame(320, 240, seed=12)
    for k in range(30):
        cw, ch = [(160, 120), (320, 240), (640, 480)][k % 3]
        box = random_box(rng, cw, ch)
        Sw, Sh, scale = [(24, 20), (7, 13), (1, 1), (33, 17), (48, 48)][k % 5] + ([1.0, 0.5, 1.5][k % 3],)
        for o, rect in ((0, (0, 0, 0, 0)), (3, (5, 30, 200, 250)), (4, (20, 10, 100, 90))):
            rc, buf = framed_crop(lib, box, cw, ch, frame, Sw, Sh, scale, o, rect)
            h, w = frame.shape[:2]
            sx, sy, sw, sh = rect_of(o, w, h, rect)
            R = np.ascontiguousarray(orient_np(frame, o)[sy:sy + sh, sx:sx + sw])
            mr, mv = (C.c_int64 * 6)(), (C.c_int64 * 6)()
            assert fo.hfo_map(C.addressof(box), cw, ch, w, h, o, (C.c_int * 4)(sx, sy, sw, sh), Sw, Sh, scale, mr, mv) == 1
            want = np.full(Sh * 4 * Sw, 0xA5, np.uint8)
            fo.hco_crop(R.ctypes.data, sw, sh, mr, want.ctypes.data, Sw, Sh, 4 * Sw)
            assert rc == 1 and np.array_equal(buf, want), (k, o, rect)


def test_invalid_boxes_make_no_crop(lib, fo):
    frame = smooth_frame(64, 48, seed=1)
    L = _lib.lib()
    for box in (_lib.FramedBox(), _lib.FramedBox(30.0, 20.0, 10.0, 10.0, 64, 48, 3, 0),
                _lib.FramedBox(math.nan, 20.0, 10.0, 10.0, 64, 48, 3, 1), _lib.FramedBox(30.0, 20.0, 1e6, 10.0, 64, 48, 3, 1)):
        rc, buf = framed_crop(lib, box, 64, 48, frame, 8, 8, 1.0)
        assert rc == 0 and (buf == 0xA5).all()
        out = (C.c_int64 * 6)(*range(1, 7))
        crop = _lib.FaceCrop(None, 8, 8, 0, 0, 1.0)
        assert L.ht_face_crop_map_framed(C.addressof(box), 64, 48, 64, 48, None, C.addressof(crop), out) == 0
        assert tuple(out) == (0,) * 6
        assert views.crop_map(None, 64, 48, 64, 48, box, 8, 8) is None


def test_map_framed_rejections():
    L = _lib.lib()
    box = _lib.FramedBox(30.0, 20.0, 10.0, 10.0, 64, 48, 3, 1)
    out = (C.c_int64 * 6)()

    def call(b=box, cw=64, ch=48, w=64, h=48, view=None, Sw=8, Sh=8, scale=1.0, o=out):
        crop = _lib.FaceCrop(None, Sw, Sh, 0, 0, scale)
        return L.ht_face_crop_map_framed(C.addressof(b) if b is not None else None, cw, ch, w, h,
                                         C.addressof(view) if view is not None else None, C.addressof(crop), o)
    assert call() == 1
    assert call(b=None) == call(o=None) == _lib.HT_ERR_ARG
    for bad in (dict(cw=0), dict(ch=16385), dict(w=0), dict(h=20000), dict(Sw=0), dict(Sh=2049)):
        assert call(**bad) == _lib.HT_ERR_SIZE, bad
    for scale in (0.0, -1.0, 16.5, math.nan):
        assert call(scale=scale) == _lib.HT_ERR_ARG
    assert call(view=view_of(8)) == _lib.HT_ERR_ARG


def test_crop_to_video_of_a_framed_box_is_upright_about_its_centre():
    box = dict(cx=100.25, cy=80.5, width=40.5, height=30.0, canvas_w=320, canvas_h=240, updates=5, valid=1)
    A = views.crop_to_video(None, 320, 240, 320, 240, box, 64, 64, 1.0)
    assert A[0][1] == 0 and A[1][0] == 0
    cx, cy = A[0][0] * 32 + A[0][2], A[1][1] * 32 + A[1][2]
    assert abs(cx - 100.25) <= 65 / 65536 and abs(cy - 80.5) <= 65 / 65536


# ---- the overlap rule, the ABI, the kernel ----------------------------------------------------------------------------

def verdict(lib, streams):
    n = len(streams)
    dbg, crops, yuv = (_lib.DebugCanvas * n)(), (_lib.FaceCrop * n)(), (_lib.FaceCropYuv * n)()
    tensors, cams, boxes, clash = (_lib.FaceTensor * n)(), (C.c_void_p * n)(), (C.c_void_p * n)(), (C.c_int32 * 4)()
    for s, x in enumerate(streams):
        for arr, key in ((dbg, "debug"), (crops, "crop"), (yuv, "yuv"), (tensors, "tensor")):
            if x.get(key):
                arr[s] = x[key]
        cams[s] = x.get("camera")
        boxes[s] = x.get("box")
    hit = lib.ht_selftest_tick_writes_framed(n, dbg, crops, yuv, tensors, cams, boxes, clash)
    return hit, ((clash[0], clash[1]), (clash[2], clash[3]))


def brute(streams):
    flat = [(k, s, set(range(a, b))) for s, x in enumerate(streams) for k, a, b in
            spans(x) + ([(FRAMING, x["box"], x["box"] + _lib.FRAMED_BOX_BYTES)] if x.get("box") else [])]
    return [((k0, s0), (k1, s1)) for (k0, s0, b0), (k1, s1, b1) in itertools.combinations(flat, 2) if b0 & b1]


def test_framed_boxes_in_the_overlap_rule(lib):
    rng = random.Random(48)
    kinds, verdicts = set(), [0, 0]
    for trial in range(2000):
        space = rng.choice([1024, 4096])
        streams = [random_stream(rng, space) for _ in range(rng.randint(1, 4))]
        for x in streams:
            if rng.random() < 0.5:
                x["box"] = rng.randrange(64, space, 8)
        hit, pair = verdict(lib, streams)
        pairs = brute(streams)
        assert hit == (len(pairs) > 0), (hit, pairs)
        if hit:
            assert pair in pairs or pair[::-1] in pairs
        verdicts[hit] += 1
        kinds |= {tuple(sorted((a[0], b[0]))) for a, b in pairs if FRAMING in (a[0], b[0])}
    assert kinds == {(k, FRAMING) for k in range(5)}, kinds
    assert min(verdicts) > 200, verdicts
    base = 1 << 20
    assert verdict(lib, [{"box": base}, {"box": base + 48}])[0] == 0
    assert verdict(lib, [{"box": base}, {"box": base + 40}])[0] == 1
    assert verdict(lib, [{"camera": base}, {"box": base + 224}])[0] == 0
    assert verdict(lib, [{"camera": base}, {"box": base + 216}])[1] in (((3, 0), (FRAMING, 1)), ((FRAMING, 1), (3, 0)))
    # the rule without boxes is the one the other setters had
    assert brute_spans([{"camera": base}, {"camera": base + 100}])


def test_abi_layout_and_rejections(lib):
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "int ht_tracker_set_framing(ht_ctx *ctx, int first, int n, const ht_framing *framings);" in header
    assert "} ht_framed_box;          /* 48 bytes */" in header and "} ht_framing;             /* 32 bytes */" in header
    assert "#define HT_FRAMED_BOX_BYTES 48\n" in header
    assert "#define HT_FRAMING_CROP 1 " in header and "#define HT_FRAMING_TENSOR 2 " in header
    assert (_lib.HT_FRAMING_CROP, _lib.HT_FRAMING_TENSOR) == (1, 2)
    assert [getattr(_lib.FramedBox, f).offset for f in ("cx", "cy", "width", "height", "canvas_w", "canvas_h", "updates",
                                                        "valid")] == [0, 8, 16, 24, 32, 36, 40, 44]
    assert [getattr(_lib.Framing, f).offset for f in ("box", "alpha", "dead_zone", "outputs", "pad_")] == [0, 8, 16, 24, 28]
    assert C.sizeof(_lib.FramedBox) == 48 and C.sizeof(_lib.Framing) == 32
    L = _lib.lib()
    for s in ("ht_tracker_set_framing", "ht_face_crop_map_framed"):
        assert hasattr(L, s) and s in _lib.EXPORTS
    assert L.ht_tracker_set_framing(None, 0, 1, (_lib.Framing * 1)()) == _lib.HT_ERR_ARG
    box, e = _lib.FramedBox(), event(2, 50.0, 50.0, 20.0, 20.0, HALF_PI)
    for alpha, dz in ((0.0, 0.1), (-0.1, 0.1), (1.0 + 2 ** -52, 0.1), (math.nan, 0.1), (0.5, -1e-300), (0.5, 0.5 + 2 ** -53),
                      (0.5, math.nan), (math.inf, 0.0), (0.5, math.inf)):
        assert lib.ht_selftest_framing_step(C.addressof(box), alpha, dz, C.addressof(e), 100, 100) == -1, (alpha, dz)
    assert bytes(box) == bytes(48)
    for alpha, dz in ((1.0, 0.0), (5e-324, 0.5)):
        assert lib.ht_selftest_framing_step(C.addressof(box), alpha, dz, C.addressof(e), 100, 100) == 1


def test_face_crop_stays_at_64_registers_without_spills(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    for name in ("k_face_crop", "k_framing_update", "k_framing_reset"):
        m = re.search(r"Function properties for \S*" + name + r"\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                      r"stores, (\d+) bytes spill loads\nptxas info\s*: Used (\d+) registers", out)
        assert m, (name, out[-2000:])
        assert m.group(2) == m.group(3) == "0", m.group(0)
        if name == "k_face_crop":
            assert int(m.group(4)) <= 64, m.group(0)
