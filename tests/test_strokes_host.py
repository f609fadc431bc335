"""CPU: main.js's strokes on the debug canvas (src/main.js:199-219) as DESIGN.md 2, "Strokes" defines them, through
the host build of k_debug_strokes's per-stream code (ht_selftest_debug_strokes, span walk included):

  * stroke_sincos equals, bit for bit, the C restatement tests/stroke_oracle.c, and is within 2 ulp of math.sin /
    math.cos on [-pi/2, pi/2], at 0 and at every rotation of reference_js_debug.json;
  * every stroke equals the C restatement (brute force over the bounding box) and a numpy brute force over every
    sample of every canvas pixel, so pixels the span walk skips have no coverage: aligned rectangles with the 128 / 64
    / 191 pins, the golden's fractional VJ boxes, rotated CS boxes (+-pi/2 and NaN included), sizes 0 / 1 / 2, lines,
    strokes partly or wholly off the canvas, 1x1 canvases, padded pitches, opaque / transparent / half-transparent
    destinations;
  * every case of reference_js_debug.json in lockstep: the oracle's back-projection composite, then the strokes of
    the tick's record (library) and of its debug_calls (restatement);
  * a spill-free k_debug_strokes, the exported symbol, and every rejection of ht_tracker_set_debug_strokes."""
import ctypes as C
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib
from headtrackr_b200.streams import debug_calls
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_debug_host import GOLD_D, composite, debug_canvas, replay

DET = {"VJ": 1, "CS": 2}


@pytest.fixture(scope="module")
def so(tmp_path_factory):
    """tests/stroke_oracle.c built into a temporary directory, without contraction"""
    lib = tmp_path_factory.mktemp("stroke_oracle") / "libstroke_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("stroke_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hso_sincos.argtypes = [C.c_double, C.c_void_p, C.c_void_p]
    L.hso_sincos.restype = None
    L.hso_rect_corners.argtypes = [C.c_double] * 7 + [C.c_void_p]
    L.hso_stroke_rect.argtypes = [C.c_double] * 7 + [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.hso_stroke.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_stroke_sincos.argtypes = [C.c_double, C.c_void_p]
    st.ht_selftest_stroke_sincos.restype = None
    st.ht_selftest_debug_strokes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    return st


def lib_sincos(lib, t):
    out = (C.c_double * 2)()
    lib.ht_selftest_stroke_sincos(t, out)
    return out[0], out[1]


def oracle_sincos(so, t):
    s, c = C.c_double(), C.c_double()
    so.hso_sincos(t, C.byref(s), C.byref(c))
    return s.value, c.value


def event(det, conf, x, y, w, h, angle):
    e = _lib.TrackerEvent()
    e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle = det, conf, x, y, w, h, angle
    return e


def canvas(dw, dh, pad=0, fill="zero", seed=0):
    """(buffer, (dh, dw, 4) view) of a dw x dh canvas with rows of 4 * dw + pad bytes"""
    pitch = 4 * dw + pad
    rng = np.random.default_rng(seed)
    buf = np.zeros(dh * pitch, np.uint8)
    if fill == "random":
        buf[:] = rng.integers(0, 256, buf.size, dtype=np.uint8)
    elif fill == "opaque":
        buf[:] = rng.integers(0, 256, buf.size, dtype=np.uint8)
        buf.reshape(dh, pitch)[:, 3:4 * dw:4] = 255
    elif fill == "half":
        buf[:] = rng.integers(0, 256, buf.size, dtype=np.uint8)
        buf.reshape(dh, pitch)[:, 3:4 * dw:4] = 128
    return buf, pitch


def lib_stroke(lib, e, buf, dw, dh, pitch):
    return lib.ht_selftest_debug_strokes(C.byref(e), buf.ctypes.data, dw, dh, pitch)


def oracle_stroke(so, e, buf, dw, dh, pitch):
    rec = (C.c_double * 7)(e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle)
    return so.hso_stroke(rec, buf.ctypes.data, dw, dh, pitch)


def oracle_calls(so, calls, buf, dw, dh, pitch):
    """the restatement of one tick's debug_calls"""
    tx = ty = theta = 0.0
    for c in calls:
        if c[0] == "translate":
            tx, ty = c[1], c[2]
        elif c[0] == "rotate":
            theta = c[1]
        else:
            _, color, x, y, w, h = c
            so.hso_stroke_rect(tx, ty, theta, x, y, w, h, int(color == "#00CC00"), buf.ctypes.data, dw, dh, pitch)
            return


# ---- numpy brute force ----------------------------------------------------------------------------------------------

def np_corners(so, e):
    """-> list of (4, 2) int64 corner arrays (outer, inner), numpy fp64 with stroke_oracle's sin / cos"""
    if e.confidence == 0 or e.detection not in (1, 2):
        return []
    x, y, w, h = e.x, e.y, e.width, e.height
    if not all(math.isfinite(v) and abs(v) <= 65536 for v in (x, y, w, h)):
        return []
    tx = ty = np.float64(0)
    s, c = np.float64(0), np.float64(1)
    if e.detection == 2:
        tx, ty = np.float64(x), np.float64(y)
        s, c = map(np.float64, oracle_sincos(so, e.angle - math.pi / 2))
        x, y = float(math.trunc(-(w / 2))), float(math.trunc(-(h / 2)))
    x, y, w, h = map(np.float64, (x, y, w, h))
    if w < 0:
        x, w = x + w, -w
    if h < 0:
        y, h = y + h, -h
    if w == 0 and h == 0:
        return []
    if h == 0:
        rects = [(x, y - 0.5, x + w, y + 0.5)]
    elif w == 0:
        rects = [(x - 0.5, y, x + 0.5, y + h)]
    else:
        rects = [(x - 0.5, y - 0.5, (x + w) + 0.5, (y + h) + 0.5)]
        if w > 1 and h > 1:
            rects.append((x + 0.5, y + 0.5, (x + w) - 0.5, (y + h) - 0.5))
    out = []
    for x0, y0, x1, y1 in rects:
        lx = np.array([x0, x1, x1, x0])
        ly = np.array([y0, y0, y1, y1])
        X = tx + (c * lx - s * ly)
        Y = ty + (s * lx + c * ly)
        out.append(np.stack([np.floor(X * 256 + 0.5), np.floor(Y * 256 + 0.5)], -1).astype(np.int64))
    return out


def np_inside(q, px, py):
    ok = np.ones(np.broadcast(px, py).shape, bool)
    for i in range(4):
        ax, ay = q[i]
        dx, dy = q[(i + 1) % 4] - q[i]
        e = dx * (py - ay) - dy * (px - ax)
        ok &= (e > 0) | ((e == 0) & bool(dy < 0 or (dy == 0 and dx > 0)))
    return ok


def np_stroke(so, e, buf, dw, dh, pitch):
    """every sample of every pixel of the canvas -> the composited canvas (in place); -> pixels written"""
    qs = np_corners(so, e)
    if not qs:
        return 0
    i = np.arange(16)
    px = (256 * np.arange(dw)[:, None] + 16 * i[None, :] + 8).reshape(-1)[None, :]
    py = (256 * np.arange(dh)[:, None] + 16 * i[None, :] + 8).reshape(-1)[:, None]
    cov = np_inside(qs[0], px, py)
    if len(qs) == 2:
        cov &= ~np_inside(qs[1], px, py)
    c = cov.reshape(dh, 16, dw, 16).sum(axis=(1, 3)).astype(np.int64)
    a = (255 * c + 128) >> 8
    view = buf.reshape(dh, pitch)[:, :4 * dw].reshape(dh, dw, 4)
    d = view.astype(np.int64)
    da = d[..., 3]
    A = a * 255 + da * (255 - a)
    src = np.array([0, 204, 0] if e.detection == 2 else [0, 0, 204], np.int64)
    Asafe = np.maximum(A, 1)
    out = d.copy()
    out[..., :3] = (src * (a * 255)[..., None] + d[..., :3] * (da * (255 - a))[..., None] + (A // 2)[..., None]) // \
        Asafe[..., None]
    out[..., 3] = (A + 127) // 255
    hit = c > 0
    view[hit] = out[hit].astype(np.uint8)
    return int(hit.sum())


def check(lib, so, e, dw, dh, pad=0, fill="zero", seed=0, brute=True):
    """the library's stroke == the C restatement's (== numpy's); -> (canvas, pixels visited)"""
    a, pitch = canvas(dw, dh, pad, fill, seed)
    b, c = a.copy(), a.copy()
    visited = lib_stroke(lib, e, a, dw, dh, pitch)
    written = oracle_stroke(so, e, b, dw, dh, pitch)
    assert np.array_equal(a, b), (e.detection, e.x, e.y, e.width, e.height, e.angle, dw, dh)
    if brute:
        assert np_stroke(so, e, c, dw, dh, pitch) == written
        assert np.array_equal(a, c)
    assert visited >= written
    return a.reshape(dh, pitch)[:, :4 * dw].reshape(dh, dw, 4), visited


# ---- stroke_sincos --------------------------------------------------------------------------------------------------

def golden_rotations():
    return [c[1] for case in GOLD_D["cases"] for s in case["steps"] for c in s["calls"] if c[0] == "rotate"]


def ulps(got, want):
    return abs(got - want) / np.spacing(abs(want)) if want != 0 else abs(got) / np.spacing(0.0)


def test_sincos_bits_and_accuracy(lib, so):
    half = math.pi / 2
    ts = list(np.linspace(-half, half, 40001)) + golden_rotations()
    ts += [0.0, -0.0, half, -half, np.nextafter(half, 0), np.nextafter(-half, 0), math.pi / 4, -math.pi / 4,
           np.nextafter(math.pi / 4, 1), 1e-300, -1e-300, 5e-324, 1e-8, 0.5, -1.2]
    worst = 0.0
    for t in ts:
        t = float(t)
        got = lib_sincos(lib, t)
        assert [x.hex() for x in got] == [x.hex() for x in oracle_sincos(so, t)], t
        worst = max(worst, ulps(got[0], math.sin(t)), ulps(got[1], math.cos(t)))
    assert worst <= 2.0, worst
    assert lib_sincos(lib, 0.0) == (0.0, 1.0)
    assert lib_sincos(lib, (math.pi / 2) - math.pi / 2) == (0.0, 1.0)          # calcAngles off: angle = pi / 2
    for t in (math.nan, math.inf, -math.inf):
        assert lib_sincos(lib, t) == (0.0, 1.0) == oracle_sincos(so, t)
    assert any(math.isnan(t) for t in golden_rotations())


def test_sincos_outside_the_range_is_deterministic(lib, so):
    """angles beyond [-pi/2, pi/2] reduce the same way on both sides (no accuracy is promised there)"""
    for t in np.linspace(-40.0, 40.0, 4001):
        assert lib_sincos(lib, float(t)) == oracle_sincos(so, float(t))


# ---- strokes --------------------------------------------------------------------------------------------------------

def test_aligned_pins(lib, so):
    """strokeRect(10, 10, 20, 20) on a transparent canvas: the half-pixel line of a browser - both rows / columns of
    every edge at 128, outer corners 64, inner corners 191, nothing else"""
    img, visited = check(lib, so, event(1, 1.0, 10, 10, 20, 20, 0.0), 48, 40)
    a = img[..., 3]
    for X in (9, 10, 29, 30):
        assert (a[11:29, X] == 128).all()
        assert (a[X, 11:29] == 128).all()
    for X, Y in ((9, 9), (30, 9), (9, 30), (30, 30)):
        assert a[Y, X] == 64
    for X, Y in ((10, 10), (29, 10), (10, 29), (29, 29)):
        assert a[Y, X] == 191
    assert (a > 0).sum() == 22 * 22 - 18 * 18          # the ring of pixels 9..30 around 11..28
    assert (img[a > 0][:, :3] == [0, 0, 204]).all()
    assert visited < 4 * 22 * 3                           # the interior is skipped


def golden_vj_boxes():
    return [tuple(c[2:]) for case in GOLD_D["cases"] for s in case["steps"] for c in s["calls"]
            if c[0] == "strokeRect" and c[1] == "#0000CC"]


def test_fractional_vj_boxes(lib, so):
    boxes = golden_vj_boxes()
    assert boxes and any(v != int(v) for b in boxes for v in b)
    for i, (x, y, w, h) in enumerate(dict.fromkeys(boxes)):
        check(lib, so, event(1, 3.5, x, y, w, h, 1.0), 160, 120, fill="random" if i % 2 else "zero", seed=i,
              brute=i < 12)


@pytest.mark.parametrize("fill", ["zero", "opaque", "half"])
def test_rotated_cs_boxes(lib, so, fill):
    """CS boxes rotated by angle - pi/2 about their centre, at angles over [0, pi], 0 and pi included, and NaN"""
    rng = np.random.default_rng(len(fill))
    angles = [0.0, math.pi / 2, math.pi, math.nan, 1e-12, math.pi / 2 + 1e-9] + list(rng.uniform(0, math.pi, 18))
    for i, a in enumerate(angles):
        w, h = float(rng.integers(3, 60)), float(rng.integers(3, 60))
        x, y = float(rng.integers(0, 80)), float(rng.integers(0, 64))
        check(lib, so, event(2, 1.0, x, y, w, h, a), 80, 64, pad=4 * (i % 3), fill=fill, seed=i)


def test_small_sizes_and_lines(lib, so):
    """sizes 0, 1, 2 (no inner rectangle below 2), lines with one zero side, negative sizes, fractional positions"""
    sizes = [0.0, 1.0, 2.0, 0.5, 1.5, 2.25, -1.0, -2.0, -3.5, 7.0]
    n = 0
    for w in sizes:
        for h in sizes:
            for det, ang in ((1, 0.0), (2, 0.3), (2, math.pi / 2)):
                for x, y in ((5.0, 6.0), (5.5, 6.25), (4.3, 7.9)):
                    _, visited = check(lib, so, event(det, 1.0, x, y, w, h, ang), 16, 16, brute=n % 3 == 0)
                    n += 1
                    if w == 0 and h == 0:
                        assert visited == 0


def test_clipped_strokes(lib, so):
    """strokes partly or wholly off the canvas, 1x1 canvases, padded pitches"""
    cases = [(1, -5.0, -5.0, 20.0, 20.0, 0.0, 12, 9), (1, 8.0, 3.0, 30.0, 4.0, 0.0, 12, 9),
             (1, -40.0, 2.0, 10.0, 10.0, 0.0, 12, 9), (1, 2.0, 50.0, 5.0, 5.0, 0.0, 12, 9),
             (2, 0.0, 0.0, 10.0, 14.0, 0.7, 12, 9), (2, 11.0, 8.0, 9.0, 9.0, 2.0, 12, 9),
             (2, 60.0, 60.0, 9.0, 9.0, 2.0, 12, 9), (1, -0.5, -0.5, 1.0, 1.0, 0.0, 1, 1),
             (1, 0.0, 0.0, 1.0, 1.0, 0.0, 1, 1), (2, 0.5, 0.5, 3.0, 3.0, 1.1, 1, 1), (1, 0.25, 0.0, 0.0, 0.5, 0.0, 1, 1),
             (2, -3.0, 4.0, 8.0, 30.0, 1.57, 7, 13), (1, 65536.0, 0.0, 5.0, 5.0, 0.0, 8, 8)]
    for i, (det, x, y, w, h, a, dw, dh) in enumerate(cases):
        for pad in (0, 4, 12):
            check(lib, so, event(det, 1.0, x, y, w, h, a), dw, dh, pad=pad, fill="random", seed=i)


def test_records_that_draw_nothing(lib, so):
    for e in (event(1, 0.0, 5, 5, 4, 4, 0.0), event(2, 0.0, 5, 5, 4, 4, 0.0), event(0, 1.0, 5, 5, 4, 4, 0.0),
              event(3, 1.0, 5, 5, 4, 4, 0.0), event(1, 1.0, math.nan, 5, 4, 4, 0.0),
              event(2, 1.0, 5, 5, math.inf, 4, 0.0), event(1, 1.0, 70000.0, 5, 4, 4, 0.0)):
        img, visited = check(lib, so, e, 16, 16, fill="random")
        assert visited == 0


def test_visits_scale_with_the_perimeter(lib, so):
    """a 300 x 200 box on a 640 x 480 canvas visits about its perimeter, not its area"""
    for det, a in ((1, 0.0), (2, 0.4), (2, 1.2)):
        _, visited = check(lib, so, event(det, 1.0, 320.0 if det == 2 else 170.0, 240.0 if det == 2 else 140.0,
                                          300.0, 200.0, a), 640, 480, brute=False)
        assert 2000 <= visited <= 8000, (det, a, visited)


@pytest.mark.parametrize("case", GOLD_D["cases"], ids=lambda c: c["name"])
def test_golden_lockstep(lib, so, case, blob):
    """every tick: back-projection composite (the oracle's), then the strokes of the tick's record (library) and of
    its debug_calls (restatement); both canvases equal after every tick"""
    a = debug_canvas(case)
    b = a.copy()
    dh, dw = a.shape[:2]
    drawn = 0
    for rec, img in replay(lib, case, blob):
        if img is not None:
            composite(a, img)
            composite(b, img)
        if rec is None:
            continue
        e = event(DET.get(rec["detection"], 0), rec["confidence"], rec["x"], rec["y"], rec["width"], rec["height"],
                  rec["angle"])
        lib_stroke(lib, e, a, dw, dh, 4 * dw)
        oracle_calls(so, debug_calls(rec), b, dw, dh, 4 * dw)
        drawn += bool(debug_calls(rec))
        assert np.array_equal(a, b)
    assert drawn > 0


# ---- the kernel and the ABI -----------------------------------------------------------------------------------------

def test_debug_strokes_does_not_spill(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    m = re.search(r"Function properties for \S*k_debug_strokes\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", out)
    assert m, out[-2000:]
    assert m.groups() == ("0", "0", "0"), m.group(0)


def test_abi_symbol_and_rejections_without_a_device():
    """the entry point is exported; before ht_tracker_config it fails with HT_ERR_STATE whatever else is wrong"""
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_set_debug_strokes") and "ht_tracker_set_debug_strokes" in _lib.EXPORTS
    assert L.ht_tracker_set_debug_strokes(None, 0, 1, (C.c_int32 * 1)(1)) == _lib.HT_ERR_ARG
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "int ht_tracker_set_debug_strokes(ht_ctx *ctx, int first, int n, const int32_t *enable);" in header
