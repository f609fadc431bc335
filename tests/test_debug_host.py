"""CPU: the debug canvas of headtrackr.Tracker (`params.debug`, src/main.js:42-50, 199-219; src/facetrackr.js:193-196)
against the reference's own src/main.js executed by oracle/jsmini.py (tests/golden/reference_js_debug.json,
tools/make_goldens_debug.py):

  * the device state machine (ht_selftest_tracker) in lockstep with the oracle gives per-tick records whose
    streams.debug_calls are the 2D-context calls main.js made on the debug canvas;
  * the oracle's back-projection of the CS frames, composited with the golden's clipping, is every debug canvas;
  * the value table and the clipped writer of k_debug_table / k_debug_backproj, run on the host, against numpy's
    fp64 floor(255 * min(m / c, 1)) and the clipping."""
import ctypes as C
import hashlib
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib
from headtrackr_b200.context import tracker_event_dict
from headtrackr_b200.streams import debug_calls
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_host_lifecycle import TM_CS, TM_IDLE, TM_STARTING, TM_VJ, TM_WB, tracker_params

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD_D = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_debug.json").read_text())
BIN_ZERO = 8 * 4096
DBG_TAB = 4112


def make_frame(kind, t):
    import make_goldens_lifecycle as lg
    return lg.make_frame(kind, t)


def debug_canvas(case):
    import make_goldens_debug as dg
    d = case["debug"]
    return dg.debug_canvas(d["width"], d["height"], d["fill"])


def composite(dst, img):
    h, w = min(img.shape[0], dst.shape[0]), min(img.shape[1], dst.shape[1])
    dst[:h, :w] = img[:h, :w]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def same_calls(got, want, angle_rtol=0.0):
    """call lists equal, NaN equal to NaN; rotation angles within angle_rtol relative"""
    if len(got) != len(want):
        return False
    for g, w in zip(got, want):
        if len(g) != len(w) or g[0] != w[0]:
            return False
        for a, b in zip(g[1:], w[1:]):
            if isinstance(b, str):
                if a != b:
                    return False
            elif not (a == b or (math.isnan(a) and math.isnan(b))
                      or (g[0] == "rotate" and abs(a - b) <= angle_rtol * max(1.0, abs(a), abs(b)))):
                return False
    return True


def replay(st, case, blob):
    """-> per step (record or None for stop, CS frame's back-projection image or None), driven like
    test_host_lifecycle's device replay: the host-compiled tracker_step fed with the oracle's pixel results"""
    st.ht_selftest_tracker_size.restype = C.c_int
    st.ht_selftest_tracker.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    W, H = GOLD_D["width"], GOLD_D["height"]
    params = tracker_params(case)
    state = C.create_string_buffer(st.ht_selftest_tracker_size())
    out = _lib.TrackerEvent()
    seed = (C.c_int32 * 5)()

    def op(code, wb=0.0, det=None, count=0, obj=None, now=0.0):
        return st.ht_selftest_tracker(state, code, C.byref(params), wb, det, count, obj, now, W, H, C.byref(out), seed)

    mode = op(0)
    assert mode == TM_IDLE
    cs, clock, steps = None, 1.0e12, []
    for s in case["steps"]:
        action, (kind, t) = s["action"], s["frame"]
        frame = make_frame(kind, t)
        clock += case["ms_per_frame"]
        if action == "stop":
            mode = op(2)
            steps.append((None, None))
            continue
        if action == "start":
            mode = op(1)
        wb, det, count, obj, img = 0.0, None, 0, None, None
        if mode in (TM_STARTING, TM_WB):
            wb = oracle.whitebalance(frame)
        elif mode == TM_VJ:
            rects = oracle.detect(frame, blob, 5, 1)
            count = len(rects)
            det = (_lib.Rect * max(1, count))(*[_lib.Rect(*r[:5], r[5], 0) for r in rects])
        elif mode == TM_CS:
            cs.track(frame)
            o = cs.track_obj()
            obj = C.byref(_lib.TrackObj(o["x"], o["y"], o["width"], o["height"], o["angle"]))
            img = cs.backprojection_img(frame)
        mode = op(3, wb, det, count, obj, clock)
        if seed[0]:
            cs = oracle.CamshiftTracker(calc_angles=bool(params.calc_angles))
            cs.init_tracker(frame, *seed[1:5])
        steps.append((tracker_event_dict(out), img))
    return steps


def test_golden_covers_the_cases():
    """every case puts at least one image; a lost face, NaN angles, a clipped and a pre-filled larger canvas, and a
    stop / start with retryDetection off are among them"""
    cases = {c["name"]: c for c in GOLD_D["cases"]}
    for c in cases.values():
        assert any(s["put"] for s in c["steps"]), c["name"]
        assert any("redetecting" == s["status"] or "lost" in [e.get("status") for e in s["events"]] for s in c["steps"])
    rot = [x[1] for s in cases["angles"]["steps"] for x in s["calls"] if x[0] == "rotate"]
    assert any(math.isnan(a) for a in rot) and any(abs(a) > 1e-3 for a in rot if not math.isnan(a))
    assert (cases["clipped"]["debug"]["width"], cases["clipped"]["debug"]["height"]) < (GOLD_D["width"], GOLD_D["height"])
    assert cases["larger"]["debug"]["width"] > GOLD_D["width"] and cases["larger"]["debug"]["height"] > GOLD_D["height"]
    assert cases["larger"]["debug"]["fill"] != "zeros"
    actions = [s["action"] for s in cases["no_retry_stop"]["steps"]]
    assert "stop" in actions and actions.count("start") >= 3
    assert not cases["no_retry_stop"]["params"]["retryDetection"]


@pytest.mark.parametrize("case", GOLD_D["cases"], ids=lambda c: c["name"])
def test_debug_calls_and_canvases_match_reference_js(st, case, blob):
    """per step: debug_calls(record) == the golden's calls, the canvas composited from the oracle's back-projection
    of the CS frames == the golden's hash, and a put happened exactly on the CS ticks"""
    dbg = debug_canvas(case)
    initial = dbg.copy()
    W, H = GOLD_D["width"], GOLD_D["height"]
    dw, dh = case["debug"]["width"], case["debug"]["height"]
    clipped_away = False
    for n, ((rec, img), want) in enumerate(zip(replay(st, case, blob), case["steps"])):
        calls = [] if rec is None else debug_calls(rec)
        assert same_calls(calls, want["calls"]), (n, calls, want["calls"])
        assert (img is not None) == want["put"], n
        if img is not None:
            assert rec["detection"] == "CS"
            composite(dbg, img)
            clipped_away |= bool(img[dh:].any() or img[:, dw:].any())
        assert sha(dbg) == want["debug_sha256"], n
        assert np.array_equal(dbg[H:], initial[H:]) and np.array_equal(dbg[:, W:], initial[:, W:])   # never cleared
    if (dw, dh) < (W, H):
        assert clipped_away            # the image had content outside the debug canvas
    if dw > W:
        assert initial[H:].any() and initial[:, W:].any()


def value_table(st, m, c):
    st.ht_selftest_debug_table.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    m = np.ascontiguousarray(m, np.uint32)
    c = np.ascontiguousarray(c, np.uint32)
    out = np.full(DBG_TAB, 77, np.uint8)
    assert st.ht_selftest_debug_table(m.ctypes.data, c.ctypes.data, out.ctypes.data) == DBG_TAB
    return out


def numpy_values(m, c):
    m, c = np.asarray(m, np.float64), np.asarray(c, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(c == 0, 0.0, np.minimum(m / c, 1.0))
    return np.floor(255 * p).astype(np.uint8)


def test_value_table_sweep(st):
    """4096 (m, c) pairs per table: c = 0, m >= c, ratios on and next to k / 255, random counts; entry 4096 (BIN_ZERO)
    is 0 and the padding is written"""
    rng = np.random.default_rng(11)
    sets = []
    m = rng.integers(0, 1 << 20, 4096)
    c = m.copy()
    c[:1024] = 0                                                     # no current pixel of that colour
    c[1024:2048] = rng.integers(1, 1 << 20, 1024) // 7 + 1            # mostly m >= c: saturates at 255
    c[2048:] = m[2048:] + rng.integers(0, 1 << 20, 2048)             # m <= c
    sets.append((m, c))
    k = np.arange(1, 255)                                            # m / c straddling k / 255
    mm, cc = [], []
    for c0 in (255, 3 * 255, 255 * 97, 255 * 4099, 65535 * 255, 1 << 24, 3, 7, 1023):
        for d in (-1, 0, 1):
            mm.append(np.clip((k * c0) // 255 + d, 0, None))
            cc.append(np.full_like(k, c0))
    mm, cc = np.concatenate(mm), np.concatenate(cc)
    pad = 4096 - len(mm) % 4096
    mm = np.concatenate([mm, rng.integers(0, 1000, pad)])
    cc = np.concatenate([cc, rng.integers(0, 1000, pad)])
    for i in range(0, len(mm), 4096):
        sets.append((mm[i:i + 4096], cc[i:i + 4096]))
    on_k = 0
    for m, c in sets:
        got = value_table(st, m, c)
        assert np.array_equal(got[:4096], numpy_values(m, c))
        assert (got[4096:] == 0).all()
        on_k += int(((255 * m) % np.maximum(c, 1) == 0).sum())
    assert on_k > 1000


@pytest.mark.parametrize("w,h,dw,dh,pad", [(160, 120, 160, 120, 0), (160, 120, 100, 80, 0), (160, 120, 200, 150, 0),
                                            (131, 37, 67, 200, 12), (640, 480, 641, 33, 4), (7, 5, 3, 9, 0),
                                            (320, 240, 320, 240, 16)])
def test_clipped_writer(st, w, h, dw, dh, pad):
    """plane entries (8 * bin, or BIN_ZERO) -> (v, v, v, 255) over min(w, dw) x min(h, dh); everything else, row
    padding included, keeps its bytes; 16-byte stores where the canvas and its pitch allow"""
    st.ht_selftest_debug_write.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int]
    rng = np.random.default_rng(w * 7 + dh)
    b = rng.integers(0, 4096, (h, w))
    plane = np.where(rng.random((h, w)) < 0.2, BIN_ZERO, 8 * b).astype(np.uint16)
    m, c = rng.integers(0, 50, 4096), rng.integers(0, 60, 4096)
    table = value_table(st, m, c)
    pitch = 4 * dw + pad
    raw = np.empty(dh * pitch + 16, np.uint8)
    off = (-raw.ctypes.data) % 16                                    # a 16-byte aligned canvas
    buf = raw[off:off + dh * pitch]
    buf[:] = rng.integers(0, 256, buf.size, dtype=np.uint8)
    before = buf.copy()
    stores = st.ht_selftest_debug_write(plane.ctypes.data, w, h, table.ctypes.data, buf.ctypes.data, dw, dh, pitch)
    got = buf.reshape(dh, pitch)
    want = before.reshape(dh, pitch).copy()
    cw, chh = min(w, dw), min(h, dh)
    v = table[plane[:chh, :cw] >> 3]
    want4 = want[:chh, :4 * cw].reshape(chh, cw, 4)
    want4[..., 0] = want4[..., 1] = want4[..., 2] = v
    want4[..., 3] = 255
    assert np.array_equal(got, want)
    assert (plane[:chh, :cw] == BIN_ZERO).any() and (v[plane[:chh, :cw] == BIN_ZERO] == 0).all()
    assert stores == (chh * (cw // 4) if pitch % 16 == 0 else 0)


def test_debug_canvas_abi(tmp_path):
    """DebugCanvas == ht_debug_canvas of the header, checked by the C compiler; the entry point is exported"""
    L = _lib.lib()
    assert hasattr(L, "ht_tracker_set_debug") and "ht_tracker_set_debug" in _lib.EXPORTS
    src = tmp_path / "layout.cpp"
    src.write_text('#include <cstdio>\n#include "headtrackr_b200.h"\nint main() {\n'
                   '  std::printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(ht_debug_canvas), offsetof(ht_debug_canvas, rgba),\n'
                   '              offsetof(ht_debug_canvas, width), offsetof(ht_debug_canvas, height),\n'
                   '              offsetof(ht_debug_canvas, pitch), offsetof(ht_debug_canvas, pad_));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([_lib.nvcc(), "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    D = _lib.DebugCanvas
    assert got == [C.sizeof(D), D.rgba.offset, D.width.offset, D.height.offset, D.pitch.offset, D.pad_.offset] == \
        [24, 0, 8, 12, 16, 20]
