"""CPU: headtrackr.Tracker with non-default parameters on canvases other than 160x120 (tests/golden/reference_js_params.json,
tools/make_goldens_params.py: calcAngles, cameraOffset, fov, headPosition, smoothing; 200x150 and a portrait 120x160)
against the reference's own src/main.js executed by oracle/jsmini.py:

  * the Python mirror main.Tracker with the oracle backend;
  * the device state machine (tracker_step, compiled for the host through ht_selftest_tracker) in lockstep with the
    oracle's whitebalance, detection and camshift, at each case's canvas size - including the NaN angle of the frame
    on which calcAngles tracking loses the face.

Also the per-record draw of ht_tracker_feed_canvases (k_feed_draw's mixed-size path, run on the host) against the
oracle's drawImage, and the ht_canvas_frame ABI."""
import ctypes as C
import json
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib, synth
from headtrackr_b200.context import tracker_event_dict
from headtrackr_b200.streams import lifecycle_events
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_feed_host import oracle_resize, padded
from test_host_lifecycle import TM_CS, TM_IDLE, TM_STARTING, TM_VJ, TM_WB, tracker_params
from test_host_main import check_events, same

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD_P = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_params.json").read_text())


def make_frame(case, kind, t):
    import make_goldens_params as pg
    return pg.make_frame(kind, t, case["width"], case["height"])


def case_spec(case):
    return [(s["action"], *s["frame"]) for s in case["steps"]]


def test_golden_covers_the_parameters():
    """two canvas sizes other than 160x120 (one portrait), calcAngles, and cameraOffset / fov / headPosition that
    differ between the cases; every case tracks, loses the face and finds it again"""
    cases = GOLD_P["cases"]
    sizes = {(c["width"], c["height"]) for c in cases}
    assert len(sizes - {(160, 120)}) >= 2 and any(h > w for w, h in sizes)
    assert any(c["params"].get("calcAngles") for c in cases)
    for key in ("cameraOffset", "fov", "headPosition"):
        assert len({repr(c["params"].get(key)) for c in cases}) >= 2, key
    for c in cases:
        statuses = [s["status"] for s in c["steps"]]
        assert {"whitebalance", "detecting", "found", "tracking", "redetecting"} <= set(statuses), c["name"]
        assert statuses.index("redetecting") < len(statuses) - 1 - statuses[::-1].index("found"), c["name"]
        head = any(e["type"] == "headtrackingEvent" for s in c["steps"] for e in s["events"])
        assert head == c["params"].get("headPosition", True), c["name"]
    lost = [e["angle"] for c in cases if c["params"].get("calcAngles") for s in c["steps"] for e in s["events"]
            if e["type"] == "facetrackingEvent" and e["detection"] == "CS" and e["width"] == 0]
    assert lost and all(math.isnan(a) for a in lost)


@pytest.mark.parametrize("case", GOLD_P["cases"], ids=lambda c: c["name"])
def test_main_tracker_matches_reference_js(case, blob):
    from headtrackr_b200 import Canvas, main
    from test_host_logic import OracleBackend
    W, H = case["width"], case["height"]
    spec = case_spec(case)
    video = Canvas(make_frame(case, *spec[0][1:]))
    canvas = Canvas(np.zeros((H, W, 4), np.uint8))
    clock = [1.0e12]
    ht = main.Tracker(dict(case["params"], ui=False), backend=OracleBackend(blob), clock=lambda: clock[0])
    log = []
    for t in ("headtrackrStatus", "facetrackingEvent", "headtrackingEvent"):
        ht.addEventListener(t, lambda e: log.append({k: v for k, v in e.items() if k != "time"}))
    ht.init(video, canvas, False)
    for n, ((action, kind, t), want) in enumerate(zip(spec, case["steps"])):
        video.pixels = make_frame(case, kind, t)
        clock[0] += case["ms_per_frame"]
        n0 = len(log)
        if action == "start":
            assert ht.start() is True
        else:
            assert ht.step() is True
        check_events(log[n0:], want["events"])
        assert ht.status == want["status"], n
        assert same(ht.getFOV(), want["fov"]), n
    n0 = len(log)
    ht.stop()
    check_events(log[n0:], case["stop_events"])
    assert same(ht.getFOV(), case["fov"])


@pytest.mark.parametrize("case", GOLD_P["cases"], ids=lambda c: c["name"])
def test_device_state_machine_replays_every_step(st, case, blob):
    """tracker_step, which k_tracker_update runs per stream with the stream's own parameters and canvas size"""
    st.ht_selftest_tracker_size.restype = C.c_int
    st.ht_selftest_tracker.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    W, H = case["width"], case["height"]
    params = tracker_params(case)
    state = C.create_string_buffer(st.ht_selftest_tracker_size())
    out = _lib.TrackerEvent()
    seed = (C.c_int32 * 5)()

    def op(code, wb=0.0, det=None, count=0, obj=None, now=0.0):
        return st.ht_selftest_tracker(state, code, C.byref(params), wb, det, count, obj, now, W, H, C.byref(out), seed)

    mode = op(0)
    assert mode == TM_IDLE
    cs = None
    clock, status, seen = 1.0e12, "", set()
    for n, ((action, kind, t), want) in enumerate(zip(case_spec(case), case["steps"])):
        frame = make_frame(case, kind, t)
        clock += case["ms_per_frame"]
        if action == "start":
            mode = op(1)
        wb, det, count, obj = 0.0, None, 0, None
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
        seen.add(mode)
        mode = op(3, wb, det, count, obj, clock)
        if seed[0]:
            cs = oracle.CamshiftTracker(calc_angles=bool(params.calc_angles))
            cs.init_tracker(frame, *seed[1:5])
        rec = tracker_event_dict(out)
        evts, status = lifecycle_events(rec, status)
        check_events(evts, want["events"])
        assert status == want["status"], (n, status, want["status"])
        assert same(out.fov, want["fov"]), n
    op(2)
    check_events([dict(type="headtrackrStatus", status="stopped")], case["stop_events"])
    assert same(out.fov, case["fov"])
    assert {TM_WB, TM_VJ, TM_CS} <= seen


def feed_canvases(st, videos, canvases, draw, out):
    st.ht_selftest_feed_canvases.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    st.ht_selftest_feed_canvases.restype = C.c_int
    recs = (_lib.CanvasFrame * len(videos))()
    for b, (v, (cw, ch)) in enumerate(zip(videos, canvases)):
        assert v.strides[1:] == (4, 1)
        recs[b] = _lib.CanvasFrame(_lib.VideoFrame(v.ctypes.data, b, v.shape[1], v.shape[0], v.strides[0], 0.0), cw, ch)
    d = np.asarray(draw, np.uint8)
    return st.ht_selftest_feed_canvases(C.addressof(recs), len(videos), d.ctypes.data, out.ctypes.data)


def test_mixed_canvas_batch_equals_the_oracle(st):
    """records of different video sizes and pitches, 1:1 records among them, each onto its own canvas size"""
    videos = [synth.frame(90, 640, 480), synth.frame(91, 333, 251), synth.frame(92, 200, 150), synth.frame(93, 120, 160),
              synth.frame(94, 160, 120), synth.frame(95, 1280, 720), synth.frame(96, 64, 48)]
    videos[1][..., 3] = (np.arange(333) % 256).astype(np.uint8)[None, :]     # a non-constant alpha channel
    videos[1] = padded(videos[1], 13)
    videos[2] = padded(videos[2], 3)                                         # a 1:1 record with a padded pitch
    canvases = [(320, 240), (240, 320), (200, 150), (120, 160), (160, 120), (97, 83), (320, 240)]
    draw = [1, 1, 1, 1, 1, 1, 0]                                             # the last stream is IDLE
    total = sum(w * h * 4 for w, h in canvases)
    out = np.random.default_rng(7).integers(0, 256, total, dtype=np.uint8)
    before = out.copy()
    tiles = feed_canvases(st, videos, canvases, draw, out)
    assert tiles == sum(((w + 63) // 64) * ((h + 15) // 16) for w, h in canvases)
    off = 0
    for b, (v, (cw, ch)) in enumerate(zip(videos, canvases)):
        got = out[off:off + cw * ch * 4].reshape(ch, cw, 4)
        if draw[b]:
            want = oracle_resize(np.ascontiguousarray(v), cw, ch)
            assert np.array_equal(got, want), (b, v.shape, cw, ch)
            if v.shape[:2] == (ch, cw):
                assert np.array_equal(got, v)                                # a 1:1 draw is a copy
        else:
            assert np.array_equal(got, before[off:off + cw * ch * 4].reshape(ch, cw, 4))
        off += cw * ch * 4


def test_mixed_canvas_draw_matches_the_one_size_draw(st):
    """a record gives the same canvas whatever else is in the call"""
    videos = [synth.frame(100 + i, w, h) for i, (w, h) in enumerate([(640, 480), (320, 240), (200, 150)])]
    canvases = [(200, 150), (120, 160), (200, 150)]
    out = np.zeros(sum(w * h * 4 for w, h in canvases), np.uint8)
    feed_canvases(st, videos, canvases, [1, 1, 1], out)
    st.ht_selftest_feed_draw.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    off = 0
    for b, (v, (cw, ch)) in enumerate(zip(videos, canvases)):
        recs = (_lib.VideoFrame * 1)(_lib.VideoFrame(v.ctypes.data, 0, v.shape[1], v.shape[0], v.strides[0], 0.0))
        one = np.zeros((1, ch, cw, 4), np.uint8)
        d = np.ones(1, np.uint8)
        assert st.ht_selftest_feed_draw(C.addressof(recs), 1, d.ctypes.data, one.ctypes.data, cw, ch) == 0
        assert np.array_equal(out[off:off + cw * ch * 4].reshape(ch, cw, 4), one[0])
        off += cw * ch * 4


def test_canvas_frame_abi(tmp_path):
    """CanvasFrame == ht_canvas_frame of the header, checked by the C compiler; the new entry points are exported"""
    L = _lib.lib()
    for name in ("ht_tracker_set_params", "ht_tracker_feed_canvases"):
        assert hasattr(L, name) and name in _lib.EXPORTS
    assert L.ht_version() == (1 << 16) | 3
    src = tmp_path / "layout.cpp"
    src.write_text('#include <cstdio>\n#include "headtrackr_b200.h"\nint main() {\n'
                   '  std::printf("%zu %zu %zu %zu %zu\\n", sizeof(ht_canvas_frame), offsetof(ht_canvas_frame, video),\n'
                   '              offsetof(ht_canvas_frame, canvas_w), offsetof(ht_canvas_frame, canvas_h),\n'
                   '              offsetof(ht_canvas_frame, pad_));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([_lib.nvcc(), "-x", "c++", "-I", str(ROOT / "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    CF = _lib.CanvasFrame
    assert got == [C.sizeof(CF), CF.video.offset, CF.canvas_w.offset, CF.canvas_h.offset, CF.pad_.offset] == [48, 0, 32, 36, 40]
