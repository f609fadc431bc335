"""CPU: headtrackr.Tracker's lifecycle from its first frame - the starter's content check, the whitebalance gate,
status events, stop() / start(), retryDetection off, the "hints" timer - against the reference's own src/main.js
executed by oracle/jsmini.py (tests/golden/reference_js_lifecycle.json, tools/make_goldens_lifecycle.py):

  * the Python mirror main.Tracker with the oracle backend;
  * the device state machine itself (tracker_step in ht_track.cuh, compiled for the host through ht_selftest_tracker),
    driven frame by frame in lockstep with the oracle's whitebalance, detection and camshift results, over every
    case of the lifecycle golden and of reference_js_main.json, from frame 0."""
import ctypes as C
import json
import sys
from pathlib import Path

import pytest

import oracle
from headtrackr_b200 import _lib
from headtrackr_b200.context import tracker_event_dict
from headtrackr_b200.streams import lifecycle_events
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_host_main import GOLD_M, check_events, same

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD_L = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_lifecycle.json").read_text())

TM_IDLE, TM_STARTING, TM_WB, TM_VJ, TM_CS = range(5)


def make_frame(kind, t):
    import make_goldens_lifecycle as lg
    return lg.make_frame(kind, t)


def case_spec(case):
    """-> [(action, kind, t)], ms per frame.  reference_js_main.json: start() on frame 0, then one timer per frame."""
    if "ms_per_frame" in case:
        return [(s["action"], *s["frame"]) for s in case["steps"]], case["ms_per_frame"]
    return [("start" if n == 0 else "tick", *s["frame"]) for n, s in enumerate(case["steps"])], 35.0


ALL_CASES = [("lifecycle", c) for c in GOLD_L["cases"]] + [("main", c) for c in GOLD_M["cases"]]


def case_id(gc):
    return f"{gc[0]}-{gc[1]['name']}"


def strip_time(evts):
    return [{k: v for k, v in e.items() if k != "time"} for e in evts]


@pytest.mark.parametrize("case", GOLD_L["cases"], ids=lambda c: c["name"])
def test_main_tracker_lifecycle_matches_reference_js(case, blob):
    from headtrackr_b200 import Canvas, main
    from test_host_logic import OracleBackend
    import numpy as np
    spec, ms = case_spec(case)
    W, H = GOLD_L["width"], GOLD_L["height"]
    video = Canvas(make_frame(*spec[0][1:]))
    canvas = Canvas(np.zeros((H, W, 4), np.uint8))
    clock = [1.0e12]
    ht = main.Tracker(dict(case["params"], ui=False), backend=OracleBackend(blob), clock=lambda: clock[0])
    log = []
    for t in ("headtrackrStatus", "facetrackingEvent", "headtrackingEvent"):
        ht.addEventListener(t, log.append)
    ht.init(video, canvas, False)
    for n, ((action, kind, t), want) in enumerate(zip(spec, case["steps"])):
        video.pixels = make_frame(kind, t)
        clock[0] += ms
        n0 = len(log)
        if action == "start":
            assert ht.start() is True
        elif action == "stop":
            ht.stop()
        else:
            ht.step()
        check_events(strip_time(log[n0:]), want["events"])
        assert ht.status == want["status"], n
        assert same(ht.getFOV(), want["fov"]), n
    n0 = len(log)
    ht.stop()
    check_events(strip_time(log[n0:]), case["stop_events"])
    assert same(ht.getFOV(), case["fov"])


def tracker_params(case):
    p = case["params"] or {}
    head = _lib.HeadParams(int(p.get("smoothing", True)), int(p.get("headPosition", True)), 1, 0, 0.35,
                           float(p["fov"]) if p.get("fov") is not None else 0.0, float(p.get("cameraOffset", 11.5)), 60.0)
    return _lib.TrackerParams(int(p.get("retryDetection", True)), int(p.get("calcAngles", False)), (C.c_int32 * 2)(), head)


@pytest.mark.parametrize("gc", ALL_CASES, ids=case_id)
def test_device_state_machine_replays_every_step(st, gc, blob):
    """tracker_step, the function k_tracker_update runs per stream, reproduces every event, status and fov."""
    _, case = gc
    st.ht_selftest_tracker_size.restype = C.c_int
    st.ht_selftest_tracker.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    spec, ms = case_spec(case)
    W, H = GOLD_L["width"], GOLD_L["height"]
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
    for n, ((action, kind, t), want) in enumerate(zip(spec, case["steps"])):
        frame = make_frame(kind, t)
        clock += ms
        if action == "stop":
            mode = op(2)
            evts, status = [dict(type="headtrackrStatus", status="stopped")], "stopped"
        else:
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
            if seed[0]:                                   # a new facetrackr's camshift.Tracker, seeded on this frame
                cs = oracle.CamshiftTracker(calc_angles=bool(params.calc_angles))
                cs.init_tracker(frame, *seed[1:5])
            rec = tracker_event_dict(out)
            evts, status = lifecycle_events(rec, status)
            assert rec["running"] == (mode in (TM_WB, TM_VJ, TM_CS)), n
        check_events(evts, want["events"])
        assert status == want["status"], (n, status, want["status"])
        if "fov" in want:                                 # (reference_js_main.json records getFOV() once per case)
            assert same(out.fov, want["fov"]), n
    op(2)
    check_events([dict(type="headtrackrStatus", status="stopped")], case["stop_events"])
    assert same(out.fov, case["fov"])
    assert {TM_WB, TM_VJ, TM_CS} <= seen
