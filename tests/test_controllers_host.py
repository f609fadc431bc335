"""CPU: the head-coupled camera controller, realisticAbsoluteCameraControl (src/controllers.js:28-68), against the
reference's own controllers.js and main.js executed by oracle/jsmini.py (tests/golden/reference_js_controllers.json,
tools/make_goldens_controllers.py):

  * the Python mirror headtrackr_b200.controllers, listening to main.Tracker with the oracle backend;
  * the device code itself (camera_step and camera_construct in ht_track.cuh, compiled for the host through
    ht_selftest_camera), fed by the device state machine tracker_step in lockstep with the oracle, as
    tests/test_host_lifecycle.py drives it;

every fp64 field of the camera after every tick bit-identical to the reference's (signed zeros included; jsmini's
Math.atan is the host libm's), the constructed camera, the float32 matrices bit-identical to a numpy restatement of
DESIGN.md 5.4 (f10), and the parameter checks of ht_tracker_set_camera."""
import ctypes as C
import json
import math
import struct
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import _lib, controllers
from headtrackr_b200.context import camera_from_bytes, tracker_event_dict
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD_C = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_controllers.json").read_text())
CASES = GOLD_C["cases"]

TM_IDLE, TM_STARTING, TM_WB, TM_VJ, TM_CS = range(5)


def make_frame(case, kind, t):
    import make_goldens_lifecycle as lg
    import make_goldens_params as pg
    if case["frames"] == "main":
        return lg.make_frame(kind, t)
    return pg.make_frame(kind, t, case["width"], case["height"])


def bits(v):
    return struct.pack("<d", float(v))


def same_bits(a, b):
    """fp64 values (or lists of them) with the same bit pattern; NaN matches NaN"""
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same_bits(x, y) for x, y in zip(a, b))
    return bits(a) == bits(b) or (a != a and b != b)


def control(case, camera=None):
    """the case's ht_camera_control (the reference's defaults for absent params)"""
    c, cam = case["control"], case["camera"]
    p = c["params"] or {}
    return _lib.CameraControl(camera, c["scaling"], tuple(c["fixedPosition"]), tuple(c["lookAt"]),
                              p.get("screenHeight", 20.0), p.get("damping", 1.0), cam["fov"], cam["aspect"],
                              cam["near"], cam["far"])


def check_camera(got, want, where):
    """got: a camera_from_bytes / controllers state dict; want: a golden camera record"""
    assert same_bits(got["position"], want["position"]), (where, got["position"], want["position"])
    assert same_bits(got["fov"], want["fov"]), (where, got["fov"], want["fov"])
    assert got["events"] == want["events"], where
    if want["view"] is None:
        assert got["has_view_offset"] == 0 and same_bits(got["view"], [0.0] * 6), where
    else:
        assert got["has_view_offset"] == 1 and same_bits(got["view"], want["view"]), (where, got["view"], want["view"])


def restated(case, cam):
    """(projection, view matrix) of a golden camera record by the numpy restatement of DESIGN.md 5.4 (f10)"""
    c, k = case["control"], case["camera"]
    rot = controllers.look_at(c["fixedPosition"], c["lookAt"])
    proj = controllers.projection_matrix(cam["fov"], k["aspect"], k["near"], k["far"], cam["view"])
    return proj, controllers.view_matrix(rot, cam["position"])


def same_f32(a, b):
    """float32 arrays with the same bit patterns; NaN matches NaN (its sign and payload are not specified)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def selftest(st):
    st.ht_selftest_camera.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_double, C.c_void_p]
    st.ht_selftest_camera.restype = C.c_int
    return st


def decode(cam):
    return camera_from_bytes(np.frombuffer(C.string_at(C.addressof(cam), C.sizeof(cam)), np.uint8))


def test_golden_covers_the_listener():
    """both sides of each ternary of src/controllers.js:51-52, a stop/start and a lost-and-refound face"""
    heads = [s["head"] for case in CASES for s in case["steps"] if s["head"]]
    assert any(h[0] > 0 for h in heads) and any(h[0] <= 0 for h in heads)
    assert any(h[1] < 0 for h in heads) and any(h[1] >= 0 for h in heads)
    assert any(s["action"] == "stop" for case in CASES for s in case["steps"])
    assert any(s["status"] == "redetecting" for case in CASES for s in case["steps"])
    assert {c["name"] for c in CASES} >= {"defaults", "damped", "angles_200x150", "portrait_120x160", "no_retry_stop"}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_construction(st, case):
    """setting a controller writes the constructed camera: position = fixedPosition, the camera's own fov, no view
    offset, no events; and its matrices are makePerspective's and lookAt's"""
    L = selftest(st)
    cam = _lib.Camera()
    assert L.ht_selftest_camera(C.byref(control(case)), 0, 0.0, 0.0, 0.0, C.byref(cam)) == 0
    got = decode(cam)
    check_camera(got, case["constructed"], "constructed")
    assert case["constructed"]["events"] == 0 and case["constructed"]["view"] is None
    assert same_bits(got["position"], case["control"]["fixedPosition"]) and got["fov"] == case["camera"]["fov"]
    proj, view = restated(case, case["constructed"])
    assert same_f32(got["projection"], proj) and same_f32(got["view_matrix"], view)
    assert list(cam.pad_) == [0, 0]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_controllers_py_replays_the_golden(case):
    """headtrackr_b200.controllers over the golden's own headtrackingEvents: every camera field bit for bit"""
    k = case["camera"]
    cam = controllers.PerspectiveCamera(k["fov"], k["aspect"], k["near"], k["far"])
    c = case["control"]
    ctl = controllers.realisticAbsoluteCameraControl(cam, c["scaling"], c["fixedPosition"], c["lookAt"], c["params"])
    check_camera(ctl.state(), case["constructed"], "constructed")
    for n, s in enumerate(case["steps"]):
        if s["head"]:
            ctl.handleEvent(dict(type="headtrackingEvent", x=s["head"][0], y=s["head"][1], z=s["head"][2]))
        check_camera(ctl.state(), s["camera"], (case["name"], n))
        proj, view = restated(case, s["camera"])
        assert same_f32(ctl.state()["projection"], proj) and same_f32(ctl.state()["view_matrix"], view), n


@pytest.mark.parametrize("case", [c for c in CASES if c["frames"] == "main"], ids=lambda c: c["name"])
def test_controllers_py_listens_to_main_tracker(case, blob):
    """the mirror registered on main.Tracker (oracle backend): it hears the tracker's headtrackingEvents and only
    those, and the cameras agree with the reference's"""
    from headtrackr_b200 import Canvas, main
    from test_host_logic import OracleBackend
    from test_host_main import same
    W, H = case["width"], case["height"]
    video = Canvas(make_frame(case, *case["steps"][0]["frame"]))
    canvas = Canvas(np.zeros((H, W, 4), np.uint8))
    clock = [1.0e12]
    ht = main.Tracker(dict(case["params"], ui=False), backend=OracleBackend(blob), clock=lambda: clock[0])
    k, c = case["camera"], case["control"]
    cam = controllers.PerspectiveCamera(k["fov"], k["aspect"], k["near"], k["far"])
    ctl = controllers.realisticAbsoluteCameraControl(cam, c["scaling"], c["fixedPosition"], c["lookAt"], c["params"],
                                                     tracker=ht)
    ht.init(video, canvas, False)
    for n, s in enumerate(case["steps"]):
        video.pixels = make_frame(case, *s["frame"])
        clock[0] += case["ms_per_frame"]
        if s["action"] == "start":
            assert ht.start() is True
        elif s["action"] == "stop":
            ht.stop()
        else:
            ht.step()
        got, want = ctl.state(), s["camera"]
        assert got["events"] == want["events"], n
        for a, b in zip(got["position"] + [got["fov"]] + got["view"], want["position"] + [want["fov"]]
                        + (want["view"] or [0.0] * 6)):
            assert same(a, b), (n, got, want)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_device_camera_in_lockstep_with_the_state_machine(st, case, blob):
    """tracker_step (k_tracker_update's per-stream code) in lockstep with the oracle, and camera_step (k_camera_update's)
    on each record with head.valid: every camera bit-identical to the reference's after every tick"""
    L = selftest(st)
    L.ht_selftest_tracker_size.restype = C.c_int
    L.ht_selftest_tracker.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p,
                                      C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    from test_host_lifecycle import tracker_params
    W, H = case["width"], case["height"]
    params = tracker_params(case)
    state = C.create_string_buffer(L.ht_selftest_tracker_size())
    out = _lib.TrackerEvent()
    seed = (C.c_int32 * 5)()
    ctl = control(case)
    cam = _lib.Camera()
    assert L.ht_selftest_camera(C.byref(ctl), 0, 0.0, 0.0, 0.0, C.byref(cam)) == 0

    def op(code, wb=0.0, det=None, count=0, obj=None, now=0.0):
        return L.ht_selftest_tracker(state, code, C.byref(params), wb, det, count, obj, now, W, H, C.byref(out), seed)

    mode = op(0)
    cs = None
    clock = 1.0e12
    for n, s in enumerate(case["steps"]):
        frame = make_frame(case, *s["frame"])
        clock += case["ms_per_frame"]
        head = None
        if s["action"] == "stop":
            mode = op(2)
        else:
            if s["action"] == "start":
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
            mode = op(3, wb, det, count, obj, clock)
            if seed[0]:
                cs = oracle.CamshiftTracker(calc_angles=bool(params.calc_angles))
                cs.init_tracker(frame, *seed[1:5])
            rec = tracker_event_dict(out)
            if out.head.valid:
                head = [out.head.x, out.head.y, out.head.z]
                assert L.ht_selftest_camera(C.byref(ctl), 1, *head, C.byref(cam)) == cam.events
        assert (head is None) == (s["head"] is None), n
        if head:
            assert same_bits(head, s["head"]), (n, rec)
        got = decode(cam)
        check_camera(got, s["camera"], (case["name"], n))
        proj, view = restated(case, s["camera"])
        assert same_f32(got["projection"], proj) and same_f32(got["view_matrix"], view), n


def test_matrices_match_the_restatement_over_random_controls(st):
    """random controls and events, including z * scaling == 0 (fov = atan(+Infinity) * 360 / PI = 180), negative
    zeros and events on both sides of the ternaries: camera_step's fields equal the mirror's bit for bit and its
    float32 matrices the numpy restatement's"""
    L = selftest(st)
    rng = np.random.default_rng(10)
    for trial in range(300):
        look = rng.normal(size=3) * 50
        fixed = rng.normal(size=3) * 50
        scaling = float(rng.choice([1.0, 0.37, 2.5, 0.0, float(rng.uniform(0.01, 10))]))
        sh, damping = float(rng.uniform(5, 40)), float(rng.choice([1.0, 0.5, float(rng.uniform(0, 2))]))
        fov, aspect = float(rng.uniform(1, 179)), float(rng.uniform(0.2, 4))
        near = float(rng.uniform(0.01, 10))
        far = near * float(rng.uniform(1.5, 1e4))
        ctl = _lib.CameraControl(None, scaling, tuple(fixed), tuple(look), sh, damping, fov, aspect, near, far)
        cam = _lib.Camera()
        assert L.ht_selftest_camera(C.byref(ctl), 0, 0.0, 0.0, 0.0, C.byref(cam)) == 0
        pc = controllers.PerspectiveCamera(fov, aspect, near, far)
        mirror = controllers.realisticAbsoluteCameraControl(pc, scaling, fixed, look, dict(screenHeight=sh,
                                                                                            damping=damping))
        for e in range(4):
            x, y, z = rng.normal(size=3) * 30
            x = [x, 0.0, -0.0][e % 3] if trial % 5 == 0 else x
            z = 0.0 if trial % 7 == 0 else abs(z) + 1
            assert L.ht_selftest_camera(C.byref(ctl), 1, x, y, z, C.byref(cam)) == e + 1
            mirror.handleEvent(dict(x=x, y=y, z=z))
            got, want = decode(cam), mirror.state()
            assert same_bits(got["position"], want["position"]) and same_bits(got["view"], want["view"])
            assert same_bits(got["fov"], want["fov"]) and got["events"] == want["events"]
            if z * scaling == 0:
                assert got["fov"] == 180.0 or got["fov"] != got["fov"]
            assert same_f32(got["projection"], want["projection"]), (trial, e)
            assert same_f32(got["view_matrix"], want["view_matrix"]), (trial, e)


def test_restatement_is_the_matrix_algebra():
    """the restated matrices are what they claim: the view matrix inverts T(position) R and maps lookAt onto the -z
    axis; the off-axis frustum with a zero offset over the full view is makePerspective with aspect fullWidth /
    fullHeight"""
    rot = controllers.look_at([1.0, 2.0, 30.0], [0.0, -1.0, 0.0])
    assert np.allclose(rot.T @ rot, np.eye(3), atol=1e-15)
    t = np.eye(4)
    t[:3, :3] = rot
    t[:3, 3] = [1.0, 2.0, 30.0]
    v = controllers.view_matrix(rot, [1.0, 2.0, 30.0]).astype(np.float64)
    assert np.allclose(v @ t, np.eye(4), atol=1e-6)
    p = v @ np.array([0.0, -1.0, 0.0, 1.0])
    assert abs(p[0]) < 1e-5 and abs(p[1]) < 1e-5 and p[2] < 0
    a = controllers.projection_matrix(50.0, 4 / 3, 1.0, 100.0, [40.0, 30.0, 0.0, 0.0, 40.0, 30.0])
    b = controllers.projection_matrix(50.0, 4 / 3, 1.0, 100.0)
    assert np.allclose(a, b, rtol=1e-6)


REJECT = [
    ("scaling NaN", dict(scaling=math.nan)),
    ("fixedPosition inf", dict(fixed_position=(0.0, math.inf, 0.0))),
    ("lookAt NaN", dict(look_at=(math.nan, 0.0, 0.0))),
    ("screenHeight inf", dict(screen_height=math.inf)),
    ("damping NaN", dict(damping=math.nan)),
    ("fov 0", dict(fov=0.0)),
    ("fov 180", dict(fov=180.0)),
    ("fov -1", dict(fov=-1.0)),
    ("fov NaN", dict(fov=math.nan)),
    ("aspect 0", dict(aspect=0.0)),
    ("aspect -1", dict(aspect=-1.0)),
    ("near 0", dict(near=0.0)),
    ("near -1", dict(near=-1.0)),
    ("far == near", dict(near=2.0, far=2.0)),
    ("far < near", dict(near=2.0, far=1.0)),
    ("far inf", dict(far=math.inf)),
    ("eye == target", dict(fixed_position=(1.0, 2.0, 3.0), look_at=(1.0, 2.0, 3.0))),
    ("looking up", dict(fixed_position=(1.0, 2.0, 3.0), look_at=(1.0, 50.0, 3.0))),
    ("looking down", dict(fixed_position=(0.0, 0.0, 0.0), look_at=(0.0, -1e-300, 0.0))),
    ("eye - target overflows", dict(fixed_position=(1e308, 0.0, 0.0), look_at=(-1e308, 0.0, 0.0))),
]


def base_control(**kw):
    d = dict(camera=None, scaling=1.0, fixed_position=(0.0, 0.0, 0.0), look_at=(0.0, 0.0, -1.0), screen_height=20.0,
             damping=1.0, fov=45.0, aspect=1.5, near=1.0, far=100.0)
    d.update(kw)
    return _lib.CameraControl(d["camera"], d["scaling"], d["fixed_position"], d["look_at"], d["screen_height"],
                              d["damping"], d["fov"], d["aspect"], d["near"], d["far"])


@pytest.mark.parametrize("name,kw", REJECT, ids=[r[0] for r in REJECT])
def test_rejections(st, name, kw):
    """the checks of ht_tracker_set_camera (camera_ctl_make); the mirror's look_at rejects the same lookAts"""
    L = selftest(st)
    cam = _lib.Camera()
    assert L.ht_selftest_camera(C.byref(base_control(**kw)), 0, 0.0, 0.0, 0.0, C.byref(cam)) == -1
    if "look_at" in kw and "fixed_position" in kw:
        with pytest.raises(ValueError):
            controllers.look_at(kw["fixed_position"], kw["look_at"])


def test_accepted_edges(st):
    """what the checks let through: scaling 0 and negative, damping 0, a nearly vertical view, fov just inside"""
    L = selftest(st)
    cam = _lib.Camera()
    for kw in (dict(scaling=0.0), dict(scaling=-2.0), dict(damping=0.0), dict(fov=1e-6), dict(fov=179.999),
               dict(fixed_position=(0.0, 0.0, 0.0), look_at=(1e-9, -1.0, 0.0)), dict(near=1e-9, far=2e-9)):
        assert L.ht_selftest_camera(C.byref(base_control(**kw)), 0, 0.0, 0.0, 0.0, C.byref(cam)) == 0, kw
