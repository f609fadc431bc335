"""GPU: the head-coupled camera of each headtrackr.Tracker stream (ht_tracker_set_camera, realisticAbsoluteCameraControl
of src/controllers.js run by the device during the tick):

  * every case of the reference's own controllers.js (reference_js_controllers.json) through TrackerSet.step (one
    context per canvas size) and TrackerSet.feed (all sizes in one context), with a stream without a controller
    beside them: after every tick the ht_camera equals the reference's camera, and the records are byte-identical
    to a context without controllers;
  * persistence across ticks without a headtrackingEvent, stop / start / reset and a lost face; ht_tracker_config
    removes every controller; ht_tracker_import and a swap leave each controller with its stream id;
  * 1024 streams of 640x480 with random controls, against the host mirror applied to the drained records;
  * a camera in a slice of a larger tensor, the bytes around it unchanged; the launch count; rejections.

The device's head positions are the tracker's own: its headposition epilogue takes tan / atan from CUDA's libm, so
they may differ from the reference's in the last bits (the GPU tracker tests compare them to 1e-9 relative).  So each
camera is checked twice: against the reference's camera to the same 1e-9 relative, with the same event count and view
offset flag; and against the host mirror (controllers.py, bit-identical to the reference's listener on the CPU) fed
with the device's own drained records, within the bounds below.

Bounds.  position, the view offset, events and has_view_offset are fp64 arithmetic without libm: bit-identical.
fov = atan(q) * 360 / PI: CUDA documents atan's error as 2 ulp, so the device's atan(q) is within a relative
2 * 2^-52 of the host's (the reference's, jsmini's Math.atan is the host libm); the two roundings that follow add at
most 2^-53 each, so fov is within a relative 5 * 2^-53 (2.5 * 2^-52) of the reference's: FOV_ULPS = 5 ulp of fov.
The matrices go through tan (CUDA: 2 ulp) and are rounded once to float32, whose ulp is 2^29 times fp64's: they are
within 1 float32 ulp of the host restatement (controllers.py, DESIGN.md 5.4 f10)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, controllers, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE
from headtrackr_b200.context import camera_from_bytes
from headtrackr_b200.streams import TrackerSet
from test_controllers_host import CASES, make_frame, same_bits
from test_gpu_feed import equal_records
from test_host_main import same

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
FOV_ULPS = 5
NB = _lib.CAMERA_BYTES


def torch():
    import torch as t
    return t


def ulps64(a, b):
    if a == b or (a != a and b != b):
        return 0
    ia, ib = (int(np.array([v], np.float64).view(np.int64)[0]) for v in (a, b))
    return abs(ia - ib) if (ia < 0) == (ib < 0) else 1 << 62


def within_1ulp_f32(a, b):
    a, b = np.asarray(a, np.float32).ravel(), np.asarray(b, np.float32).ravel()
    if not (np.isfinite(a) == np.isfinite(b)).all():
        return False
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    both_zero = (a == 0) & (b == 0)
    return bool(((np.abs(ia - ib) <= 1) & (np.sign(a) * np.sign(b) >= 0) | both_zero).all())


def check_device_camera(got, want, proj, view, where):
    """got: camera_from_bytes of the device camera; want: a reference camera record (position, fov, view, events)"""
    assert same_bits(got["position"], want["position"]), (where, got["position"], want["position"])
    assert got["events"] == want["events"], where
    if want["view"] is None:
        assert got["has_view_offset"] == 0 and same_bits(got["view"], [0.0] * 6), where
    else:
        assert got["has_view_offset"] == 1 and same_bits(got["view"], want["view"]), where
    assert ulps64(got["fov"], want["fov"]) <= FOV_ULPS, (where, got["fov"], want["fov"])
    assert within_1ulp_f32(got["projection"], proj), (where, got["projection"], proj)
    assert within_1ulp_f32(got["view_matrix"], view), (where, got["view_matrix"], view)


def near_reference(got, want, where):
    """the device camera against the reference's: the head positions it was moved by agree to 1e-9 relative"""
    assert got["events"] == want["events"] and got["has_view_offset"] == int(want["view"] is not None), where
    for a, b in zip(got["position"] + [got["fov"]] + got["view"], want["position"] + [want["fov"]]
                    + (want["view"] or [0.0] * 6)):
        assert same(a, b), (where, got, want)


def camera_dict(case, out):
    c, k = case["control"], case["camera"]
    d = dict(scaling=c["scaling"], fixedPosition=c["fixedPosition"], lookAt=c["lookAt"], fov=k["fov"],
             aspect=k["aspect"], near=k["near"], far=k["far"], out=out)
    d.update(c["params"] or {})
    return d


def black(w, h):
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 3] = 255
    return f


# ---- the reference's runs -------------------------------------------------------------------------------------------

def replay(cases, path):
    """cases (+ a copy of cases[0] without a controller) on one context, against one without controllers"""
    T = torch()
    n = len(cases) + 1
    W, H = max(c["width"] for c in cases), max(c["height"] for c in cases)
    streams = list(cases) + [cases[0]]
    buf = T.zeros(n * NB, dtype=T.uint8, device="cuda")
    outs = [buf[NB * k: NB * (k + 1)] for k in range(n)]
    c = Context(max_width=W, max_height=H, max_frames=n)
    ref = Context(max_width=W, max_height=H, max_frames=n)
    try:
        ts = TrackerSet(c, n, [dict(case["params"], camera=camera_dict(case, outs[k]) if k < n - 1 else None)
                               for k, case in enumerate(streams)])
        tr = TrackerSet(ref, n, [case["params"] for case in streams])
        mirrors = [Mirror(camera_dict(case, None)) for case in cases]
        for k, case in enumerate(cases):
            mirrors[k].check(outs[k], (case["name"], "constructed"))
            near_reference(camera_from_bytes(outs[k]), case["constructed"], (case["name"], "constructed"))
        assert not outs[-1].any()
        clock = 1.0e12
        events = 0
        for i in range(max(len(case["steps"]) for case in streams)):
            clock += 35.0
            frames, listed = [], []
            for k, case in enumerate(streams):
                f = black(case["width"], case["height"])
                if i < len(case["steps"]):
                    s = case["steps"][i]
                    f = make_frame(case, *s["frame"])
                    if s["action"] == "start":
                        ts.start(k), tr.start(k)
                    elif s["action"] == "stop":
                        ts.stop(k), tr.stop(k)
                    if s["action"] != "stop":
                        listed.append(k)
                elif i == len(case["steps"]):
                    ts.stop(k), tr.stop(k)
                frames.append(f)
            recs = {}
            if path == "step":
                batch = T.from_numpy(np.stack(frames)).cuda()
                T.cuda.synchronize()
                got = ts.step(batch, clock)
                assert equal_records(got, tr.step(batch, clock)), i
                recs = dict(enumerate(got))
            elif listed:
                vids = {k: T.from_numpy(frames[k]).cuda() for k in listed}
                wh = ({k: streams[k]["width"] for k in listed}, {k: streams[k]["height"] for k in listed})
                T.cuda.synchronize()
                recs = ts.feed(vids, clock, *wh)
                assert equal_records(recs, tr.feed(vids, clock, *wh)), i
            for k, case in enumerate(cases):
                if k in recs:
                    mirrors[k].feed(recs[k])
                mirrors[k].check(outs[k], (case["name"], i))
                if i < len(case["steps"]):
                    near_reference(camera_from_bytes(outs[k]), case["steps"][i]["camera"], (case["name"], i))
            events += sum(case["steps"][i]["head"] is not None for case in cases if i < len(case["steps"]))
        assert not outs[-1].any()
        assert events == sum(case["steps"][-1]["camera"]["events"] for case in cases) > 0
    finally:
        c.close()
        ref.close()


@pytest.mark.parametrize("size", sorted({(c["width"], c["height"]) for c in CASES}), ids=lambda s: "%dx%d" % s)
def test_golden_replay_step(size):
    replay([c for c in CASES if (c["width"], c["height"]) == size], "step")


def test_golden_replay_feed():
    replay(CASES, "feed")


# ---- lifetime ---------------------------------------------------------------------------------------------------------

def face(t, W=160, H=120):
    import make_goldens_params as pg
    return pg.make_frame("face", t, W, H)


def empty(W=160, H=120):
    import make_goldens_params as pg
    return pg.make_frame("empty", 0, W, H)


CONTROL = dict(scaling=0.8, fixedPosition=[1.0, 2.0, 30.0], lookAt=[0.0, 0.0, 0.0], screenHeight=25.0, damping=0.7,
               fov=55.0, aspect=1.25, near=0.5, far=500.0)


class Mirror:
    """controllers.py's camera for one stream, fed with the stream's drained records"""

    def __init__(self, d=CONTROL):
        self.cam = controllers.PerspectiveCamera(d["fov"], d["aspect"], d["near"], d["far"])
        self.ctl = controllers.realisticAbsoluteCameraControl(
            self.cam, d["scaling"], d["fixedPosition"], d["lookAt"],
            dict(screenHeight=d.get("screenHeight", 20.0), damping=d.get("damping", 1.0)))

    def feed(self, rec):
        h = rec["head"]
        if h["valid"]:
            self.ctl.handleEvent(h)

    def check(self, out, where):
        s = self.ctl.state()
        want = dict(position=s["position"], fov=s["fov"], view=s["view"] if s["has_view_offset"] else None,
                    events=s["events"])
        check_device_camera(camera_from_bytes(out), want, s["projection"], s["view_matrix"], where)


def test_persistence_stop_start_reset_lost_face_and_config():
    T = torch()
    ctx = Context(max_width=160, max_height=120, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        out = T.zeros(NB, dtype=T.uint8, device="cuda")
        ctx.tracker_set_camera(0, [dict(CONTROL, out=out)])
        m = Mirror()
        m.check(out, "constructed")
        plan = [("tick", face(t)) for t in range(26)] + [("tick", empty())] * 4 + [("tick", face(t)) for t in range(40, 52)]
        plan += [("stop", None), ("tick", face(52)), ("tick", face(53)), ("start", None)]
        plan += [("tick", face(t)) for t in range(54, 70)] + [("reset", None), ("tick", face(70)), ("start", None)]
        plan += [("tick", face(t)) for t in range(71, 100)]
        quiet, moved, kinds = 0, 0, set()
        for n, (what, f) in enumerate(plan):
            if what != "tick":
                {"stop": ctx.tracker_stop, "start": ctx.tracker_start, "reset": ctx.tracker_reset}[what](0, 1)
                continue
            before = out.clone()
            rec = ctx.tracker_feed([0, 1], [f, f], 1.0e12 + 35.0 * n, 160, 120)[0]
            kinds.add(rec["detection"])
            m.feed(rec)
            if rec["head"]["valid"]:
                moved += 1
            else:
                assert T.equal(out, before), n                 # no headtrackingEvent: the camera is as it was
                quiet += 1
            m.check(out, n)
        assert moved > 20 and quiet > 20 and {"WB", "VJ", "CS"} <= kinds
        # the controller survived the lost face, stop, start and reset: events after each of them
        assert camera_from_bytes(out)["events"] == m.ctl.events
        ctx.tracker_set_params(0, [dict(calcAngles=True)])     # keeps the controller
        before = camera_from_bytes(out)["events"]
        for t in range(100, 104):
            m.feed(ctx.tracker_feed([0], [face(t)], 1.0e12 + 35.0 * t, 160, 120)[0])
        m.check(out, "set_params")
        assert camera_from_bytes(out)["events"] > before
        ctx.tracker_config()                                   # removes every controller
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        out.fill_(0x77)
        T.cuda.synchronize()
        for t in range(40):
            ctx.tracker_feed([0], [face(t)], 2.0e12 + 35.0 * t, 160, 120)
        assert (out == 0x77).all()
    finally:
        ctx.close()


def test_set_again_reconstructs_and_none_removes():
    T = torch()
    ctx = Context(max_width=160, max_height=120, max_frames=1)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        out = T.zeros(NB, dtype=T.uint8, device="cuda")
        ctx.tracker_set_camera(0, [dict(CONTROL, out=out)])
        for t in range(30):
            ctx.tracker_feed([0], [face(t)], 1.0e12 + 35.0 * t, 160, 120)
        assert camera_from_bytes(out)["events"] > 0
        ctx.tracker_set_camera(0, [dict(CONTROL, out=out)])
        Mirror().check(out, "re-constructed")
        ctx.tracker_set_camera(0, [None])
        snap = out.clone()
        valid = sum(ctx.tracker_feed([0], [face(t)], 1.0e12 + 35.0 * t, 160, 120)[0]["head"]["valid"]
                    for t in range(30, 36))
        assert valid > 0 and T.equal(out, snap)
    finally:
        ctx.close()


def test_import_and_swap_leave_the_controller_with_the_id():
    T = torch()
    ctx = Context(max_width=160, max_height=120, max_frames=3)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 3)
        ctx.tracker_start(0, 2)                                 # stream 2 stays idle
        outs = [T.zeros(NB, dtype=T.uint8, device="cuda") for _ in range(2)]
        d1 = dict(CONTROL, scaling=1.3, fixedPosition=[-5.0, 0.0, 10.0], lookAt=[0.0, 1.0, -20.0])
        ctx.tracker_set_camera(0, [dict(CONTROL, out=outs[0]), dict(d1, out=outs[1])])
        mir = [Mirror(), Mirror(d1)]
        t = 0
        for t in range(30):                                     # stream 1 starts 10 ticks later: different states
            ks = [0, 1] if t >= 10 else [0]
            recs = ctx.tracker_feed(ks, [face(t)] * len(ks), 1.0e12 + 35.0 * t, 160, 120)
            for k, r in zip(ks, recs):
                mir[k].feed(r)
        recs = ctx.tracker_export([0, 1])
        ctx.tracker_import([1, 0], recs)                        # swap the Trackers; the controllers stay with the ids
        ctx.tracker_import([2], recs[:1])                       # a clone of stream 0 in idle stream 2, no controller
        for t in range(30, 50):
            got = ctx.tracker_feed([0, 1, 2], [face(t)] * 3, 1.0e12 + 35.0 * t, 160, 120)
            for k in range(2):
                mir[k].feed(got[k])
                mir[k].check(outs[k], (t, k))
            assert got[2]["head"] == got[1]["head"]            # the clone follows the Tracker now in slot 1
        assert all(camera_from_bytes(o)["events"] > 10 for o in outs)
    finally:
        ctx.close()


# ---- scale, layout, launches ------------------------------------------------------------------------------------------

def test_1024_streams_640x480_random_controls():
    T = torch()
    n, W, H = 1024, 640, 480
    rng = np.random.default_rng(41)
    frames = [T.from_numpy(synth.frame(900 + i, W, H, n_faces=1)).cuda() for i in range(16)]
    buf = T.zeros(n * NB, dtype=T.uint8, device="cuda")
    order = rng.permutation(n)                                  # camera k at slot order[k] of one buffer
    ctrl = [None] * n
    for k in range(n):
        if rng.random() < 0.9:
            look = rng.normal(size=3) * 40
            ctrl[k] = dict(scaling=float(rng.uniform(0.1, 4)), fixedPosition=list(rng.normal(size=3) * 20),
                           lookAt=[float(look[0]), float(look[1]), float(look[2]) - 60.0],
                           screenHeight=float(rng.uniform(10, 40)), damping=float(rng.uniform(0, 1.5)),
                           fov=float(rng.uniform(20, 120)), aspect=float(rng.uniform(0.5, 2.5)),
                           near=float(rng.uniform(0.1, 2)), far=float(rng.uniform(100, 5000)))
    outs = [buf[NB * int(order[k]): NB * (int(order[k]) + 1)] for k in range(n)]
    ctx = Context(max_width=W, max_height=H, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        ctx.tracker_set_camera(0, [dict(d, out=outs[k]) if d else None for k, d in enumerate(ctrl)])
        mir = [Mirror(d) if d else None for d in ctrl]
        clock = [1.0e12 + 13.0 * k for k in range(n)]
        for tick in range(50):
            ks = [k for k in range(n) if rng.random() < 0.85]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            recs = ctx.tracker_feed(ks, [frames[k % 16] for k in ks], [clock[k] for k in ks], W, H)
            for k, rec in zip(ks, recs):
                if mir[k]:
                    mir[k].feed(rec)
        host = buf.cpu()
        for k in range(n):
            if mir[k]:
                mir[k].check(host[NB * int(order[k]): NB * (int(order[k]) + 1)], k)
            else:
                assert not host[NB * int(order[k]): NB * (int(order[k]) + 1)].any()
        assert sum(m.ctl.events for m in mir if m) > 5 * n
    finally:
        ctx.close()


def test_camera_in_a_slice_of_a_larger_tensor():
    T = torch()
    big = T.full((4096,), 0x5A, dtype=T.uint8, device="cuda")
    out = big[1040: 1040 + NB]                                  # 16-byte aligned inside a renderer's buffer
    ctx = Context(max_width=160, max_height=120, max_frames=1)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        ctx.tracker_set_camera(0, [dict(CONTROL, out=out)])
        m = Mirror()
        for t in range(40):
            m.feed(ctx.tracker_feed([0], [face(t)], 1.0e12 + 35.0 * t, 160, 120)[0])
        m.check(out, "slice")
        assert m.ctl.events > 5
        assert (big[:1040] == 0x5A).all() and (big[1040 + NB:] == 0x5A).all()
    finally:
        ctx.close()


def test_launch_count():
    T = torch()
    a = Context(max_width=160, max_height=120, max_frames=4)
    b = Context(max_width=160, max_height=120, max_frames=4)
    try:
        for x in (a, b):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        outs = [T.zeros(NB, dtype=T.uint8, device="cuda") for _ in range(2)]
        for t in range(40):
            if t == 10:
                b.tracker_set_camera(1, [dict(CONTROL, out=o) for o in outs])
            if t == 30:
                b.tracker_set_camera(1, [None, None])
            la, lb = a.launch_count, b.launch_count
            ra = a.tracker_feed(range(4), [face(t)] * 4, 1.0e12 + 35.0 * t, 160, 120)
            rb = b.tracker_feed(range(4), [face(t)] * 4, 1.0e12 + 35.0 * t, 160, 120)
            assert equal_records(ra, rb)
            extra = 1 if 10 <= t < 30 else 0                    # k_camera_update
            assert b.launch_count - lb == a.launch_count - la + extra, t
        assert all(camera_from_bytes(o)["events"] > 0 for o in outs)
    finally:
        a.close()
        b.close()


# ---- rejections ---------------------------------------------------------------------------------------------------------

def raw(ctx, first, recs, null=False):
    arr = (_lib.CameraControl * max(1, len(recs)))(*recs)
    return ctx._L.ht_tracker_set_camera(ctx._h, first, len(recs), None if null else C.addressof(arr))


def cc(ptr, **kw):
    d = dict(scaling=1.0, fixed_position=(0.0, 0.0, 10.0), look_at=(0.0, 0.0, 0.0), screen_height=20.0, damping=1.0,
             fov=45.0, aspect=1.5, near=1.0, far=100.0)
    d.update(kw)
    return _lib.CameraControl(ptr, d["scaling"], d["fixed_position"], d["look_at"], d["screen_height"], d["damping"],
                              d["fov"], d["aspect"], d["near"], d["far"])


def test_rejections_change_nothing():
    T = torch()
    mf = 3
    ctx = Context(max_width=160, max_height=120, max_frames=mf)
    buf = T.zeros(8 * NB, dtype=T.uint8, device="cuda")
    base = buf.data_ptr()
    host = np.zeros(2 * NB, np.uint8)
    try:
        assert raw(ctx, 0, [cc(base)]) == HT_ERR_STATE
        ctx.tracker_config()
        ctx.tracker_reset(0, mf)
        ctx.tracker_start(0, mf)
        assert raw(ctx, 0, [cc(base), cc(None), cc(base + 4 * NB)]) == 0
        for t in range(30):
            ctx.tracker_feed(range(mf), [face(t)] * mf, 1.0e12 + 35.0 * t, 160, 120)
        T.cuda.synchronize()
        free = base + 6 * NB
        nan, inf = float("nan"), float("inf")
        cases = [
            ("range", -1, [cc(free)]),
            ("empty", 0, []),
            ("past max_frames", 2, [cc(free), cc(free + NB)]),
            ("host memory", 1, [cc(host.ctypes.data)]),
            ("misaligned", 1, [cc(free + 8)]),
            ("overlaps stream 0", 1, [cc(base + NB - 16)]),
            ("overlaps stream 2", 1, [cc(base + 4 * NB - 16)]),
            ("two records share bytes", 0, [cc(free), cc(free + NB - 16)]),
            ("scaling NaN", 1, [cc(free, scaling=nan)]),
            ("damping inf", 1, [cc(free, damping=inf)]),
            ("lookAt NaN", 1, [cc(free, look_at=(nan, 0.0, 0.0))]),
            ("fov 0", 1, [cc(free, fov=0.0)]),
            ("fov 180", 1, [cc(free, fov=180.0)]),
            ("aspect 0", 1, [cc(free, aspect=0.0)]),
            ("near 0", 1, [cc(free, near=0.0)]),
            ("far <= near", 1, [cc(free, near=5.0, far=5.0)]),
            ("eye == target", 1, [cc(free, look_at=(0.0, 0.0, 10.0))]),
            ("view parallel to up", 1, [cc(free, look_at=(0.0, 40.0, 10.0))]),
            ("a later record is bad", 1, [cc(free), cc(free + NB, fov=-3.0)]),
        ]
        if T.cuda.device_count() > 1:
            other = T.zeros(NB, dtype=T.uint8, device="cuda:1")
            cases.append(("another device", 1, [cc(other.data_ptr())]))
        for name, first, recs in cases:
            cams = buf.clone()
            states = ctx.tracker_export(list(range(mf)))
            assert raw(ctx, first, recs) == HT_ERR_ARG, (name, ctx._L.ht_last_error(ctx._h))
            T.cuda.synchronize()
            assert T.equal(buf, cams), name
            assert np.array_equal(ctx.tracker_export(list(range(mf))), states), name
        assert raw(ctx, 0, [cc(free)], null=True) == HT_ERR_ARG
        # nothing was replaced: streams 0 and 2 still move their cameras, stream 1 still has none
        ev = [camera_from_bytes(buf[NB * i: NB * (i + 1)])["events"] for i in (0, 4)]
        for t in range(30, 36):
            recs = ctx.tracker_feed(range(mf), [face(t)] * mf, 1.0e12 + 35.0 * t, 160, 120)
            ev = [e + recs[k]["head"]["valid"] for e, k in zip(ev, (0, 2))]
        assert [camera_from_bytes(buf[NB * i: NB * (i + 1)])["events"] for i in (0, 4)] == ev and ev[0] > 6
        assert not buf[NB: 4 * NB].any() and not buf[5 * NB:].any()
        # a camera may take the gap between two others, and replace its own stream's
        assert raw(ctx, 1, [cc(base + 2 * NB)]) == 0
        assert raw(ctx, 0, [cc(base)]) == 0
    finally:
        ctx.close()


def test_cameras_and_images_share_no_byte():
    """A camera is bytes the tick writes, like a debug canvas, a face crop or a face tensor: a camera on any of them,
    and any of them on a camera, is refused, and the outputs in force stay as they were."""
    T = torch()
    mf = 4
    ctx = Context(max_width=160, max_height=120, max_frames=mf)
    buf = T.zeros(64 * NB, dtype=T.uint8, device="cuda")
    base = buf.data_ptr()
    regions = [(0, 1024), (2048, 3072), (4096, 5120), (8192, 8192 + NB)]     # canvas, crop, tensor, camera
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, mf)
        ctx.tracker_start(0, mf)
        ctx.tracker_set_debug(0, [buf[0:1024].view(16, 16, 4)])
        ctx.tracker_set_face_crop(1, [dict(out=buf[2048:3072].view(16, 16, 4))])
        ctx.tracker_set_face_tensor(2, [dict(out=buf[4096:5120].view(T.float32).view(1, 16, 16), channels="gray")])
        ctx.tracker_set_camera(3, [dict(CONTROL, out=buf[8192:8192 + NB])])
        for t in range(30):
            ctx.tracker_feed(range(mf), [face(t)] * mf, 1.0e12 + 35.0 * t, 160, 120)
        L, h = ctx._L, ctx._h
        canvas = (_lib.DebugCanvas * 1)(_lib.DebugCanvas(base + 8192 - 64, 8, 4, 0, 0))
        crop = (_lib.FaceCrop * 1)(_lib.FaceCrop(base + 8192 + NB - 32, 4, 4, 0, 0, 1.0))
        tensor = (_lib.FaceTensor * 1)(_lib.FaceTensor(base + 8192 - 32, 4, 0, 4, 4, _lib.HT_TENSOR_F32, _lib.HT_TENSOR_CHW,
                                                       _lib.HT_TENSOR_GRAY, 0, (1.0,) * 3, (0.0,) * 3, 1.0))
        cases = [
            ("camera on the canvas", lambda: raw(ctx, 0, [cc(base + 512)])),
            ("camera on the crop", lambda: raw(ctx, 0, [cc(base + 2048 + 512)])),
            ("camera on the tensor", lambda: raw(ctx, 0, [cc(base + 4096 + 1024 - 16)])),
            ("canvas on the camera", lambda: L.ht_tracker_set_debug(h, 3, 1, C.addressof(canvas))),
            ("crop on the camera", lambda: L.ht_tracker_set_face_crop(h, 1, 1, C.addressof(crop))),
            ("tensor on the camera", lambda: L.ht_tracker_set_face_tensor(h, 2, 1, C.addressof(tensor))),
        ]
        for name, call in cases:
            T.cuda.synchronize()
            before = buf.clone()
            assert call() == HT_ERR_ARG, (name, L.ht_last_error(h))
            assert "overlaps" in L.ht_last_error(h).decode(), name
            T.cuda.synchronize()
            assert T.equal(buf, before), name
        # every output still in force, and nothing written outside them
        events = camera_from_bytes(buf[8192:8192 + NB])["events"]
        buf[:8192].zero_()                                # the camera keeps its state
        buf[8192 + NB:].zero_()
        T.cuda.synchronize()
        for t in range(30, 36):
            ctx.tracker_feed(range(mf), [face(t)] * mf, 1.0e12 + 35.0 * t, 160, 120)
        T.cuda.synchronize()
        assert all(buf[a:b].any() for a, b in regions[:3])
        assert camera_from_bytes(buf[8192:8192 + NB])["events"] > events > 0
        outside = T.ones_like(buf, dtype=T.bool)
        for a, b in regions:
            outside[a:b] = False
        assert not buf[outside].any()
    finally:
        ctx.close()
