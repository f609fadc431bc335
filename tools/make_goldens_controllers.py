#!/usr/bin/env python
"""Golden cameras of the reference's head-coupled controller, headtrackr.controllers.three.
realisticAbsoluteCameraControl (src/controllers.js:28-68), executed by oracle/jsmini.py on top of the unmodified
src/main.js and the sources under it -> tests/golden/reference_js_controllers.json.

The harness is that of tools/make_goldens_lifecycle.py (a canvas shim as the <video> element, recorded timers,
`it.now_ms` as the clock, the actions tick / start / stop).  Two additions:

  * `document.addEventListener(type, fn)`: jsmini's document only logs what main.js dispatches; here dispatchEvent
    also calls the listeners of the event's type with the live event, as a browser does.  Each case has its own
    listener list, as each page has its own document.
  * the camera is a recording shim of a three.js r48 PerspectiveCamera: `position` {x, y, z}, `aspect`, `fov`,
    `lookAt(v)` and `setViewOffset(fullWidth, fullHeight, x, y, width, height)` (both recorded), and
    `updateProjectionMatrix()`, which records the values it is called with.  No THREE global is needed.

Cases (the frame sequences of the main, params and debug goldens):
  defaults          the main.js stream (160x120): found, tracked, lost -> "redetecting", found again; the reference's
                    defaults (screenHeight 20, damping 1), scaling 1
  damped            the same stream, damping 0.5, screenHeight 30, scaling 0.37, an off-centre fixedPosition
  angles_200x150    calcAngles, cameraOffset 5 (reference_js_params.json): head x > 0 and y < 0
  portrait_120x160  calcAngles, cameraOffset 5, fov 60, no smoothing (reference_js_params.json), a portrait camera
  no_retry_stop     retryDetection: false with stop() / start() (reference_js_debug.json): the camera survives both

Each step records the action and frame, the tick's headtrackingEvent {x, y, z} (or null) and the camera after the
tick: position, fov, the view offset (null before the first event) and `events`, the updateProjectionMatrix calls so
far.  Each case records the constructed camera.  Both sides of each ternary of the listener (x > 0, x <= 0, y < 0,
y >= 0) are asserted to be taken somewhere in the corpus.
"""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import make_goldens_debug as dg  # noqa: E402
import make_goldens_lifecycle as lg  # noqa: E402
import make_goldens_main as mg  # noqa: E402
import make_goldens_params as pg  # noqa: E402
from oracle import jsmini  # noqa: E402

REF = mg.REF
OUT = ROOT / "tests" / "golden" / "reference_js_controllers.json"


def cases():
    """-> [(name, tracker params, (W, H, frames), control, camera, [(action, kind, t)])].  frames: "main" (the 160x120
    frames of make_goldens_lifecycle.make_frame) or "params" (make_goldens_params.make_frame at W x H).  control: the
    controller's arguments (params None: the call passes no params object); camera: the camera's own fov, aspect,
    near, far."""
    main = [("start" if n == 0 else "tick", kind, t) for n, (kind, t) in enumerate(mg.stream_frames())]
    stop = dict((c[0], c[3]) for c in dg.cases())["no_retry_stop"]
    prm = {c[0]: c[1] for c in pg.cases()}
    cam = lambda fov, aspect: dict(fov=fov, aspect=aspect, near=1.0, far=10000.0)
    return [
        ("defaults", {}, (160, 120, "main"),
         dict(scaling=1.0, fixedPosition=[0.0, 0.0, 0.0], lookAt=[0.0, 0.0, -1.0], params=None), cam(75.0, 4 / 3), main),
        ("damped", {}, (160, 120, "main"),
         dict(scaling=0.37, fixedPosition=[1.5, -2.0, 40.0], lookAt=[0.0, 0.0, 0.0],
              params=dict(screenHeight=30.0, damping=0.5)), cam(60.0, 16 / 9), main),
        ("angles_200x150", prm["angles_200x150"], (200, 150, "params"),
         dict(scaling=2.5, fixedPosition=[0.0, 10.0, 0.0], lookAt=[3.0, 10.0, -50.0], params=dict(damping=1.0)),
         cam(45.0, 4 / 3), pg.case_spec()),
        ("portrait_120x160", prm["portrait_120x160"], (120, 160, "params"),
         dict(scaling=1.0, fixedPosition=[-4.0, 0.0, 25.0], lookAt=[0.0, -1.0, 0.0], params=dict(screenHeight=25.0)),
         cam(50.0, 0.75), pg.case_spec()),
        ("no_retry_stop", {"retryDetection": False}, (160, 120, "main"),
         dict(scaling=1.0, fixedPosition=[0.0, 0.0, 0.0], lookAt=[0.0, 0.0, -1.0], params=None), cam(75.0, 4 / 3), stop),
    ]


def make_frame(frames, kind, t, W, H):
    return lg.make_frame(kind, t) if frames == "main" else pg.make_frame(kind, t, W, H)


class CameraShim(jsmini.JSObject):
    """a three.js r48 PerspectiveCamera as far as src/controllers.js:40-65 uses it, recording what it is called with"""

    def __init__(self, fov, aspect):
        jsmini.JSObject.__init__(self)
        pos = jsmini.JSObject()
        pos.props.update(x=0.0, y=0.0, z=0.0)
        self.props.update(position=pos, fov=fov, aspect=aspect)
        self.look_at = []
        self.view = None
        self.updates = []
        num = jsmini.to_number
        self.props["lookAt"] = jsmini.NativeFunction(
            lambda this, a: self.look_at.append([num(a[0].get(k)) for k in "xyz"]) or jsmini.undefined)
        self.props["setViewOffset"] = jsmini.NativeFunction(lambda this, a: self._set_view([num(v) for v in a[:6]]))
        self.props["updateProjectionMatrix"] = jsmini.NativeFunction(lambda this, a: self._update())

    def _set_view(self, v):
        self.view = v
        return jsmini.undefined

    def state(self):
        p = self.props["position"]
        return dict(position=[jsmini.to_number(p.get(k)) for k in "xyz"], fov=jsmini.to_number(self.props["fov"]),
                    view=self.view, events=len(self.updates))

    def _update(self):
        s = self.state()
        s["events"] += 1                # this call is the camera's events-th update
        self.updates.append(s)
        return jsmini.undefined


def with_listeners(it):
    """document.addEventListener, and a dispatchEvent that calls the listeners of the event's type with the live
    event after logging it.  -> the listener list ([(type, fn)]; a case clears it)."""
    doc = it.get(["document"])
    listeners = []
    log = doc.props["dispatchEvent"]

    def add(this, a):
        listeners.append((a[0], a[1]))
        return jsmini.undefined

    def dispatch(this, a):
        log_result = jsmini.call_function(log, this, a)
        for typ, fn in list(listeners):
            if typ == a[0].get("type"):
                jsmini.call_function(fn, doc, [a[0]])
        return log_result
    doc.props["addEventListener"] = jsmini.NativeFunction(add)
    doc.props["dispatchEvent"] = jsmini.NativeFunction(dispatch)
    return listeners


def js_literal(v):
    if isinstance(v, dict):
        return "{" + ", ".join(f"{k}: {js_literal(x)}" for k, x in v.items()) + "}"
    if isinstance(v, list):
        return "[" + ", ".join(js_literal(x) for x in v) + "]"
    return repr(float(v))


def main():
    it = jsmini.Interpreter()
    it.run(mg.cut_main())
    it.run("headtrackr.headposition = {};")
    for f in ("ccv.js", "cascade.js", "camshift.js", "whitebalance.js", "facetrackr.js", "smoother.js", "headposition.js",
              "controllers.js"):
        it.run((REF / f).read_text())
    listeners = with_listeners(it)
    out = []
    sides = set()
    for name, params, (W, H, frames), control, camera, spec in cases():
        t_case = time.time()
        listeners.clear()
        p = jsmini.JSObject()
        p.props["ui"] = False
        for k, v in params.items():
            p.props[k] = v
        video = jsmini.CanvasShim(make_frame(frames, *spec[0][1:], W, H).copy())
        video.props.update(currentTime=1.0, paused=False, ended=False)
        canvas = jsmini.CanvasShim(np.zeros((H, W, 4), np.uint8))
        cam = CameraShim(camera["fov"], camera["aspect"])
        it.genv.vars["camera_"] = cam
        la = control["lookAt"]
        args = [js_literal(control["scaling"]), js_literal(control["fixedPosition"]),
                "{x: %s, y: %s, z: %s}" % tuple(js_literal(v) for v in la)]
        if control["params"] is not None:
            args.append(js_literal(control["params"]))
        it.run("headtrackr.controllers.three.realisticAbsoluteCameraControl(camera_, %s);" % ", ".join(args))
        assert cam.look_at == [la] and len(listeners) == 1
        constructed = cam.state()
        ht = it.get(["headtrackr", "Tracker"]).construct([p])
        it.events.clear()
        it.timers.clear()
        it.call(ht.get("init"), ht, video, canvas, False)
        steps = []
        for n, (action, kind, t) in enumerate(spec):
            video.pix = make_frame(frames, kind, t, W, H).copy()
            it.now_ms += 35.0
            n0, u0 = len(it.events), len(cam.updates)
            if action == "start":
                assert it.call(ht.get("start"), ht) is True
            elif action == "stop":
                it.call(ht.get("stop"), ht)
            else:
                live = [tm for tm in it.timers if not tm[3]]
                if live:
                    tm = live[-1]
                    tm[3] = True
                    it.call(tm[1])
            heads = [mg.event_record(e) for e in it.events[n0:] if e.get("type") == "headtrackingEvent"]
            assert len(heads) <= 1 and len(cam.updates) - u0 == len(heads)
            head = [heads[0][k] for k in "xyz"] if heads else None
            if head:
                sides.add("x>0" if head[0] > 0 else "x<=0")
                sides.add("y<0" if head[1] < 0 else "y>=0")
                assert cam.updates[-1] == cam.state()
            steps.append(dict(action=action, frame=[kind, t], status=ht.get("status"), head=head, camera=cam.state()))
            print(name, n, action, kind, t, ht.get("status"), head, flush=True)
        assert any(s["head"] for s in steps), name
        out.append(dict(name=name, params=params, width=W, height=H, frames=frames, ms_per_frame=35.0, control=control,
                        camera=camera, constructed=constructed, steps=steps))
        print(name, "took %.0f s" % (time.time() - t_case), flush=True)
    assert sides == {"x>0", "x<=0", "y<0", "y>=0"}, sides
    OUT.write_text(json.dumps(dict(generator="tools/make_goldens_controllers.py (src/main.js and src/controllers.js "
                                             "executed by oracle/jsmini.py)", cases=out), indent=1))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
