#!/usr/bin/env python
"""Golden event streams of headtrackr.Tracker's lifecycle (src/main.js) from its first frame, executed by
oracle/jsmini.py on top of the unmodified ccv / cascade / camshift / whitebalance / facetrackr / smoother /
headposition sources -> tests/golden/reference_js_lifecycle.json.

Same cut of main.js and the same harness as tools/make_goldens_main.py (a canvas shim as the <video> element,
`window.setTimeout` only records its callback, `it.now_ms` is the clock), driven by a per-frame action list:

  tick   fire the newest live timer, if there is one (the track() timer or the starter's retry)
  start  Tracker.start() - runs starter() on the current frame at once (the video is "playing")
  stop   Tracker.stop()

Each step records the events in dispatch order, `ht.status` and `getFOV()`.  Each case ends with one more stop().

  starter_black  all-black frames: the starter retries without events (also across a stop(), which does not cancel
                 the starter's timer); the first frame with content opens the whitebalance gate, then found
  wb_unstable    the frame brightness ramps by >= 2 gray levels per frame, then holds: the gate opens only after 15
                 samples within 2 levels
  no_retry       retryDetection: false - lost -> "lost" + "stopped", idle frames without events, start() again: a
                 fresh whitebalance gate, "found", and head positions at once (headposition, smoother and fov survive)
  hints          1000 ms per frame over face-free detection frames: "hints" after 5000 ms; a CS frame clears the
                 detection timer, stop() does not
"""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import make_goldens_main as mg  # noqa: E402
from oracle import jsmini  # noqa: E402

REF = mg.REF
OUT = ROOT / "tests" / "golden" / "reference_js_lifecycle.json"
W, H = mg.W, mg.H
RAMP = 20                     # wb_unstable: frames of the brightness ramp


def make_frame(kind, t):
    """kinds of make_goldens_main ("face", "empty") plus "black" (RGB 0, alpha 255) and "ramp" (frame t of a
    brightness ramp up to the face frame)"""
    if kind == "black":
        f = np.zeros((H, W, 4), np.uint8)
        f[..., 3] = 255
        return f
    if kind == "ramp":
        f = mg.make_frame("face", t).astype(np.int64)
        num = 100 - 2 * (RAMP - t)                       # gain 60% .. 98%: integer arithmetic, no clipping
        f[..., :3] = (f[..., :3] * num) // 100
        return f.astype(np.uint8)
    return mg.make_frame(kind, t)


def cases():
    """name -> (params, ms per frame, [(action, kind, t)])"""
    tick = lambda kind, ts: [("tick", kind, t) for t in ts]
    face = lambda a, b: tick("face", range(a, b))
    return [
        ("starter_black", {}, 35.0,
         [("start", "black", 0), ("tick", "black", 0), ("stop", "black", 0), ("tick", "black", 0)] + face(0, 19)),
        ("wb_unstable", {}, 35.0, [("start", "ramp", 0)] + tick("ramp", range(1, RAMP)) + face(0, 18)),
        ("no_retry", {"retryDetection": False}, 35.0,
         [("start", "face", 0)] + face(1, 28) + tick("empty", [0, 0, 0]) + [("start", "face", 40)] + face(41, 60)),
        ("hints", {}, 1000.0,
         [("start", "empty", 0)] + tick("empty", [0] * 21) + face(0, 2) + tick("empty", [0] * 3)
         + [("stop", "empty", 0), ("start", "empty", 0)] + tick("empty", [0] * 15)),
    ]


def whitebalance(f):
    return float(f[..., :3].astype(np.float64).mean(axis=(0, 1)).sum() / 3)


def main():
    ramp = [whitebalance(make_frame("ramp", t)) for t in range(RAMP)] + [whitebalance(make_frame("face", 0))]
    assert all(b - a >= 2 for a, b in zip(ramp, ramp[1:])), ramp
    it = jsmini.Interpreter()
    it.run(mg.cut_main())
    it.run("headtrackr.headposition = {};")
    for f in ("ccv.js", "cascade.js", "camshift.js", "whitebalance.js", "facetrackr.js", "smoother.js", "headposition.js"):
        it.run((REF / f).read_text())
    out = []
    for name, params, dt, spec in cases():
        t_case = time.time()
        p = jsmini.JSObject()
        p.props["ui"] = False
        for k, v in params.items():
            p.props[k] = v
        video = jsmini.CanvasShim(make_frame(*spec[0][1:]).copy())
        video.props.update(currentTime=1.0, paused=False, ended=False)
        canvas = jsmini.CanvasShim(np.zeros((H, W, 4), np.uint8))
        ht = it.get(["headtrackr", "Tracker"]).construct([p])
        it.events.clear()
        it.timers.clear()
        it.call(ht.get("init"), ht, video, canvas, False)
        steps = []
        for n, (action, kind, t) in enumerate(spec):
            video.pix = make_frame(kind, t).copy()
            it.now_ms += dt
            n0 = len(it.events)
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
            ev = [mg.event_record(e) for e in it.events[n0:]]
            steps.append(dict(action=action, frame=[kind, t], status=ht.get("status"), events=ev,
                              fov=it.call(ht.get("getFOV"), ht)))
            print(name, n, action, kind, t, ht.get("status"),
                  [(e.get("type"), e.get("status", e.get("detection", ""))) for e in ev], flush=True)
        n0 = len(it.events)
        it.call(ht.get("stop"), ht)
        out.append(dict(name=name, params=params, ms_per_frame=dt, steps=steps,
                        stop_events=[mg.event_record(e) for e in it.events[n0:]], fov=it.call(ht.get("getFOV"), ht)))
        print(name, "took %.0f s" % (time.time() - t_case), flush=True)
    OUT.write_text(json.dumps(dict(generator="tools/make_goldens_lifecycle.py (src/main.js executed by oracle/jsmini.py)",
                                   width=W, height=H, cases=out), indent=1))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
