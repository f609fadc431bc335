#!/usr/bin/env python
"""Golden event streams of headtrackr.Tracker (src/main.js) with non-default parameters on canvases other than
160x120, executed by oracle/jsmini.py on top of the unmodified ccv / cascade / camshift / whitebalance / facetrackr /
smoother / headposition sources -> tests/golden/reference_js_params.json.

Same cut of main.js, the same harness and the same 42-frame stream as tools/make_goldens_main.py (start() on frame
0, then the newest timer once per frame, 35 ms apart): a face is detected, tracked, lost (three empty frames ->
"redetecting" -> a fresh facetrackr) and found again.  Only the frame size changes: the frame generator draws the
synth face frame at each case's canvas size, and the <video> and the canvas both have that size.

  angles_200x150     calcAngles: true, cameraOffset: 5                     (the lost frame's angle is NaN)
  portrait_120x160   calcAngles: true, cameraOffset: 5, fov: 60, no smoothing   (a portrait canvas)
  no_head_200x150    headPosition: false, retryDetection: true (explicit), fov: 40

Each step records the action, the events in dispatch order, `ht.status` and `getFOV()`; each case ends with one
more stop().
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
from headtrackr_b200 import synth  # noqa: E402
from oracle import jsmini  # noqa: E402

REF = mg.REF
OUT = ROOT / "tests" / "golden" / "reference_js_params.json"


def cases():
    """name -> (params, width, height)"""
    return [
        ("angles_200x150", {"calcAngles": True, "cameraOffset": 5.0}, 200, 150),
        ("portrait_120x160", {"calcAngles": True, "cameraOffset": 5.0, "fov": 60.0, "smoothing": False}, 120, 160),
        ("no_head_200x150", {"headPosition": False, "retryDetection": True, "fov": 40.0}, 200, 150),
    ]


def make_frame(kind, t, W, H):
    """make_goldens_main.make_frame at W x H: the synth face frame, jittered by t; "empty" is a constant frame"""
    if kind == "empty":
        return synth.frame(0, W, H, kind="constant")
    base = synth.frame(3, W, H, n_faces=1)
    return np.roll(base, (t % 3, (2 * t) % 5), axis=(0, 1))


def case_spec():
    """[(action, kind, t)]: start() on the first frame, then one timer per frame"""
    return [("start" if n == 0 else "tick", kind, t) for n, (kind, t) in enumerate(mg.stream_frames())]


def main():
    it = jsmini.Interpreter()
    it.run(mg.cut_main())
    it.run("headtrackr.headposition = {};")
    for f in ("ccv.js", "cascade.js", "camshift.js", "whitebalance.js", "facetrackr.js", "smoother.js", "headposition.js"):
        it.run((REF / f).read_text())
    out = []
    for name, params, W, H in cases():
        t_case = time.time()
        p = jsmini.JSObject()
        p.props["ui"] = False
        for k, v in params.items():
            p.props[k] = v
        spec = case_spec()
        video = jsmini.CanvasShim(make_frame(*spec[0][1:], W, H).copy())
        video.props.update(currentTime=1.0, paused=False, ended=False)
        canvas = jsmini.CanvasShim(np.zeros((H, W, 4), np.uint8))
        ht = it.get(["headtrackr", "Tracker"]).construct([p])
        it.events.clear()
        it.timers.clear()
        it.call(ht.get("init"), ht, video, canvas, False)
        steps = []
        for n, (action, kind, t) in enumerate(spec):
            video.pix = make_frame(kind, t, W, H).copy()
            it.now_ms += 35.0
            n0 = len(it.events)
            if action == "start":
                assert it.call(ht.get("start"), ht) is True
            else:
                live = [tm for tm in it.timers if not tm[3]]
                assert live, "no pending timer"
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
        out.append(dict(name=name, params=params, width=W, height=H, ms_per_frame=35.0, steps=steps,
                        stop_events=[mg.event_record(e) for e in it.events[n0:]], fov=it.call(ht.get("getFOV"), ht)))
        print(name, "took %.0f s" % (time.time() - t_case), flush=True)
    OUT.write_text(json.dumps(dict(generator="tools/make_goldens_params.py (src/main.js executed by oracle/jsmini.py)",
                                   cases=out), indent=1))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
