#!/usr/bin/env python
"""Golden debug canvases of headtrackr.Tracker (src/main.js, `params.debug`), executed by oracle/jsmini.py on top of
the unmodified ccv / cascade / camshift / whitebalance / facetrackr / smoother / headposition sources
-> tests/golden/reference_js_debug.json.

Same cut of main.js and the same harness as tools/make_goldens_lifecycle.py (a canvas shim as the <video> element,
recorded timers, `it.now_ms` as the clock, the actions tick / start / stop).  `params.debug` is a DebugCanvas: a
canvas shim whose 2D context also records strokeRect (with the strokeStyle current at the call), translate and
rotate, and takes putImageData - facetrackr's getBackProjectionImg on every CS pass (src/facetrackr.js:193-196) -
through CanvasShim's clipping.  Strokes are recorded, not rasterized.

Cases (160x120 working canvases):
  main_stream    the main.js stream: VJ -> CS -> lost -> "redetecting" -> found again
  angles         calcAngles: true (rotations by the tracked angle; NaN angles once the face is lost)
  clipped        a 100x80 debug canvas: the image is clipped to it
  larger         a 200x150 debug canvas pre-filled with a pattern: the border outside 160x120 keeps it
  no_retry_stop  retryDetection: false with stop() / start(): the debug canvas persists across both

Each step records the action and frame, the events, `ht.status`, the debug-context calls made during the step and
the sha256 of the debug canvas bytes afterwards.  The C oracle's hto_backprojection_img, composited with the same
clipping, is asserted to reproduce every debug canvas the JS drew.
"""
import hashlib
import json
import math
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import make_goldens_lifecycle as lg  # noqa: E402
import make_goldens_main as mg  # noqa: E402
import oracle  # noqa: E402
from headtrackr_b200 import synth  # noqa: E402
from oracle import jsmini  # noqa: E402

REF = mg.REF
OUT = ROOT / "tests" / "golden" / "reference_js_debug.json"
W, H = mg.W, mg.H


def cases():
    """name -> (params, (debug width, debug height, fill), [(action, kind, t)])"""
    tick = lambda kind, ts: [("tick", kind, t) for t in ts]
    main = [("start" if n == 0 else "tick", kind, t) for n, (kind, t) in enumerate(mg.stream_frames())]
    return [
        ("main_stream", {}, (W, H, "zeros"), main),
        ("angles", {"calcAngles": True}, (W, H, "zeros"), main),
        ("clipped", {}, (100, 80, "zeros"), main),
        ("larger", {}, (200, 150, "pattern"), main),
        ("no_retry_stop", {"retryDetection": False}, (W, H, "zeros"),
         [("start", "face", 0)] + tick("face", range(1, 22)) + [("stop", "face", 22), ("tick", "face", 22),
                                                                 ("start", "face", 23)]
         + tick("face", range(24, 42)) + tick("empty", [0, 0]) + [("start", "face", 50)] + tick("face", range(51, 70))),
    ]


def debug_canvas(dw, dh, fill):
    """the debug canvas a case starts with: transparent black, or a fixed pattern"""
    if fill == "zeros":
        return np.zeros((dh, dw, 4), np.uint8)
    return np.random.default_rng(20261016).integers(0, 256, (dh, dw, 4), dtype=np.uint8)


def composite(dst, img):
    """putImageData(img, 0, 0) clipped to dst (pixels outside img's extent keep their value)"""
    h, w = min(img.shape[0], dst.shape[0]), min(img.shape[1], dst.shape[1])
    dst[:h, :w] = img[:h, :w]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class DebugCanvas(jsmini.CanvasShim):
    """params.debug: CanvasShim plus a log of the 2D-context calls main.js makes on it"""

    def __init__(self, pixels, working):
        jsmini.CanvasShim.__init__(self, pixels)
        self.working = working
        self.calls = []
        self.puts = []              # the working canvas at each putImageData

    def context(self):
        if self._ctx is None:
            c = jsmini.CanvasShim.context(self)
            num = jsmini.to_number
            c.props["strokeRect"] = jsmini.NativeFunction(lambda this, a: self._log(
                ("strokeRect", c.get("strokeStyle"), *[num(v) for v in a[:4]])))
            c.props["translate"] = jsmini.NativeFunction(lambda this, a: self._log(("translate", num(a[0]), num(a[1]))))
            c.props["rotate"] = jsmini.NativeFunction(lambda this, a: self._log(("rotate", num(a[0]))))
            put = c.props["putImageData"]
            c.props["putImageData"] = jsmini.NativeFunction(lambda this, a: self._put(put, this, a))
        return self._ctx

    def _log(self, call):
        self.calls.append(call)
        return jsmini.undefined

    def _put(self, put, this, a):
        self.puts.append(self.working.pix.copy())
        return jsmini.call_function(put, this, a)


def main():
    it = jsmini.Interpreter()
    it.run(mg.cut_main())
    it.run("headtrackr.headposition = {};")
    for f in ("ccv.js", "cascade.js", "camshift.js", "whitebalance.js", "facetrackr.js", "smoother.js", "headposition.js"):
        it.run((REF / f).read_text())
    blob = synth.load_cascade_blob()
    out = []
    for name, params, (dw, dh, fill), spec in cases():
        t_case = time.time()
        p = jsmini.JSObject()
        p.props["ui"] = False
        for k, v in params.items():
            p.props[k] = v
        video = jsmini.CanvasShim(lg.make_frame(*spec[0][1:]).copy())
        video.props.update(currentTime=1.0, paused=False, ended=False)
        canvas = jsmini.CanvasShim(np.zeros((H, W, 4), np.uint8))
        dbg = DebugCanvas(debug_canvas(dw, dh, fill), canvas)
        p.props["debug"] = dbg
        ht = it.get(["headtrackr", "Tracker"]).construct([p])
        it.events.clear()
        it.timers.clear()
        it.call(ht.get("init"), ht, video, canvas, False)
        # the oracle's composite: camshift seeded from the last VJ frame before each CS run (src/facetrackr.js:97-108)
        want = debug_canvas(dw, dh, fill)
        cs, vj_frame, seeded_from, last_vj = None, None, None, None
        steps = []
        n_puts = 0
        for n, (action, kind, t) in enumerate(spec):
            video.pix = lg.make_frame(kind, t).copy()
            it.now_ms += 35.0
            n0, c0, p0 = len(it.events), len(dbg.calls), len(dbg.puts)
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
            calls = dbg.calls[c0:]
            assert len(dbg.puts) - p0 <= 1
            for frame in dbg.puts[p0:]:
                if seeded_from != last_vj:
                    det = oracle.detect(vj_frame, blob, 5, 1)
                    best = det[0]
                    for r in det[1:]:
                        if r[4] > best[4]:
                            best = r
                    cs = oracle.CamshiftTracker(calc_angles=bool(params.get("calcAngles", False)))
                    cs.init_tracker(vj_frame, *[int(math.floor(v)) for v in best[:4]])
                    seeded_from = last_vj
                composite(want, cs.backprojection_img(frame))
                n_puts += 1
            if any(c[0] == "strokeRect" and c[1] == "#0000CC" for c in calls):
                vj_frame, last_vj = canvas.pix.copy(), n
            assert np.array_equal(dbg.pix, want), f"{name} step {n}: reference JS != C oracle composite"
            ev = [mg.event_record(e) for e in it.events[n0:]]
            steps.append(dict(action=action, frame=[kind, t], status=ht.get("status"), events=ev,
                              calls=[list(c) for c in calls], put=len(dbg.puts) > p0, debug_sha256=sha(dbg.pix)))
            print(name, n, action, kind, t, ht.get("status"), [c[0] for c in calls], flush=True)
        assert n_puts > 0, name
        out.append(dict(name=name, params=params, debug=dict(width=dw, height=dh, fill=fill), ms_per_frame=35.0,
                        steps=steps))
        print(name, "took %.0f s" % (time.time() - t_case), flush=True)
    OUT.write_text(json.dumps(dict(generator="tools/make_goldens_debug.py (src/main.js executed by oracle/jsmini.py)",
                                   width=W, height=H, cases=out), indent=1))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
