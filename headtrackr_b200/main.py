"""headtrackr.Tracker mirror — /root/reference/src/main.js:35-379 without the browser glue.

The reference's top-level object wires the camera to a canvas and then, every `detectionInterval` ms, runs one
`track()` pass (src/main.js:168-305): facetrackr step -> status events -> lost-face re-detection -> smoothing ->
head-position estimate.  Everything below the facetrackr step is the accelerated path; this file mirrors the
orchestration ABOVE it so that a user of `headtrackr.Tracker` finds the same methods, statuses and event payloads:

  * camera / getUserMedia / <video> handling (src/main.js:100-157, 328-345) is not mirrored: `init(video, canvas)`
    takes two `Canvas` objects and behaves like `init(video, canvas, false)`; the caller replaces `video.pixels`
    for every new frame and calls `step()` where the browser would fire the `setTimeout(track, interval)` timer;
  * DOM events (`headtrackrStatus`, `facetrackingEvent`, `headtrackingEvent`, dispatched on `document` in the
    reference) become callbacks registered with `addEventListener(type, fn)`; payload keys are the reference's;
  * the debug overlay (on the device it is `params.debug` of streams.TrackerSet, ht_tracker_set_debug), the UI
    messages (src/ui.js) and the video fade are dropped.

Pinned against the reference's own main.js executed by oracle/jsmini.py (tests/golden/reference_js_main.json,
tools/make_goldens_main.py, tests/test_host_main.py).
"""
import math
import time

import numpy as np

from . import facetrackr as _facetrackr
from . import headposition as _headposition
from .smoother import Smoother


class Tracker:
    def __init__(self, params=None, backend=None, clock=None):
        p = dict(params or {})
        p.setdefault("smoothing", True)                             # src/main.js:39-55
        p.setdefault("retryDetection", True)
        p.setdefault("ui", True)
        p["debug"] = False
        p.setdefault("detectionInterval", 20)
        p.setdefault("fadeVideo", False)
        p.setdefault("cameraOffset", 11.5)
        p.setdefault("calcAngles", False)
        p.setdefault("headPosition", True)
        self.params = p
        self._backend = backend
        self._clock = clock or (lambda: time.time() * 1000.0)      # (new Date).getTime()
        self._smoother = None
        self._facetracker = None
        self._headposition = None
        self._detectionTimer = None
        self._fov = 0
        self._run = False
        self._faceFound = False
        self._firstRun = True
        self._headDiagonal = []
        self._timer = None                                          # pending setTimeout callback: "track" / "starter"
        self.status = ""                                            # :67
        self.initialized = False
        self._listeners = {"headtrackrStatus": [], "facetrackingEvent": [], "headtrackingEvent": []}

    # ---- events ----
    def addEventListener(self, type_, fn):
        self._listeners[type_].append(fn)

    def _emit(self, evt):
        for fn in self._listeners[evt["type"]]:
            fn(evt)

    def _headtrackerStatus(self, message):                          # :73-77
        self._emit(dict(type="headtrackrStatus", status=message))
        self.status = message

    # ---- set-up ----
    def init(self, video, canvas, setupVideo=False):                # :99-166
        if setupVideo:
            raise NotImplementedError("camera set-up (getUserMedia) is browser glue; pass setupVideo=False")
        self._video, self._canvas = video, canvas
        self._smoother = Smoother(0.35, self.params["detectionInterval"] + 15)   # :163
        self.initialized = True

    def _new_facetracker(self, params):
        ft = _facetrackr.Tracker(params, backend=self._backend)
        ft.addEventListener(self._emit)
        return ft

    def _draw_video(self):                                          # canvasContext.drawImage(videoElement, 0, 0, w, h)
        src = self._video.pixels
        if tuple(src.shape) != tuple(self._canvas.pixels.shape):
            raise ValueError("video and canvas sizes differ: scaling video frames is browser glue (src/main.js:170)")
        self._canvas.pixels = src.clone() if hasattr(src, "is_cuda") else np.array(src, copy=True)

    # ---- one pass of the timer callback: src/main.js:168-305 ----
    def _track(self):
        p = self.params
        self._draw_video()
        if self._facetracker is None:                               # :173-176
            self._facetracker = self._new_facetracker({"calcAngles": p["calcAngles"]})
            self._facetracker.init(self._canvas)
        self._facetracker.track()                                   # :179-180
        o = self._facetracker.getTrackingObject()
        faceObj = dict(o.__dict__)
        if faceObj["detection"] == "WB":
            self._headtrackerStatus("whitebalance")
        if self._firstRun and faceObj["detection"] == "VJ":
            self._headtrackerStatus("detecting")
        if not (faceObj["confidence"] == 0):                        # :186
            if faceObj["detection"] == "VJ":
                if self._detectionTimer is None:
                    self._detectionTimer = self._clock()
                if (self._clock() - self._detectionTimer) > 5000:
                    self._headtrackerStatus("hints")
            if faceObj["detection"] == "CS":
                if self._detectionTimer is not None:
                    self._detectionTimer = None
                self.status = "tracking"                            # :227 (no event)
                if faceObj["width"] == 0 or faceObj["height"] == 0:  # :230 lost face
                    if p["retryDetection"]:
                        self._headtrackerStatus("redetecting")
                        self._facetracker = self._new_facetracker({"whitebalancing": False, "calcAngles": p["calcAngles"]})
                        self._facetracker.init(self._canvas)
                        self._faceFound = False
                        self._headposition = None
                    else:
                        self._headtrackerStatus("lost")
                        self.stop()
                else:
                    if not self._faceFound:
                        self._headtrackerStatus("found")
                        self._faceFound = True
                    if p["smoothing"]:                              # :255-261
                        if not self._smoother.initialized:
                            self._smoother.init(faceObj)
                        faceObj = self._smoother.smooth(faceObj)
                    if self._headposition is None and p["headPosition"]:
                        stable = False                              # :265-281
                        headdiag = math.sqrt(faceObj["width"] * faceObj["width"] + faceObj["height"] * faceObj["height"])
                        if len(self._headDiagonal) < 6:
                            self._headDiagonal.append(headdiag)
                        else:
                            del self._headDiagonal[0]
                            self._headDiagonal.append(headdiag)
                            if (_js_max(self._headDiagonal) - _js_min(self._headDiagonal)) < 5:
                                stable = True
                        if stable:
                            W, H = self._canvas.width, self._canvas.height
                            if self._firstRun:
                                hp_params = {"distance_from_camera_to_screen": p["cameraOffset"]}
                                if p.get("fov") is not None:
                                    hp_params["fov"] = p["fov"]
                                self._headposition = self._new_headposition(faceObj, W, H, hp_params)
                                self._fov = self._headposition.getFOV()
                                self._firstRun = False
                            else:
                                self._headposition = self._new_headposition(
                                    faceObj, W, H, {"fov": self._fov, "distance_from_camera_to_screen": p["cameraOffset"]})
                            self._headposition.track(faceObj)
                    elif p["headPosition"]:
                        self._headposition.track(faceObj)
        if self._run:                                               # :302-304
            self._timer = "track"
        return faceObj

    def _new_headposition(self, faceObj, W, H, params):
        hp = _headposition.Tracker(faceObj, W, H, params)
        hp.addEventListener(self._emit)
        return hp

    def _starter(self):                                             # :307-326
        self._draw_video()
        backend = self._backend or _facetrackr.CudaBackend()
        if backend.whitebalance(self._canvas) > 0:
            self._run = True
            self._track()
        else:
            self._timer = "starter"

    # ---- public API ----
    def start(self):                                                # :328-345 (the video is always "playing")
        if not self.initialized:
            return False
        self._starter()
        return True

    def step(self):
        """Fire the pending setTimeout callback (one tracking pass, or another start attempt).  -> True if one ran."""
        t, self._timer = self._timer, None
        if t == "track":
            self._track()
            return True
        if t == "starter":
            self._starter()
            return True
        return False

    def stop(self):                                                 # :347-355
        if self._timer == "track":                                  # clearTimeout(detector): a pending starter() retry survives
            self._timer = None
        self._run = False
        self._headtrackerStatus("stopped")
        self._facetracker = None
        self._faceFound = False
        return True

    def getFOV(self):                                               # :363-365
        return self._fov


def _js_max(values):                                                # Math.max.apply(null, a): NaN if any element is NaN
    return math.nan if any(v != v for v in values) else max(values)


def _js_min(values):
    return math.nan if any(v != v for v in values) else min(values)
