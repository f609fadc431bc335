"""Many independent video streams through facetrackr's state machine, batched on the GPU (ht_stream_step).

What `headtrackr.facetrackr.Tracker.track()` does for ONE stream per call in the reference
(/root/reference/src/facetrackr.js:67-126, with the lost-face re-detection of src/main.js:230-244) this class does
for n streams per call: stream k owns tracker slot k of the context; the mode switches ("VJ" -> "CS" on a face,
"CS" -> "VJ" on a lost one), the max-confidence pick and the tracker seeding run in kernels, and the host only
drains one event record per stream and frame.  `facetrackingEvent`s are dispatched exactly as the reference does:
for records with detection == "CS" (src/facetrackr.js:112-125).
"""
import math
import time

import numpy as np

from . import _lib
from .context import tracker_events_from_bytes


class StreamSet:
    def __init__(self, context, n_streams, interval=5, min_neighbors=1, calc_angles=False):
        if n_streams > context.max_frames:
            raise ValueError("more streams than tracker slots in the context")
        self.ctx, self.n = context, n_streams
        self.interval, self.min_neighbors, self.calc_angles = interval, min_neighbors, calc_angles
        self._listeners = []
        self.current = [None] * n_streams            # getTrackingObject() per stream
        context.stream_reset(0, n_streams)

    def addEventListener(self, fn):
        """fn(stream_index, evt): evt is the facetrackingEvent dict (src/facetrackr.js:112-125)."""
        self._listeners.append(fn)

    def reset(self, stream):
        """A new facetrackr.Tracker({whitebalancing: false}) for one stream (src/main.js:236)."""
        self.ctx.stream_reset(stream, 1)

    def enable_head_position(self, **params):
        """headtrackr.Tracker's smoothing + head position per stream (src/main.js:246-300) as a GPU epilogue: the
        listeners then also receive `headtrackingEvent {x, y, z}` and `headtrackrStatus {status: "found"}` dicts."""
        self.ctx.stream_head_config(**params)
        self._head = True

    def track(self, frames):
        """frames: (n, H, W, 4) u8 (numpy or torch CUDA) - the current frame of every stream."""
        t0 = time.time()
        heads = None
        if getattr(self, "_head", False):
            events, heads = self.ctx.stream_step_head(frames, self.interval, self.min_neighbors, self.calc_angles)
        else:
            events = self.ctx.stream_step(frames, self.interval, self.min_neighbors, self.calc_angles)
        dt = int((time.time() - t0) * 1000)
        for k, e in enumerate(events):
            e["time"] = dt
            self.current[k] = e
            if e["detection"] == "CS":
                evt = dict(type="facetrackingEvent", height=e["height"], width=e["width"], angle=e["angle"], x=e["x"],
                           y=e["y"], confidence=e["confidence"], detection="CS", time=dt)
                for fn in self._listeners:
                    fn(k, evt)
            if heads is not None:
                if heads[k]["found"]:
                    for fn in self._listeners:
                        fn(k, dict(type="headtrackrStatus", status="found"))
                if heads[k]["valid"]:
                    for fn in self._listeners:
                        fn(k, dict(type="headtrackingEvent", x=heads[k]["x"], y=heads[k]["y"], z=heads[k]["z"]))
        return events

    def getTrackingObject(self, stream):
        return dict(self.current[stream]) if self.current[stream] is not None else None


def lifecycle_events(rec, status):
    """One ht_tracker_event record (Context.tracker_step dict) -> (the payload dicts headtrackr.Tracker dispatches on
    that frame, in its order; ht.status after the frame).  facetrackingEvent first (src/facetrackr.js:112-125), then the
    headtrackrStatus messages, with status "tracking" set silently on every CS frame before redetecting / lost / found
    (src/main.js:227), then headtrackingEvent (src/headposition.js:183-188)."""
    out = []
    if rec["detection"] == "CS":
        out.append(dict(type="facetrackingEvent", height=rec["height"], width=rec["width"], angle=rec["angle"], x=rec["x"],
                        y=rec["y"], confidence=rec["confidence"], detection="CS"))
        status = "tracking"             # whitebalance / detecting / hints, dispatched before :227, never come with CS
    for msg in rec["status"]:
        out.append(dict(type="headtrackrStatus", status=msg))
        status = msg
    if rec["head"]["valid"]:
        h = rec["head"]
        out.append(dict(type="headtrackingEvent", x=h["x"], y=h["y"], z=h["z"]))
    return out, status


def face_written(records):
    """Which slots a tick refreshed in its face crops and tensors: the bool mask detection == "CS" (2) and width > 0 and
    height > 0, per record.  records: the tick's record dicts (Context.tracker_step / tracker_feed; None: not ticked),
    raw ht_tracker_event bytes (host), or a torch CUDA uint8 buffer of device records (the `out` of a tick) - then the
    mask is a torch CUDA bool tensor, computed by torch ops on torch's current stream without a host sync.  The library
    writes `out` on the context's stream, so those ops read the tick's records only if they are ordered after it: create
    the Context with stream= torch's current stream (then the tick, this mask and a model reading the face tensors run
    in order on one stream), or call Context.sync() (or wait on an event recorded on the context's stream) first."""
    if hasattr(records, "is_cuda"):
        import torch
        b = records.reshape(-1)
        det = b.view(torch.int32).reshape(-1, 36)[:, 0]          # detection at byte 0
        wh = b.view(torch.float64).reshape(-1, 18)                 # width at byte 24, height at 32
        return (det == 2) & (wh[:, 3] > 0) & (wh[:, 4] > 0)
    if isinstance(records, (bytes, bytearray, memoryview)) or hasattr(records, "dtype"):
        raw = np.frombuffer(bytes(records) if not hasattr(records, "dtype") else np.ascontiguousarray(records).tobytes(),
                            np.uint8).reshape(-1, 144)
        det = raw[:, 0:4].copy().view(np.int32)[:, 0]
        wh = raw[:, 24:40].copy().view(np.float64)
        return (det == 2) & (wh[:, 0] > 0) & (wh[:, 1] > 0)
    return np.array([r is not None and r["detection"] == "CS" and r["width"] > 0 and r["height"] > 0 for r in records],
                    dtype=bool)


def _to_int32(v):
    """JavaScript's `v >> 0` (ToInt32)"""
    if not math.isfinite(v):
        return 0
    n = math.trunc(v) & 0xffffffff
    return n - (1 << 32) if n >= 1 << 31 else n


def debug_calls(rec):
    """The 2D-context calls src/main.js:199-219 makes on the debug canvas after one tick's record, in order, as tuples
    ("strokeRect", strokeStyle, x, y, w, h), ("translate", x, y), ("rotate", angle): the detected face on a "VJ" record
    whose confidence is not 0 (a VJ tick without a face strokes 0, 0, 0, 0), the tracked face, rotated about its
    centre, on a "CS" one.  The library puts the back-projection image under them (ht_tracker_set_debug); the strokes
    are left to the caller's 2D library."""
    if rec is None or rec["confidence"] == 0:
        return []
    x, y, w, h = rec["x"], rec["y"], rec["width"], rec["height"]
    if rec["detection"] == "VJ":
        return [("strokeRect", "#0000CC", x, y, w, h)]
    if rec["detection"] == "CS":
        a = rec["angle"]
        return [("translate", x, y), ("rotate", a - math.pi / 2),
                ("strokeRect", "#00CC00", _to_int32(-(w / 2)), _to_int32(-(h / 2)), w, h),
                ("rotate", math.pi / 2 - a), ("translate", -x, -y)]
    return []


def _tracker_kwargs(params):
    """Context.tracker_config keywords of one Tracker's parameter dict (src/main.js:39-55 names and defaults)"""
    p = dict(params or {})
    return dict(retryDetection=p.get("retryDetection", True), calcAngles=p.get("calcAngles", False),
                smoothing=p.get("smoothing", True), fov=p.get("fov"), cameraOffset=p.get("cameraOffset", 11.5),
                headPosition=p.get("headPosition", True))


class TrackerSet:
    """headtrackr.Tracker (src/main.js) for n streams on the GPU (ht_tracker_step): stream k is one Tracker whose
    `setTimeout` fires once per step() call.  start(k) / stop(k) are the Tracker's start() / stop() (stop() emits
    "stopped" at once, src/main.js:350); step(frames) runs one timer tick of every stream - starter, whitebalance gate,
    detection, tracking, status events and head position all on the device - and dispatches the reference's payload
    dicts in the reference's order to the listeners as fn(stream, evt).  feed({stream: video}) ticks only the listed
    streams, each on its own video frame (any size) and clock, as cameras whose timers fire independently do.
    `status[k]` is ht.status, getFOV(k) its fov.  params: one dict of the reference's parameters for every stream, or
    a list of n dicts, one per stream (each stream its own `new headtrackr.Tracker(params)`); set_params(k, params)
    changes one stream's.  A stream's "debug" key is its debug canvas, a torch CUDA uint8 (Dh, Dw, 4) tensor: the
    library puts the back-projection image of every "CS" tick on it, and debug_calls(k) gives the strokes main.js
    draws on top; with "debugStrokes": True the library also draws those strokes on the device (DESIGN.md 2,
    "Strokes").  No two streams may share a debug canvas.  A stream's "camera" key is its head-coupled camera
    controller, a dict as Context.tracker_set_camera takes (realisticAbsoluteCameraControl on the device, written to
    its `out` tensor on every tick with a headtrackingEvent).  A stream's "faceCrop" key is its face crop, a dict as
    Context.tracker_set_face_crop takes: the tracked face cut upright out of the video into its `out` tensor (or, with
    "format": "nv12" / "i420" and a "color", its NV12 / I420 planes for a video encoder) on every tick that keeps the
    face.  A stream's "faceTensor" key is its face tensor, a dict as Context.tracker_set_face_tensor takes: the same
    face as a model's normalised input, independent of "faceCrop".  A stream's "framing" key is its framing, a dict as
    Context.tracker_set_framing takes: a steady face-cam box in its `out` tensor that the crop (and, with "tensor":
    True, the tensor) is cut from instead of the tracked box.  A stream's "redact" key is its face redaction, a dict
    as Context.tracker_set_redact takes: its tracked face hidden in its own (device) video after each tick.  A
    stream's "bestShot" key is its best shot, a dict as Context.tracker_set_best_shot takes: the sharpest face of its
    current or last track in its `out` image(s), with its state.
    Differs from the reference in one place: start() on a running stream does nothing (the reference runs an extra,
    unscheduled pass)."""

    def __init__(self, context, n_streams, params=None, device_events=False):
        if n_streams > context.max_frames:
            raise ValueError("more streams than tracker slots in the context")
        per_stream = isinstance(params, (list, tuple))
        if per_stream and len(params) != n_streams:
            raise ValueError("one params dict per stream")
        self.ctx, self.n = context, n_streams
        self._device_events = device_events          # records written to a torch CUDA buffer, then copied back
        self._listeners = []
        self.status = [""] * n_streams
        self._fov = [0] * n_streams
        self.current = [None] * n_streams
        context.tracker_config(**_tracker_kwargs(None if per_stream else params))
        if per_stream:
            context.tracker_set_params(0, [_tracker_kwargs(p) for p in params])
        context.tracker_reset(0, n_streams)
        debug = [(p or {}).get("debug") for p in (params if per_stream else [params] * n_streams)]
        if any(d is not None for d in debug):      # after tracker_config, which clears every debug canvas
            context.tracker_set_debug(0, debug)
        strokes = [bool((p or {}).get("debugStrokes")) for p in (params if per_stream else [params] * n_streams)]
        if any(strokes):                           # and every stroke flag
            context.tracker_set_debug_strokes(0, strokes)
        camera = [(p or {}).get("camera") for p in (params if per_stream else [params] * n_streams)]
        if any(c is not None for c in camera):     # likewise for camera controllers
            context.tracker_set_camera(0, camera)
        crops = [(p or {}).get("faceCrop") for p in (params if per_stream else [params] * n_streams)]
        if any(c is not None for c in crops):      # and face crops
            context.tracker_set_face_crop(0, crops)
        tensors = [(p or {}).get("faceTensor") for p in (params if per_stream else [params] * n_streams)]
        if any(t is not None for t in tensors):    # and face tensors
            context.tracker_set_face_tensor(0, tensors)
        framings = [(p or {}).get("framing") for p in (params if per_stream else [params] * n_streams)]
        if any(f is not None for f in framings):   # and framings
            context.tracker_set_framing(0, framings)
        redactions = [(p or {}).get("redact") for p in (params if per_stream else [params] * n_streams)]
        if any(r is not None for r in redactions):   # and face redactions
            context.tracker_set_redact(0, redactions)
        shots = [(p or {}).get("bestShot") for p in (params if per_stream else [params] * n_streams)]
        if any(b is not None for b in shots):     # and best shots
            context.tracker_set_best_shot(0, shots)

    def set_params(self, k, params):
        """The parameters of stream k (a dict as for the constructor).  Its state is kept: calcAngles takes effect at
        its next hand-off to camshift, the other parameters on its next tick."""
        if not 0 <= k < self.n:
            raise ValueError(f"stream {k} outside [0, {self.n})")
        self.ctx.tracker_set_params(k, [_tracker_kwargs(params)])
        self.ctx.tracker_set_debug(k, [(params or {}).get("debug")])   # no "debug" key: none, as in the reference
        self.ctx.tracker_set_debug_strokes(k, [bool((params or {}).get("debugStrokes"))])   # no key: off
        self.ctx.tracker_set_camera(k, [(params or {}).get("camera")])  # no "camera" key: none
        self.ctx.tracker_set_face_crop(k, [(params or {}).get("faceCrop")])   # no "faceCrop" key: none
        self.ctx.tracker_set_face_tensor(k, [(params or {}).get("faceTensor")])   # no "faceTensor" key: none
        self.ctx.tracker_set_framing(k, [(params or {}).get("framing")])   # no "framing" key: none
        self.ctx.tracker_set_redact(k, [(params or {}).get("redact")])   # no "redact" key: none
        self.ctx.tracker_set_best_shot(k, [(params or {}).get("bestShot")])   # no "bestShot" key: none

    def addEventListener(self, fn):
        """fn(stream_index, evt): evt is a headtrackrStatus / facetrackingEvent / headtrackingEvent payload dict."""
        self._listeners.append(fn)

    def _emit(self, k, evt):
        for fn in self._listeners:
            fn(k, evt)

    def _range(self, k):
        return (0, self.n) if k is None else (k, 1)

    def start(self, k=None):
        """start() of stream k (all streams if None): the next step() runs its starter."""
        self.ctx.tracker_start(*self._range(k))
        return True

    def stop(self, k=None):
        """stop() of stream k (all streams if None): "stopped" is dispatched now."""
        first, n = self._range(k)
        self.ctx.tracker_stop(first, n)
        for s in range(first, first + n):
            self.status[s] = "stopped"
            self._emit(s, dict(type="headtrackrStatus", status="stopped"))
        return True

    def reset(self, k=None):
        """A new headtrackr.Tracker for stream k (all streams if None), initialised and not running."""
        first, n = self._range(k)
        self.ctx.tracker_reset(first, n)
        for s in range(first, first + n):
            self.status[s], self._fov[s], self.current[s] = "", 0, None

    def step(self, frames, now_ms=None):
        """frames: (n, H, W, 4) u8 (numpy or torch CUDA) - the current frame of every stream."""
        now = time.time() * 1000.0 if now_ms is None else now_ms
        t0 = time.time()
        if self._device_events:
            import torch
            buf = torch.empty(self.n * 144, dtype=torch.uint8, device="cuda")
            self.ctx.tracker_step(frames, now, out=buf)
            self.ctx.sync()                            # the records are written on the library's stream
            recs = tracker_events_from_bytes(buf.cpu().numpy().tobytes())
        else:
            recs = self.ctx.tracker_step(frames, now)
        self._dispatch(range(len(recs)), recs, int((time.time() - t0) * 1000))
        return recs

    def feed(self, frames, now_ms=None, width=None, height=None, view=None):
        """One timer tick of the listed streams only (ht_tracker_feed): frames = {stream: (h, w, 4) u8 video frame}
        (numpy or torch CUDA, any video size), drawn onto a width x height canvas; now_ms = None (the wall clock), one
        clock, or {stream: ms}; width and height: one canvas size for all, or {stream: pixels} (each stream on its own
        canvas, ht_tracker_feed_canvases).  view: None, one view for all (headtrackr_b200.views), or {stream: view}
        (ht_tracker_feed_views).  Streams not listed do not tick.  -> {stream: record}."""
        views = self._views(frames, view)

        def call(ks, vids, now, width, height, out=None):
            return self.ctx.tracker_feed(ks, vids, now, width, height, out=out, view=views)
        return self._feed(frames, now_ms, width, height, call)

    @staticmethod
    def _views(frames, view):
        """view= of feed / feed_yuv -> Context's (None, one view, or a list in the order of frames)"""
        if isinstance(view, dict) and view and all(isinstance(k, int) for k in view):
            return [view[k] for k in frames]
        return view

    def feed_yuv(self, frames, now_ms=None, width=None, height=None, format="nv12", color="bt601", view=None):
        """feed on video in any of _lib.YUV_FORMATS (ht_tracker_feed_yuv): frames = {stream: planes or packed array}
        (Context.tracker_feed_yuv), format and color one for all or {stream: value}; the rest (view included) as for
        feed, and events are dispatched as feed dispatches them."""
        ks = list(frames)
        views = self._views(frames, view)
        fmts = [format[k] for k in ks] if isinstance(format, dict) else format
        colors = [color[k] for k in ks] if isinstance(color, dict) else color

        def call(ks, vids, now, width, height, out=None):
            return self.ctx.tracker_feed_yuv(ks, vids, now, width, height, format=fmts, color=colors, out=out, view=views)
        return self._feed(frames, now_ms, width, height, call)

    def _feed(self, frames, now_ms, width, height, tick):
        if width is None or height is None:
            raise ValueError("the canvas size (width, height) is required")
        ks = list(frames)
        if isinstance(width, dict):
            width = [width[k] for k in ks]
        if isinstance(height, dict):
            height = [height[k] for k in ks]
        for k in ks:
            if not 0 <= k < self.n:
                raise ValueError(f"stream {k} outside [0, {self.n})")
        wall = time.time() * 1000.0
        if isinstance(now_ms, dict):
            now = [now_ms[k] for k in ks]
        else:
            now = wall if now_ms is None else now_ms
        t0 = time.time()
        if self._device_events:
            import torch
            buf = torch.empty(len(ks) * 144, dtype=torch.uint8, device="cuda")
            tick(ks, [frames[k] for k in ks], now, width, height, out=buf)
            self.ctx.sync()                            # the records are written on the library's stream
            recs = tracker_events_from_bytes(buf.cpu().numpy().tobytes())
        else:
            recs = tick(ks, [frames[k] for k in ks], now, width, height)
        self._dispatch(ks, recs, int((time.time() - t0) * 1000))
        return dict(zip(ks, recs))

    def _dispatch(self, ks, recs, dt):
        for k, rec in zip(ks, recs):
            self.current[k] = rec
            self._fov[k] = rec["fov"]
            evts, self.status[k] = lifecycle_events(rec, self.status[k])
            for e in evts:
                if e["type"] == "facetrackingEvent":
                    e["time"] = dt
                self._emit(k, e)

    def snapshot(self, ks, device=False):
        """The Trackers of streams ks as they stand: {"records": their tracker records (Context.tracker_export; a torch
        CUDA tensor on this context's device if `device`, else numpy), and the fields a Tracker has on the host:
        "status" (ht.status, derived from the events), "current" (the last record, for debug_calls), "fov" (getFOV)}."""
        ks = [int(k) for k in ks]
        if device:
            import torch
            out = torch.empty((len(ks), _lib.TRACKER_RECORD_BYTES), dtype=torch.uint8, device=f"cuda:{self.ctx.device}")
            recs = self.ctx.tracker_export(ks, out=out)
            self.ctx.sync()                            # the records are written on the library's stream
        else:
            recs = self.ctx.tracker_export(ks)
        return dict(records=recs, status=[self.status[k] for k in ks], current=[self.current[k] for k in ks],
                    fov=[self._fov[k] for k in ks])

    def restore(self, ks, snap):
        """Streams ks of this set become the Trackers of a snapshot, taken from any set, context or GPU: the records go
        to this context's device through the host, or by a torch copy when they are on another device.  Each stream
        keeps its debug canvas."""
        ks = [int(k) for k in ks]
        for k in ks:
            if not 0 <= k < self.n:
                raise ValueError(f"stream {k} outside [0, {self.n})")
        recs = snap["records"]
        if hasattr(recs, "is_cuda") and recs.is_cuda:
            import torch
            recs = recs.to(f"cuda:{self.ctx.device}")
            torch.cuda.synchronize(recs.device)        # torch's copy runs on its stream, the import on the library's
        self.ctx.tracker_import(ks, recs)
        for k, s, cur, fov in zip(ks, snap["status"], snap["current"], snap["fov"]):
            self.status[k], self.current[k], self._fov[k] = s, cur, fov

    def debug_calls(self, k):
        """debug_calls of stream k's last record"""
        return debug_calls(self.current[k])

    def getFOV(self, k):
        return self._fov[k]
