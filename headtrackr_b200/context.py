"""Batched context over the C ABI: frames in, rect lists / track objects out.

Accepts numpy uint8 arrays (host memory) or torch CUDA uint8 tensors (device memory, zero copy) of
shape (n, H, W, 4) or (H, W, 4).  torch is optional and only used for device-resident batches.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (HeadEvent, HeadParams, HtError, Rect, StreamEvent, TrackerEvent, TrackerParams, TrackObj, VideoFrame,
                   Window)
from .synth import load_cascade_blob


def _is_torch(x):
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _frames_ptr(frames):
    """-> (address, n, H, W, keepalive)"""
    if _is_torch(frames):
        t = frames
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if not t.is_contiguous() or t.element_size() != 1 or t.shape[-1] != 4:
            raise ValueError("frames tensor must be contiguous uint8 (n,H,W,4)")
        return t.data_ptr(), t.shape[0], t.shape[1], t.shape[2], t
    a = np.ascontiguousarray(frames, dtype=np.uint8)
    if a.ndim == 3:
        a = a[None]
    if a.ndim != 4 or a.shape[-1] != 4:
        raise ValueError("frames must be (n,H,W,4) uint8")
    return a.ctypes.data, a.shape[0], a.shape[1], a.shape[2], a


def rect_to_dict(r, raw=False):
    d = {"x": r.x, "y": r.y, "width": r.width, "height": r.height}
    d["neighbor" if raw else "neighbors"] = r.neighbors  # src/ccv.js:232 vs :301
    d["confidence"] = r.confidence
    return d


class Context:
    def __init__(self, max_width=1280, max_height=720, max_frames=64, device=0, cascade=None, stream=None,
                 max_raw_per_frame=0, max_rects_per_frame=0):
        self._h = C.c_void_p()
        self._L = _lib.lib()
        blob = cascade if cascade is not None else load_cascade_blob()
        cfg = _lib.Config(device, max_width, max_height, max_frames, max_raw_per_frame, max_rects_per_frame,
                          C.c_void_p(stream) if stream else None)
        rc = self._L.ht_create(C.byref(self._h), C.byref(cfg), blob, len(blob))
        if rc != 0:
            raise HtError(rc, (self._L.ht_last_error(None) or b"").decode())
        self.K = self._L.ht_max_rects(self._h)
        self.raw_cap = max_raw_per_frame if max_raw_per_frame > 0 else 1024   # ht_config.max_raw_per_frame's default
        self.max_frames = max_frames
        self.last_warning = None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._L.ht_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise HtError(rc, (self._L.ht_last_error(self._h) or b"").decode())
        self.last_warning = (self._L.ht_last_error(self._h) or b"").decode() if rc > 0 else None
        return rc

    def sync(self):
        return self._check(self._L.ht_sync(self._h))

    @property
    def launch_count(self):
        return int(self._L.ht_launch_count(self._h))

    def profile(self, enable=True):
        self._check(self._L.ht_profile(self._h, int(bool(enable))))

    def profile_read(self, reset=True):
        """-> {class: (milliseconds, launches)} accumulated while profiling was enabled."""
        n = len(_lib.PROF_CLASSES)
        ms = (C.c_double * n)()
        ln = (C.c_uint64 * n)()
        self._check(self._L.ht_profile_read(self._h, C.addressof(ms), C.addressof(ln), int(bool(reset))))
        return {name: (ms[i], int(ln[i])) for i, name in enumerate(_lib.PROF_CLASSES)}

    # ---- ccv.detect_objects ----
    def detect_raw(self, frames, interval=5, min_neighbors=1, out_rects=None, out_counts=None):
        """Low-level: returns (rects, counts).  With torch device outputs the call is asynchronous."""
        ptr, n, H, W, keep = _frames_ptr(frames)
        if out_rects is None:
            rects = (Rect * (n * self.K))()
            counts = (C.c_int32 * n)()
            self._check(self._L.ht_detect(self._h, ptr, n, W, H, interval, min_neighbors,
                                          C.addressof(rects), C.addressof(counts)))
            return rects, counts
        self._check(self._L.ht_detect(self._h, ptr, n, W, H, interval, min_neighbors,
                                      out_rects.data_ptr(), out_counts.data_ptr()))
        return out_rects, out_counts

    def detect(self, frames, interval=5, min_neighbors=1):
        """-> per frame, the list detect_objects returns: dicts {x,y,width,height,neighbors,confidence}."""
        rects, counts = self.detect_raw(frames, interval, min_neighbors)
        raw = not (min_neighbors > 0)
        return [[rect_to_dict(rects[f * self.K + i], raw) for i in range(counts[f])] for f in range(len(counts))]

    # ---- camshift ----
    @staticmethod
    def _slots(slots, n):
        if slots is None:
            return None, None
        a = (C.c_int32 * n)(*slots)
        return C.addressof(a), a

    def track_init(self, frames, rects, slots=None, calc_angles=True):
        ptr, n, H, W, keep = _frames_ptr(frames)
        r = np.ascontiguousarray(rects, dtype=np.int32).reshape(n, 4)
        sp, skeep = self._slots(slots, n)
        self._check(self._L.ht_track_init(self._h, sp, n, ptr, W, H, r.ctypes.data, int(bool(calc_angles))))

    def track_init_from_detect(self, frames, det_rects, det_counts, slots=None, calc_angles=True):
        ptr, n, H, W, keep = _frames_ptr(frames)
        sp, skeep = self._slots(slots, n)
        found = (C.c_int32 * n)()
        dr = det_rects.data_ptr() if _is_torch(det_rects) else C.addressof(det_rects)
        dc = det_counts.data_ptr() if _is_torch(det_counts) else C.addressof(det_counts)
        self._check(self._L.ht_track_init_from_detect(self._h, sp, n, ptr, W, H, dr, dc, int(bool(calc_angles)),
                                                      C.addressof(found)))
        return list(found)

    def track(self, frames, slots=None, n_calls=1, out_objs=None, out_windows=None):
        ptr, n, H, W, keep = _frames_ptr(frames)
        sp, skeep = self._slots(slots, n)
        if out_objs is not None:
            self._check(self._L.ht_track(self._h, sp, n, ptr, W, H, n_calls, out_objs.data_ptr(),
                                         out_windows.data_ptr() if out_windows is not None else None))
            return out_objs, out_windows
        objs = (TrackObj * n)()
        wins = (Window * n)()
        self._check(self._L.ht_track(self._h, sp, n, ptr, W, H, n_calls, C.addressof(objs), C.addressof(wins)))
        return ([dict(x=o.x, y=o.y, width=o.width, height=o.height, angle=o.angle) for o in objs],
                [(w.x, w.y, w.width, w.height) for w in wins])

    def detect_track(self, frames, interval=5, min_neighbors=1, calc_angles=False, n_calls=1, outputs=None):
        """Batched facetrackr VJ->CS flow (ht_detect_track).

        outputs=None: host results -> (rect lists, found, track objects, windows).
        outputs=(rects, counts, found, objs, windows) torch CUDA tensors: asynchronous, nothing returned to the host.
        """
        ptr, n, H, W, keep = _frames_ptr(frames)
        if outputs is not None:
            r, cnt, fnd, ob, wn = outputs
            self._check(self._L.ht_detect_track(self._h, ptr, n, W, H, interval, min_neighbors, int(bool(calc_angles)),
                                                n_calls, r.data_ptr(), cnt.data_ptr(),
                                                fnd.data_ptr() if fnd is not None else None, ob.data_ptr(),
                                                wn.data_ptr() if wn is not None else None))
            return None
        rects = (Rect * (n * self.K))()
        counts = (C.c_int32 * n)()
        found = (C.c_int32 * n)()
        objs = (TrackObj * n)()
        wins = (Window * n)()
        self._check(self._L.ht_detect_track(self._h, ptr, n, W, H, interval, min_neighbors, int(bool(calc_angles)),
                                            n_calls, C.addressof(rects), C.addressof(counts), C.addressof(found),
                                            C.addressof(objs), C.addressof(wins)))
        dets = [[rect_to_dict(rects[f * self.K + i]) for i in range(counts[f])] for f in range(n)]
        return (dets, list(found),
                [dict(x=o.x, y=o.y, width=o.width, height=o.height, angle=o.angle) for o in objs],
                [(w.x, w.y, w.width, w.height) for w in wins])

    # ---- facetrackr state machine for n streams, on the device ----
    def stream_reset(self, first=0, n=None):
        """Streams [first, first+n) start over in "VJ" (a new facetrackr.Tracker with whitebalancing off)."""
        self._check(self._L.ht_stream_reset(self._h, first, self.max_frames - first if n is None else n))

    def stream_head_config(self, smoothing=True, fov=None, camera_offset=11.5, head_position=True, edgecorrection=True,
                           alpha=0.35, distance_to_screen=60.0, enable=True):
        """Head-position epilogue of stream_step (src/main.js:246-300): parameters of headtrackr.Tracker
        ({smoothing, fov, cameraOffset, headPosition}); enable=False switches it off."""
        if not enable:
            self._check(self._L.ht_stream_head_config(self._h, None))
            return
        p = HeadParams(int(bool(smoothing)), int(bool(head_position)), int(bool(edgecorrection)), 0, alpha,
                       float(fov) if fov is not None else 0.0, camera_offset, distance_to_screen)
        self._check(self._L.ht_stream_head_config(self._h, C.addressof(p)))

    def stream_step_head(self, frames, interval=5, min_neighbors=1, calc_angles=False):
        """stream_step plus the head epilogue -> (events, heads); heads[k] = dict(valid, found, x, y, z, face=(x,y,w,h))."""
        ptr, n, H, W, keep = _frames_ptr(frames)
        ev = (StreamEvent * n)()
        he = (HeadEvent * n)()
        self._check(self._L.ht_stream_step_head(self._h, ptr, n, W, H, interval, min_neighbors, int(bool(calc_angles)),
                                                C.addressof(ev), C.addressof(he)))
        events = [dict(detection=("", "VJ", "CS")[e.detection], x=e.x, y=e.y, width=e.width, height=e.height, angle=e.angle,
                       confidence=e.confidence, found=bool(e.status & 1), lost=bool(e.status & 2)) for e in ev]
        heads = [dict(valid=bool(h.valid), found=bool(h.status & 1), x=h.x, y=h.y, z=h.z,
                      face=(h.fx, h.fy, h.fwidth, h.fheight)) for h in he]
        return events, heads

    def stream_step(self, frames, interval=5, min_neighbors=1, calc_angles=False, out_events=None):
        """One frame per stream through ht_stream_step.  -> per stream, the TrackObj facetrackr.getTrackingObject()
        would return after track(): dict(detection="VJ"|"CS", x, y, width, height, angle, confidence, found, lost).
        out_events (a torch CUDA uint8 tensor of n*56 bytes): asynchronous, nothing returned."""
        ptr, n, H, W, keep = _frames_ptr(frames)
        if out_events is not None:
            self._check(self._L.ht_stream_step(self._h, ptr, n, W, H, interval, min_neighbors, int(bool(calc_angles)),
                                               out_events.data_ptr()))
            return None
        ev = (StreamEvent * n)()
        self._check(self._L.ht_stream_step(self._h, ptr, n, W, H, interval, min_neighbors, int(bool(calc_angles)),
                                           C.addressof(ev)))
        return [dict(detection=("", "VJ", "CS")[e.detection], x=e.x, y=e.y, width=e.width, height=e.height, angle=e.angle,
                     confidence=e.confidence, found=bool(e.status & 1), lost=bool(e.status & 2)) for e in ev]

    # ---- headtrackr.Tracker lifecycle for n streams, on the device ----
    def tracker_config(self, retryDetection=True, calcAngles=False, smoothing=True, fov=None, cameraOffset=11.5,
                       headPosition=True, edgecorrection=True, alpha=0.35, distance_to_screen=60.0, enable=True):
        """Switch the per-stream headtrackr.Tracker lifecycle on with the reference's parameters (src/main.js:39-55),
        or off (enable=False: every stream goes back to stream_reset's state)."""
        if not enable:
            self._check(self._L.ht_tracker_config(self._h, None))
            return
        head = HeadParams(int(bool(smoothing)), int(bool(headPosition)), int(bool(edgecorrection)), 0, alpha,
                          float(fov) if fov is not None else 0.0, cameraOffset, distance_to_screen)
        p = TrackerParams(int(bool(retryDetection)), int(bool(calcAngles)), (C.c_int32 * 2)(), head)
        self._check(self._L.ht_tracker_config(self._h, C.addressof(p)))

    def tracker_reset(self, first=0, n=None):
        """Streams [first, first+n): a new headtrackr.Tracker, initialised, not running."""
        self._check(self._L.ht_tracker_reset(self._h, first, self.max_frames - first if n is None else n))

    def tracker_start(self, first=0, n=None):
        """start() for streams [first, first+n): their next frame goes through the starter (no-op if running)."""
        self._check(self._L.ht_tracker_start(self._h, first, self.max_frames - first if n is None else n))

    def tracker_stop(self, first=0, n=None):
        """stop() for streams [first, first+n); the "stopped" status is the caller's to emit."""
        self._check(self._L.ht_tracker_stop(self._h, first, self.max_frames - first if n is None else n))

    def tracker_step(self, frames, now_ms, out=None):
        """One timer tick of streams [0, n) -> list of ht_tracker_event records as dicts (tracker_event_dict).
        out: a torch CUDA uint8 tensor of n*144 bytes -> asynchronous, nothing returned (tracker_events_from_bytes)."""
        ptr, n, H, W, keep = _frames_ptr(frames)
        if out is not None:
            self._check(self._L.ht_tracker_step(self._h, ptr, n, W, H, float(now_ms), out.data_ptr()))
            return None
        ev = (TrackerEvent * n)()
        self._check(self._L.ht_tracker_step(self._h, ptr, n, W, H, float(now_ms), C.addressof(ev)))
        return [tracker_event_dict(e) for e in ev]

    def tracker_feed(self, streams, frames, now_ms, width, height, out=None):
        """One timer tick of each listed stream on its own video frame and clock (ht_tracker_feed): drawImage(video, 0,
        0, width, height) onto the working canvas, then what tracker_step does for that stream.  Unlisted streams do
        not tick.  streams: distinct stream ids; frames: one (h, w, 4) u8 video frame per stream, all numpy arrays or
        all torch CUDA tensors (any size; a row-padded view - last two strides (4, 1) - passes its row stride as the
        pitch); now_ms: one clock for all or one per record.  -> event dicts in record order; with a torch CUDA `out`
        tensor of len(streams)*144 bytes: asynchronous, nothing returned."""
        streams = list(streams)
        n = len(frames)
        if len(streams) != n or n == 0:
            raise ValueError("one frame per listed stream")
        clocks = [float(t) for t in now_ms] if hasattr(now_ms, "__len__") else [float(now_ms)] * n
        if len(clocks) != n:
            raise ValueError("one clock per listed stream")
        on_device = _is_torch(frames[0])
        recs = (VideoFrame * n)()
        keep = []
        for b, (k, f) in enumerate(zip(streams, frames)):
            if _is_torch(f) != on_device:
                raise ValueError("frames must be all numpy arrays or all torch CUDA tensors")
            if on_device:
                if f.dim() != 3 or f.element_size() != 1 or f.shape[2] != 4 or f.stride(2) != 1 or f.stride(1) != 4:
                    raise ValueError("frame tensors must be uint8 (h, w, 4) with strides (pitch, 4, 1)")
                ptr, pitch = f.data_ptr(), f.stride(0)
            else:
                a = np.asarray(f)
                if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 4:
                    raise ValueError("frames must be (h, w, 4) uint8")
                if a.strides[2] != 1 or a.strides[1] != 4 or a.strides[0] < 4 * a.shape[1]:
                    a = np.ascontiguousarray(a)
                ptr, pitch = a.ctypes.data, a.strides[0]
                f = a
            keep.append(f)
            recs[b] = VideoFrame(ptr, int(k), f.shape[1], f.shape[0], pitch, clocks[b])
        if out is not None:
            self._check(self._L.ht_tracker_feed(self._h, C.addressof(recs), n, int(on_device), width, height,
                                                out.data_ptr()))
            return None
        ev = (TrackerEvent * n)()
        self._check(self._L.ht_tracker_feed(self._h, C.addressof(recs), n, int(on_device), width, height, C.addressof(ev)))
        return [tracker_event_dict(e) for e in ev]

    def ingest(self, frames, width, height, out=None):
        """drawImage(video, 0, 0, width, height) for a batch (src/main.js:170).  numpy in -> numpy (n, height, width, 4)
        out; with a torch CUDA `out` tensor the result stays on the device."""
        ptr, n, H, W, keep = _frames_ptr(frames)
        if out is not None:
            self._check(self._L.ht_ingest(self._h, ptr, n, W, H, out.data_ptr(), width, height))
            return out
        dst = np.zeros((n, height, width, 4), np.uint8)
        self._check(self._L.ht_ingest(self._h, ptr, n, W, H, dst.ctypes.data, width, height))
        return dst

    def backprojection(self, frame, slot=0):
        ptr, n, H, W, keep = _frames_ptr(frame)
        out = np.zeros((H, W, 4), np.uint8)
        self._check(self._L.ht_backprojection(self._h, slot, ptr, W, H, out.ctypes.data))
        return out

    def whitebalance(self, frames):
        ptr, n, H, W, keep = _frames_ptr(frames)
        out = np.zeros(n, np.float64)
        self._check(self._L.ht_whitebalance(self._h, ptr, n, W, H, out.ctypes.data))
        return out

    # ---- introspection (parity tests) ----
    def plan_info(self, W, H, interval=5):
        ns, su = C.c_int32(), C.c_int32()
        sw, sh = (C.c_int32 * 128)(), (C.c_int32 * 128)()
        self._check(self._L.ht_plan_info(self._h, W, H, interval, C.addressof(ns), C.addressof(su),
                                         C.addressof(sw), C.addressof(sh), 128))
        return dict(n_slots=ns.value, scale_upto=su.value, w=list(sw[:ns.value]), h=list(sh[:ns.value]))

    def debug_plane(self, frame, slot, q=0):
        w, h = C.c_int32(), C.c_int32()
        buf = np.zeros(2048 * 2048, np.uint8)
        rc = self._L.ht_debug_plane(self._h, frame, slot, q, buf.ctypes.data, buf.size, C.addressof(w), C.addressof(h))
        self._check(rc)
        return buf[: w.value * h.value].reshape(h.value, w.value).copy()

    def debug_raw(self, frame, cap=65536):
        """-> (the raw list k_group sorted, at most min(cap, raw_cap) entries; the number of windows the cascade found,
        which exceeds raw_cap when the list overflowed)"""
        out = (Rect * cap)()
        cnt = C.c_int32()
        self._check(self._L.ht_debug_raw(self._h, frame, C.addressof(out), cap, C.addressof(cnt)))
        kept = min(cnt.value, cap, self.raw_cap)
        return [(r.x, r.y, r.width, r.height, r.confidence, r.neighbors) for r in out[:kept]], cnt.value

    def debug_track_stats(self, reset=True):
        out = (C.c_uint64 * 5)()
        self._check(self._L.ht_debug_track_stats(self._h, C.addressof(out), int(bool(reset))))
        return dict(passes=int(out[0]), serial_passes=int(out[1]), pixels=int(out[2]), calls=int(out[3]),
                    memo_hits=int(out[4]))

    def set_track_memo(self, enable=True):
        """Re-use the moments of windows already summed in the same launch (default on; results are identical)."""
        self._check(self._L.ht_set_track_memo(self._h, int(bool(enable))))

    def set_pipeline(self, enable=True):
        """Pipelined batches: a detect_track call with device frames and device outputs leaves its tracking on a second
        stream, where it runs under the next call's detection (identical results; read them after sync() / join())."""
        self._check(self._L.ht_set_pipeline(self._h, int(bool(enable))))

    def join(self):
        """Stream-level join of a pipelined call's tracking (no host wait)."""
        self._check(self._L.ht_join(self._h))

    def debug_set_exactness(self, flags):
        """Force the exactness fallbacks (bit 0: generated cascade stages, 1: late stages, 2: mean-shift moments)."""
        self._check(self._L.ht_debug_set_exactness(self._h, int(flags)))

    def debug_track_trace(self, n):
        """(n, 4) uint64: {start ns, end ns, SM id, passes} per stream (contexts created under HT_TRACK_TRACE=1)."""
        out = np.zeros((n, 4), np.uint64)
        self._check(self._L.ht_debug_track_trace(self._h, out.ctypes.data, n))
        return out

    def debug_track_phases(self, n):
        """(n, 8) uint64 phase totals in SM cycles (profiling builds with -DHT_TRACK_PASSTRACE=1; zeros otherwise)."""
        out = np.zeros((n, 8), np.uint64)
        self._check(self._L.ht_debug_track_phases(self._h, out.ctypes.data, n))
        return out

    def debug_model_hist(self, slot):
        out = np.zeros(4096, np.uint32)
        self._check(self._L.ht_debug_model_hist(self._h, slot, out.ctypes.data))
        return out


def tracker_event_dict(e):
    """ht_tracker_event -> dict with the reference's names; status = the list of headtrackrStatus messages dispatched"""
    return dict(detection=("", "VJ", "CS", "WB")[e.detection], x=e.x, y=e.y, width=e.width, height=e.height,
                angle=e.angle, confidence=e.confidence, wb=e.wb, running=bool(e.running), fov=e.fov,
                status=[s for b, s in enumerate(_lib.TRACKER_STATUS) if e.status >> b & 1],
                head=dict(valid=bool(e.head.valid), x=e.head.x, y=e.head.y, z=e.head.z,
                          face=(e.head.fx, e.head.fy, e.head.fwidth, e.head.fheight)))


def tracker_events_from_bytes(buf):
    """records written to a device buffer by Context.tracker_step(out=...), copied back as bytes"""
    n = len(buf) // C.sizeof(TrackerEvent)
    arr = (TrackerEvent * n).from_buffer_copy(bytes(buf[: n * C.sizeof(TrackerEvent)]))
    return [tracker_event_dict(e) for e in arr]
