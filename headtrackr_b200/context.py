"""Batched context over the C ABI: frames in, rect lists / track objects out.

Accepts numpy uint8 arrays (host memory) or torch CUDA uint8 tensors (device memory, zero copy) of
shape (n, H, W, 4) or (H, W, 4).  torch is optional and only used for device-resident batches.
"""
import ctypes as C
import math

import numpy as np

from . import _lib, framing
from ._lib import (Camera, CameraControl, CanvasFrame, DebugCanvas, FaceCrop, FaceCropYuv, FaceTensor, HeadEvent, HeadParams, HtError, Rect, StreamEvent, TrackerEvent, TrackerParams, TrackObj, VideoFrame,
                   VideoView, Window, YuvFrame, YuvImage)
from .views import video_view
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


# planes of the planar formats, channels of the packed ones (an (h, w, channels) array)
_PLANAR = {"nv12": 2, "i420": 3, "nv21": 2, "i422": 3, "i444": 3, "p010": 2}
_PACKED = {"yuyv": 2, "uyvy": 2, "bgra": 4, "bgr24": 3, "rgb24": 3}


def _plane(p, ndim, wide):
    """one plane: a numpy array or torch tensor of `ndim` dimensions, uint8 (wide: 16-bit samples), unit column stride
    (a packed array: contiguous pixels) -> (address, pitch in bytes, shape, on_device, the object to keep alive)"""
    item = 2 if wide else 1
    what = "uint16" if wide else "uint8"
    if _is_torch(p):
        inner = p.dim() == ndim and p.stride(ndim - 1) == 1 and (ndim == 2 or p.stride(1) == p.shape[2])
        if not inner or p.element_size() != item or p.is_floating_point():
            raise ValueError(f"plane tensors must be {ndim}-D {what} with unit column stride"
                             + ("" if ndim == 2 else " and contiguous pixels"))
        return p.data_ptr(), p.stride(0) * item, tuple(p.shape), bool(p.is_cuda), p
    a = np.asarray(p)
    if a.dtype != (np.uint16 if wide else np.uint8) or a.ndim != ndim:
        raise ValueError(f"planes must be {ndim}-D {what}")
    row = item * int(np.prod(a.shape[1:]))
    if a.strides[-1] != item or (ndim == 3 and a.strides[1] != item * a.shape[2]) or a.strides[0] < row:
        a = np.ascontiguousarray(a)
    return a.ctypes.data, a.strides[0], tuple(a.shape), False, a


def _yuv_image(planes, fmt, color, keep):
    """a video frame of one of _lib.YUV_FORMATS -> (ht_yuv_image, on_device); the planes are appended to `keep`.
      planar formats: a tuple of 2-D planes, (Y, UV) for NV12, (Y, VU) for NV21, (Y, U, V) for I420, I422 and I444,
        (Y, UV) of 16-bit samples for P010 (numpy uint16, torch uint16 or int16);
      packed formats: ONE array, (h, w, 2) uint8 for YUYV and UYVY, (h, w, 4) for BGRA, (h, w, 3) for BGR24 and RGB24
        (an OpenCV frame as it is); an odd-width packed 4:2:2 frame needs a row stride of at least 4 * ceil(w / 2).
    numpy arrays or torch tensors (CPU or CUDA) with unit column stride; row strides become pitches."""
    if fmt not in _lib.YUV_FORMATS:
        raise ValueError(f"format must be one of {sorted(_lib.YUV_FORMATS)}")
    if color not in _lib.YUV_COLORS:
        raise ValueError(f"color must be one of {sorted(_lib.YUV_COLORS)}")
    if fmt in _PACKED:
        if isinstance(planes, (tuple, list)):
            raise ValueError(f"a {fmt} frame is one (h, w, {_PACKED[fmt]}) array")
        ptr, pitch, shape, dev, obj = _plane(planes, 3, False)
        if shape[2] != _PACKED[fmt]:
            raise ValueError(f"a {fmt} frame is one (h, w, {_PACKED[fmt]}) array, not {shape}")
        keep.append(obj)
        img = YuvImage((C.c_void_p * 3)(ptr, None, None), (C.c_int32 * 3)(pitch, 0, 0), shape[1], shape[0],
                       _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color])
        return img, dev
    if len(planes) != _PLANAR[fmt]:
        if fmt in ("nv12", "i420"):
            raise ValueError("an NV12 frame is (Y, UV), an I420 frame (Y, U, V)")
        raise ValueError(f"a {fmt} frame is {_PLANAR[fmt]} planes")
    ptrs, pitches, shapes, where = [], [], [], set()
    for p in planes:
        ptr, pitch, shape, dev, obj = _plane(p, 2, fmt == "p010")
        ptrs.append(ptr)
        pitches.append(pitch)
        shapes.append(shape)
        where.add(dev)
        keep.append(obj)
    if len(where) != 1:
        raise ValueError("the planes of a frame must all be host or all be device memory")
    h, w = shapes[0]
    ch, cw = (h + 1) // 2, (w + 1) // 2
    need = {"nv12": (ch, 2 * cw), "nv21": (ch, 2 * cw), "p010": (ch, 2 * cw), "i420": (ch, cw), "i422": (h, cw),
            "i444": (h, w)}[fmt]
    for i, shape in enumerate(shapes[1:], 1):
        if shape[0] < need[0] or shape[1] < need[1]:
            raise ValueError(f"plane {i} is {shape}, a {w}x{h} {fmt} frame needs {need}")
    img = YuvImage((C.c_void_p * 3)(*(ptrs + [None] * (3 - len(ptrs)))), (C.c_int32 * 3)(*(pitches + [0] * (3 - len(pitches)))),
                   w, h, _lib.YUV_FORMATS[fmt], _lib.YUV_COLORS[color])
    return img, where.pop()


def _face_crop_record(c):
    """a face crop dict of Context.tracker_set_face_crop -> its FaceCrop or FaceCropYuv (None: no crop)"""
    if c is None:
        return None
    fmt, out = c.get("format", "rgba"), c["out"]
    if fmt == "rgba":
        if not _is_torch(out) or not out.is_cuda:
            raise ValueError("a face crop is a torch CUDA tensor")
        if out.dim() != 3 or out.element_size() != 1 or out.shape[2] != 4 or out.stride(2) != 1 or out.stride(1) != 4:
            raise ValueError("face crops must be uint8 (S_h, S_w, 4) with strides (pitch, 4, 1)")
        return FaceCrop(out.data_ptr(), out.shape[1], out.shape[0], out.stride(0), 0, float(c.get("scale", 1.0)))
    if fmt not in ("nv12", "i420"):
        raise ValueError("a face crop's format is 'rgba', 'nv12' or 'i420'")
    color = c.get("color", "bt601")
    if color not in _lib.YUV_COLORS:
        raise ValueError(f"color must be one of {sorted(_lib.YUV_COLORS)}")
    planes = tuple(out) if isinstance(out, (tuple, list)) else (out,)
    if len(planes) != (2 if fmt == "nv12" else 3):
        raise ValueError("an NV12 face crop is (Y, UV), an I420 face crop (Y, U, V)")
    for p in planes:
        if not _is_torch(p) or not p.is_cuda or p.dim() != 2 or p.element_size() != 1 or p.is_floating_point() \
                or p.stride(1) != 1:
            raise ValueError("YUV face crop planes are 2-D uint8 torch CUDA tensors with unit column stride")
    h, w = planes[0].shape
    need = (h // 2, w if fmt == "nv12" else w // 2)
    for i, p in enumerate(planes[1:], 1):
        if p.shape[0] < need[0] or p.shape[1] < need[1]:
            raise ValueError(f"plane {i} is {tuple(p.shape)}, a {w}x{h} {fmt} face crop needs {need}")
    ptrs = [p.data_ptr() for p in planes] + [None] * (3 - len(planes))
    pitches = [p.stride(0) for p in planes] + [0] * (3 - len(planes))
    return FaceCropYuv((C.c_void_p * 3)(*ptrs), (C.c_int32 * 3)(*pitches), w, h, _lib.YUV_FORMATS[fmt],
                       _lib.YUV_COLORS[color], 0, float(c.get("scale", 1.0)))


def _crop_runs(recs):
    """[a, b) ranges of records of one layout, each as long as possible (None joins any run)"""
    runs, kind = [], None
    for i, r in enumerate(recs):
        k = None if r is None else isinstance(r, FaceCropYuv)
        if runs and (k is None or kind is None or k == kind):
            runs[-1][1] = i + 1
            kind = k if kind is None else kind
        else:
            runs.append([i, i + 1])
            kind = k
    return [tuple(r) for r in runs]


_TENSOR_LAYOUTS = {"chw": _lib.HT_TENSOR_CHW, "hwc": _lib.HT_TENSOR_HWC}
_TENSOR_CHANNELS = {"rgb": _lib.HT_TENSOR_RGB, "bgr": _lib.HT_TENSOR_BGR, "gray": _lib.HT_TENSOR_GRAY}


def _tensor_dtype(dtype):
    import torch
    codes = {torch.uint8: _lib.HT_TENSOR_U8, torch.float16: _lib.HT_TENSOR_F16, torch.bfloat16: _lib.HT_TENSOR_BF16,
             torch.float32: _lib.HT_TENSOR_F32}
    if dtype not in codes:
        raise ValueError("a face tensor is uint8, float16, bfloat16 or float32")
    return codes[dtype]


def _channel_values(v, n, fill, what):
    """a scalar, n per-channel values or all 3 of the record -> 3 floats, the unused ones `fill`"""
    vs = [float(x) for x in v] if isinstance(v, (list, tuple)) or hasattr(v, "__len__") else [float(v)] * n
    if len(vs) == 3:
        return vs
    if len(vs) != n:
        raise ValueError(f"{what} needs {n} value(s), one per channel")
    return vs + [fill] * (3 - n)


def tensor_affine(dtype, channels="rgb", mean=None, std=None):
    """(mul, add) of a face tensor, 3 floats each, from a torchvision-style mean / std (in the tensor's channel order,
    on the 0..1 scale): mul = float32(1 / (255 std)) and add = float32(-mean / std), each computed in float64 and
    rounded once.  A uint8 tensor takes no mean / std: (1, 0).  Floats without mean / std: mean 0, std 1 (x / 255)."""
    n = 1 if channels == "gray" else 3
    if _tensor_dtype(dtype) == _lib.HT_TENSOR_U8:
        if mean is not None or std is not None:
            raise ValueError("a uint8 face tensor takes no mean / std")
        return [1.0] * 3, [0.0] * 3
    m = _channel_values(0.0 if mean is None else mean, n, 0.0, "mean")
    sd = _channel_values(1.0 if std is None else std, n, 1.0, "std")
    if not all(math.isfinite(x) and x != 0 for x in sd):
        raise ValueError("std must be finite and non-zero")
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    return [f32(1.0 / (255.0 * x)) for x in sd], [f32(-a / b) for a, b in zip(m, sd)]


def _face_tensor_record(c):
    """a face tensor dict of Context.tracker_set_face_tensor -> its FaceTensor (None: no tensor)"""
    if c is None:
        return None
    out = c["out"]
    if not _is_torch(out) or not out.is_cuda:
        raise ValueError("a face tensor is a torch CUDA tensor")
    layout, channels = c.get("layout", "chw"), c.get("channels", "rgb")
    if layout not in _TENSOR_LAYOUTS or channels not in _TENSOR_CHANNELS:
        raise ValueError("a face tensor's layout is 'chw' or 'hwc', its channels 'rgb', 'bgr' or 'gray'")
    dtype, n = _tensor_dtype(out.dtype), 1 if channels == "gray" else 3
    if out.dim() != 3:
        raise ValueError("a face tensor is 3-D: (C, S_h, S_w) or (S_h, S_w, C)")
    if layout == "chw":
        if out.shape[0] != n or out.stride(2) != 1:
            raise ValueError(f"a CHW {channels} face tensor is ({n}, S_h, S_w) with unit x stride")
        h, w, row, plane = out.shape[1], out.shape[2], out.stride(1), out.stride(0) if n == 3 else 0
    else:
        if out.shape[2] != n or out.stride(2) != 1 or out.stride(1) != n:
            raise ValueError(f"an HWC {channels} face tensor is (S_h, S_w, {n}) with strides (row, {n}, 1)")
        h, w, row, plane = out.shape[0], out.shape[1], out.stride(0), 0
    if "mul" in c or "add" in c:
        if "mean" in c or "std" in c:
            raise ValueError("a face tensor takes mean / std or mul / add, not both")
        mul = _channel_values(c.get("mul", 1.0), n, 1.0, "mul")
        add = _channel_values(c.get("add", 0.0), n, 0.0, "add")
    else:
        mul, add = tensor_affine(out.dtype, channels, c.get("mean"), c.get("std"))
    return FaceTensor(out.data_ptr(), row, plane, w, h, dtype, _TENSOR_LAYOUTS[layout], _TENSOR_CHANNELS[channels], 0,
                      (C.c_float * 3)(*mul), (C.c_float * 3)(*add), float(c.get("scale", 1.0)))


def _per_record(v, n, what):
    vs = list(v) if isinstance(v, (list, tuple)) else [v] * n
    if len(vs) != n:
        raise ValueError(f"one {what} per frame")
    return vs


def _rgba_frame(f, on_device):
    """one (h, w, 4) uint8 video frame, a numpy array or (on_device) a torch CUDA tensor, rows of any stride ->
    (address, pitch in bytes, the array to keep alive)"""
    if on_device:
        if f.dim() != 3 or f.element_size() != 1 or f.shape[2] != 4 or f.stride(2) != 1 or f.stride(1) != 4:
            raise ValueError("frame tensors must be uint8 (h, w, 4) with strides (pitch, 4, 1)")
        return f.data_ptr(), f.stride(0), f
    a = np.asarray(f)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 4:
        raise ValueError("frames must be (h, w, 4) uint8")
    if a.strides[2] != 1 or a.strides[1] != 4 or a.strides[0] < 4 * a.shape[1]:
        a = np.ascontiguousarray(a)
    return a.ctypes.data, a.strides[0], a


def _views(view, n):
    """view= of the feed and ingest methods (one view dict for all records, or a list of one per record) -> an
    ht_video_view array"""
    return (VideoView * n)(*[video_view(v) for v in _per_record(view, n, "view")])


def camera_from_bytes(b):
    """An ht_camera (CAMERA_BYTES bytes: numpy, bytes, or a torch tensor, copied to the host) -> dict: position [3],
    fov, view [6] (fullWidth, fullHeight, x, y, width, height), events, has_view_offset, and projection and
    view_matrix as float32 (4, 4) numpy arrays (row-major views of the column-major matrices, so m[row, col])."""
    if _is_torch(b):
        b = b.detach().cpu().numpy()
    raw = np.frombuffer(bytes(np.ascontiguousarray(b, dtype=np.uint8).reshape(-1)), np.uint8)
    if raw.size != _lib.CAMERA_BYTES:
        raise ValueError(f"an ht_camera is {_lib.CAMERA_BYTES} bytes")
    c = Camera.from_buffer_copy(raw.tobytes())
    return dict(position=list(c.position), fov=c.fov, view=list(c.view), events=c.events,
                has_view_offset=c.has_view_offset,
                projection=np.frombuffer(raw[88:152].tobytes(), np.float32).reshape(4, 4).T.copy(),
                view_matrix=np.frombuffer(raw[152:216].tobytes(), np.float32).reshape(4, 4).T.copy())


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
        self.max_width, self.max_height, self.device = max_width, max_height, device
        self.last_warning = None
        self._outputs = {}                # (kind, stream) -> what the library writes for that output, kept alive while set

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
        p = tracker_params(retryDetection, calcAngles, smoothing, fov, cameraOffset, headPosition, edgecorrection, alpha,
                           distance_to_screen) if enable else None
        self._check(self._L.ht_tracker_config(self._h, None if p is None else C.addressof(p)))
        self._outputs = {}                # ht_tracker_config discards every stream's outputs

    def _keep(self, kind, first, items):
        """keeps items[i] (None: nothing) alive as stream first+i's `kind` output, after the library accepted them"""
        for i, v in enumerate(items):
            if v is None:
                self._outputs.pop((kind, first + i), None)
            else:
                self._outputs[(kind, first + i)] = v

    def tracker_set_params(self, first, params):
        """Parameters of streams first, first+1, ...: one dict of tracker_config's keywords (enable excluded) per stream,
        each its own `new headtrackr.Tracker(params)`.  Stream states are kept; calcAngles takes effect at the stream's
        next hand-off to camshift, the other fields at its next tick.  tracker_config() sets every stream again."""
        params = list(params)
        arr = (TrackerParams * max(1, len(params)))(*[tracker_params(**d) for d in params])
        self._check(self._L.ht_tracker_set_params(self._h, int(first), len(params), C.addressof(arr)))

    def tracker_set_debug(self, first, canvases):
        """Debug canvases (params.debug) of streams first, first+1, ...: per stream None (none) or a torch CUDA uint8
        (Dh, Dw, 4) tensor; a row-padded view - last two strides (4, 1) - passes its row stride as the pitch.  On every
        tick whose facetrackr pass is "CS" the library puts the stream's back-projection image at its top-left corner,
        clipped to it (src/facetrackr.js:193-196).  The context keeps the tensors alive while they are set."""
        canvases = list(canvases)
        arr = (DebugCanvas * max(1, len(canvases)))()
        for i, t in enumerate(canvases):
            if t is None:
                continue
            if not _is_torch(t) or not t.is_cuda:
                raise ValueError("a debug canvas is a torch CUDA tensor")
            if t.dim() != 3 or t.element_size() != 1 or t.shape[2] != 4 or t.stride(2) != 1 or t.stride(1) != 4:
                raise ValueError("debug canvases must be uint8 (Dh, Dw, 4) with strides (pitch, 4, 1)")
            arr[i] = DebugCanvas(t.data_ptr(), t.shape[1], t.shape[0], t.stride(0), 0)
        self._check(self._L.ht_tracker_set_debug(self._h, int(first), len(canvases), C.addressof(arr)))
        self._keep("debug", int(first), canvases)

    def tracker_set_debug_strokes(self, first, flags):
        """Whether streams first, first+1, ... stroke main.js's face rectangles onto their debug canvases
        (ht_tracker_set_debug_strokes): after every tick, on top of its back-projection, the "VJ" box in #0000CC or the
        "CS" box rotated about its centre in #00CC00 (src/main.js:199-219), rasterized as DESIGN.md 2 defines.  The
        flag is the stream's: it outlives set_debug, set_params, stop, start, reset and import; tracker_config clears
        it."""
        flags = [bool(f) for f in flags]
        arr = (C.c_int32 * max(1, len(flags)))(*[int(f) for f in flags])
        self._check(self._L.ht_tracker_set_debug_strokes(self._h, int(first), len(flags), arr))

    def tracker_set_face_crop(self, first, crops):
        """Face crops of streams first, first+1, ... (ht_tracker_set_face_crop / ht_tracker_set_face_crop_yuv): per
        stream None (none) or a dict {"out": ..., "scale": 1.0, "format": "rgba", "color": "bt601"}.  With format
        "rgba" (the default) `out` is a torch CUDA uint8 (S_h, S_w, 4) tensor; a row-padded view - last two strides
        (4, 1) - passes its row stride as the pitch.  With "nv12" or "i420" - what video encoders take - `out` is a
        tuple of 2-D uint8 CUDA planes as tracker_feed_yuv takes them, (Y, UV) or (Y, U, V), with unit column stride
        (row strides become pitches); the Y plane is S_h x S_w, both even, and `color` is one of _lib.YUV_COLORS
        (BT.2020 is rejected).  After every tick on which track() kept the face ("CS", width and height > 0), `out`
        holds the green rectangle main.js strokes, scaled by `scale` about its centre and grown to the crop's aspect
        ratio, cut upright out of the tick's video at video resolution; a YUV crop is the RGBA crop of its size and
        scale converted, alpha ignored (DESIGN.md 2, "Face crops").  A stream has one crop, in one layout: setting
        either replaces it.  The crop is the stream's: it outlives set_params, stop, start, reset and import;
        tracker_config removes it.  The context keeps the tensors alive while they are set.  A list mixing RGBA and
        YUV crops is set one run of equal layout at a time; if the library rejects a run, the runs before it are set
        back, so a rejected call changes nothing."""
        first, crops = int(first), list(crops)
        recs = [_face_crop_record(c) for c in crops]
        prev = [self._outputs.get(("crop", first + i)) for i in range(len(crops))]
        done = 0
        try:
            for a, b in _crop_runs(recs) or [(0, 0)]:   # no crops at all: the library's rejection of n = 0
                self._set_crop_run(first + a, recs[a:b])
                done = b
        except HtError:
            back = [_face_crop_record(c) for c in prev[:done]]
            for a, b in _crop_runs(back):             # the state before the call, which the library accepted
                self._set_crop_run(first + a, back[a:b])
            raise
        self._keep("crop", first, crops)

    def _set_crop_run(self, first, recs):
        """one setter call over records of one layout (None: no crop) from _face_crop_record"""
        yuv = any(isinstance(r, FaceCropYuv) for r in recs)
        T = FaceCropYuv if yuv else FaceCrop
        arr = (T * len(recs))(*[r if r is not None else T() for r in recs])
        setter = self._L.ht_tracker_set_face_crop_yuv if yuv else self._L.ht_tracker_set_face_crop
        self._check(setter(self._h, first, len(recs), C.addressof(arr)))

    def tracker_set_face_tensor(self, first, tensors):
        """Face tensors of streams first, first+1, ... (ht_tracker_set_face_tensor): per stream None (none) or a dict
        {"out": torch CUDA tensor, "layout": "chw", "channels": "rgb", "mean": ..., "std": ... | "mul": ..., "add": ...,
        "scale": 1.0}.  `out` is uint8, float16, bfloat16 or float32 - its dtype is the tensor's - shaped (C, S_h, S_w)
        with unit x stride ("chw") or (S_h, S_w, C) with strides (row, C, 1) ("hwc"), C = 3 ("rgb", "bgr") or 1
        ("gray", the detector's gray); other strides pass through, so a slice of a batch tensor works.  Each element is
        fmaf(c, mul[k], add[k]) rounded to the dtype, c the channel byte of the RGBA crop of the same size and scale
        (uint8: c itself).  mean / std (scalars or one per channel, in the tensor's channel order, on the 0..1 scale
        as torchvision's Normalize takes them) give mul = float32(1 / (255 std)), add = float32(-mean / std), computed
        in float64 and rounded once (tensor_affine); without either, a float tensor holds c / 255.  After every tick
        on which track() kept the face, `out` holds that tick's face (DESIGN.md 2, "Face crops", item 6).  The tensor
        is independent of the stream's face crop - tracker_set_face_crop never touches it - and outlives set_params,
        stop, start, reset and import; tracker_config removes it.  The context keeps the tensors alive while set."""
        first, tensors = int(first), list(tensors)
        recs = [_face_tensor_record(t) for t in tensors]
        arr = (FaceTensor * max(1, len(recs)))(*[r if r is not None else FaceTensor() for r in recs])
        self._check(self._L.ht_tracker_set_face_tensor(self._h, first, len(recs), C.addressof(arr)))
        self._keep("tensor", first, tensors)

    def face_tensor_batch(self, first, n, height, width, dtype=None, layout="chw", channels="rgb", mean=None, std=None,
                          scale=1.0):
        """A batch of face tensors for streams first .. first+n-1: allocates (n, C, height, width) ("chw") or
        (n, height, width, C) ("hwc") of `dtype` (default torch.float16) on the context's device, sets stream first+i
        to slice i (tracker_set_face_tensor, mean / std as there) and returns it.  It starts as what a black crop
        converts to (add[k] per channel), so a slot without a face yet reads as black; streams.face_written(records)
        says which slots a tick refreshed.  The fill has completed when this returns, whatever stream the library and
        torch run on."""
        import torch
        dtype = torch.float16 if dtype is None else dtype
        c = 1 if channels == "gray" else 3
        shape = (n, c, height, width) if layout == "chw" else (n, height, width, c)
        out = torch.empty(shape, dtype=dtype, device=f"cuda:{self.device}")
        _, add = tensor_affine(dtype, channels, mean, std)
        for k in range(c):
            (out[:, k] if layout == "chw" else out[..., k]).fill_(add[k] + 0.0)   # fmaf(0, mul, -0.0) is +0.0
        # the fill runs on torch's stream, the ticks that write faces on the library's: the fill must have landed
        # before a tick can write, or it would blacken faces that face_written reports as fresh
        torch.cuda.current_stream(out.device).synchronize()
        keys = {} if mean is None else {"mean": mean}
        if std is not None:
            keys["std"] = std
        self.tracker_set_face_tensor(first, [dict(out=out[i], layout=layout, channels=channels, scale=scale, **keys)
                                             for i in range(n)])
        return out

    def tracker_set_camera(self, first, controls):
        """Head-coupled camera controllers of streams first, first+1, ...: per stream None (none) or a dict of
        realisticAbsoluteCameraControl's arguments (src/controllers.js:28-38) - scaling, fixedPosition, lookAt (three
        numbers each), screenHeight (default 20), damping (default 1) - the camera's own fov, aspect, near and far, and
        `out`: a torch CUDA uint8 tensor of CAMERA_BYTES bytes, 16-byte aligned, on this context's device (it may be a
        slice of a larger renderer buffer).  Setting a controller writes the constructed camera; then every tick with a
        headtrackingEvent moves it on the device (camera_from_bytes decodes it).  The context keeps the tensors
        alive while they are set."""
        controls = list(controls)
        arr = (CameraControl * max(1, len(controls)))()
        for i, d in enumerate(controls):
            if d is None:
                continue
            t = d["out"]
            if not _is_torch(t) or not t.is_cuda:
                raise ValueError("a camera is a torch CUDA tensor")
            if t.element_size() != 1 or t.numel() != _lib.CAMERA_BYTES or not t.is_contiguous():
                raise ValueError(f"a camera is a contiguous uint8 tensor of {_lib.CAMERA_BYTES} bytes")
            arr[i] = CameraControl(t.data_ptr(), float(d["scaling"]), tuple(float(v) for v in d["fixedPosition"]),
                                   tuple(float(v) for v in d["lookAt"]), float(d.get("screenHeight", 20.0)),
                                   float(d.get("damping", 1.0)), float(d["fov"]), float(d["aspect"]),
                                   float(d["near"]), float(d["far"]))
        self._check(self._L.ht_tracker_set_camera(self._h, int(first), len(controls), C.addressof(arr)))
        self._keep("camera", int(first), [None if d is None else d["out"] for d in controls])

    def tracker_set_framing(self, first, framings):
        """Framings of streams first, first+1, ... (ht_tracker_set_framing): per stream None (none) or a dict {"out":
        torch CUDA uint8 tensor of FRAMED_BOX_BYTES bytes, 8-byte aligned, on this context's device; "alpha": 0.25;
        "dead_zone": 0.1; "crop": True; "tensor": False}.  `out` holds the framed box, a steady face-cam box: on every
        tick that writes crops it snaps to the tracked face when the face has left it (or on the first such tick, or
        a canvas-size change) and otherwise glides towards it by `alpha` of the error outside a dead zone of
        `dead_zone` times its size (DESIGN.md 2, "Face crops", item 7; framing.py replays it on the host and
        box_from_bytes decodes it).  The face crop ("crop") and / or the face tensor ("tensor") are then cut upright
        from the framed box, the others from the tracked one.  Setting a framing starts its box anew.  The framing is
        the stream's: it outlives set_params, stop, start, reset and import; tracker_config removes it.  The context
        keeps the tensors alive while they are set."""
        framings = list(framings)
        arr = (_lib.Framing * max(1, len(framings)))()
        for i, d in enumerate(framings):
            if d is None:
                continue
            t = d["out"]
            if not _is_torch(t) or not t.is_cuda:
                raise ValueError("a framed box is a torch CUDA tensor")
            if t.element_size() != 1 or t.numel() != _lib.FRAMED_BOX_BYTES or not t.is_contiguous():
                raise ValueError(f"a framed box is a contiguous uint8 tensor of {_lib.FRAMED_BOX_BYTES} bytes")
            outputs = (_lib.HT_FRAMING_CROP if d.get("crop", True) else 0) | \
                (_lib.HT_FRAMING_TENSOR if d.get("tensor", False) else 0)
            arr[i] = _lib.Framing(t.data_ptr(), float(d.get("alpha", framing.ALPHA)),
                                  float(d.get("dead_zone", framing.DEAD_ZONE)), outputs, 0)
        self._check(self._L.ht_tracker_set_framing(self._h, int(first), len(framings), C.addressof(arr)))
        self._keep("framing", int(first), [None if d is None else d["out"] for d in framings])

    def tracker_set_best_shot(self, first, shots):
        """Best shots of streams first, first+1, ... (ht_tracker_set_best_shot): per stream None (none) or a dict
        {"out": torch CUDA uint8 (S_h, S_w, 4) tensor, or a pair of two such of one shape and row stride; "state":
        torch CUDA uint8 tensor of BEST_SHOT_STATE_BYTES bytes, 8-byte aligned, on this context's device; "scale":
        1.0}.  A row-padded view - last two strides (4, 1) - passes its row stride as the pitch.  On every tick that
        writes crops the candidate - the RGBA crop of the shot's size and scale, before any redaction, never framed -
        is scored by its Laplacian energy (bestshot.score); the first tick of a track and every later one that scores
        strictly higher write it into `out` (with a pair: track t's into out[(t - 1) % 2], so the last track's best
        stays intact during the next one) and into the state (bestshot.state_from_bytes decodes it; a track ends on
        the stream's first tick that is not a crop tick).  Setting a best shot zeroes its state; the images are not
        touched.  The best shot is the stream's: it outlives set_params, stop, start and reset; import ends its open
        track; tracker_config removes it.  The context keeps the tensors alive while they are set."""
        shots = list(shots)
        arr = (_lib.BestShot * max(1, len(shots)))()
        for i, d in enumerate(shots):
            if d is None:
                continue
            outs = tuple(d["out"]) if isinstance(d["out"], (tuple, list)) else (d["out"],)
            if len(outs) not in (1, 2):
                raise ValueError("a best shot's out is one image or a pair")
            for t in outs:
                if not _is_torch(t) or not t.is_cuda:
                    raise ValueError("a best-shot image is a torch CUDA tensor")
                if t.dim() != 3 or t.element_size() != 1 or t.shape[2] != 4 or t.stride(2) != 1 or t.stride(1) != 4:
                    raise ValueError("best-shot images must be uint8 (S_h, S_w, 4) with strides (pitch, 4, 1)")
            if len(outs) == 2 and (outs[0].shape != outs[1].shape or outs[0].stride(0) != outs[1].stride(0)):
                raise ValueError("the two images of a best shot have one shape and one row stride")
            st = d["state"]
            if not _is_torch(st) or not st.is_cuda:
                raise ValueError("a best-shot state is a torch CUDA tensor")
            if st.element_size() != 1 or st.numel() != _lib.BEST_SHOT_STATE_BYTES or not st.is_contiguous():
                raise ValueError(f"a best-shot state is a contiguous uint8 tensor of {_lib.BEST_SHOT_STATE_BYTES} bytes")
            o = outs[0]
            arr[i] = _lib.BestShot((C.c_void_p * 2)(o.data_ptr(), outs[1].data_ptr() if len(outs) == 2 else None),
                                   st.data_ptr(), o.shape[1], o.shape[0], o.stride(0), 0, float(d.get("scale", 1.0)))
        self._check(self._L.ht_tracker_set_best_shot(self._h, int(first), len(shots), C.addressof(arr)))
        self._keep("best_shot", int(first), [None if d is None else (d["out"], d["state"]) for d in shots])

    def tracker_set_redact(self, first, redactions):
        """Face redactions of streams first, first+1, ... (ht_tracker_set_redact): per stream None (none) or a dict
        {"mode": "mosaic" | "fill"; "block": 16; "scale": 1.25; "hold": 10; "fill_rgb": (0, 0, 0); "fill_yuv": (16, 128,
        128)}.  After each tick the stream's tracked face is hidden in its own video, in place: every cell of a block x
        block grid anchored at video pixel (0, 0) that meets the face box scaled by `scale` becomes its mean (mosaic)
        or the fill colour (fill_rgb on RGBA8 and packed RGB video, fill_yuv on YUV video), and the last face box
        stays hidden for `hold` ticks after the face is lost (DESIGN.md 2, "Face redaction"; views.redact_rect gives
        the rectangle).  headtrackr tracks one face per stream: this hides that face, not every face in the frame.
        The library writes the stream's video, which must then be device memory and shared with no other redacting
        stream of the tick.  The crops and tensors of the tick see the unredacted face.  The redaction is the
        stream's: it outlives set_params, stop, start, reset and import; tracker_config removes it."""
        redactions = list(redactions)
        arr = (_lib.FaceRedact * max(1, len(redactions)))()
        modes = {"mosaic": _lib.HT_REDACT_MOSAIC, "fill": _lib.HT_REDACT_FILL}
        for i, d in enumerate(redactions):
            if d is None:
                continue
            mode = d.get("mode", "mosaic")
            r = arr[i]
            r.mode = modes[mode] if isinstance(mode, str) else int(mode)
            r.block, r.hold, r.scale = int(d.get("block", 16)), int(d.get("hold", 10)), float(d.get("scale", 1.25))
            r.fill_rgb[:] = [int(v) for v in d.get("fill_rgb", (0, 0, 0))]
            r.fill_yuv[:] = [int(v) for v in d.get("fill_yuv", (16, 128, 128))]
        self._check(self._L.ht_tracker_set_redact(self._h, int(first), len(redactions), C.addressof(arr)))

    def tracker_export(self, streams, out=None):
        """The tracker records of the listed streams (ht_tracker_export): a (len(streams), TRACKER_RECORD_BYTES) uint8
        numpy array, or with a contiguous torch CUDA uint8 `out` of that many bytes on this context's device the
        records written there, asynchronously on the library's stream (sync() before reading them elsewhere)."""
        ids = (C.c_int32 * max(1, len(streams)))(*[int(k) for k in streams])
        n = len(streams)
        if out is not None:
            if not _is_torch(out) or not out.is_cuda or not out.is_contiguous() or out.element_size() != 1 or \
                    out.numel() != n * _lib.TRACKER_RECORD_BYTES:
                raise ValueError("out must be a contiguous torch CUDA uint8 tensor of len(streams) records")
            self._check(self._L.ht_tracker_export(self._h, C.addressof(ids), n, out.data_ptr()))
            return out
        recs = np.zeros((n, _lib.TRACKER_RECORD_BYTES), np.uint8)
        self._check(self._L.ht_tracker_export(self._h, C.addressof(ids), n, recs.ctypes.data))
        return recs

    def tracker_import(self, streams, records):
        """Stream streams[i] := records[i] (ht_tracker_import): its state, parameters and camshift tracker become the
        exported stream's; its debug canvas stays.  records: (n, TRACKER_RECORD_BYTES) uint8, a numpy array or a
        contiguous torch CUDA tensor on this context's device.  Every record is checked first; on an error (HtError)
        no stream changes."""
        n = len(streams)
        ids = (C.c_int32 * max(1, n))(*[int(k) for k in streams])
        if _is_torch(records):
            if not records.is_contiguous() or records.element_size() != 1 or records.numel() != n * _lib.TRACKER_RECORD_BYTES:
                raise ValueError("records must be a contiguous uint8 tensor of len(streams) records")
            self._check(self._L.ht_tracker_import(self._h, C.addressof(ids), n, records.data_ptr()))
            return
        a = np.ascontiguousarray(records, dtype=np.uint8)
        if a.size != n * _lib.TRACKER_RECORD_BYTES:
            raise ValueError("records must hold len(streams) records")
        self._check(self._L.ht_tracker_import(self._h, C.addressof(ids), n, a.ctypes.data))

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

    def tracker_feed(self, streams, frames, now_ms, width, height, out=None, view=None):
        """One timer tick of each listed stream on its own video frame and clock (ht_tracker_feed): drawImage(video, 0,
        0, width, height) onto the working canvas, then what tracker_step does for that stream.  Unlisted streams do
        not tick.  streams: distinct stream ids; frames: one (h, w, 4) u8 video frame per stream, all numpy arrays or
        all torch CUDA tensors (any size; a row-padded view - last two strides (4, 1) - passes its row stride as the
        pitch); now_ms: one clock for all or one per record; width, height: one canvas for all (ht_tracker_feed) or one
        size per record (ht_tracker_feed_canvases: each stream on its own canvas).  view: None, or a view
        (headtrackr_b200.views: {"rotate", "mirror", "crop"}) for all records or a list of one per record, drawn
        through ht_tracker_feed_views.  -> event dicts in record order; with a torch CUDA `out` tensor of
        len(streams)*144 bytes: asynchronous, nothing returned."""
        streams = list(streams)
        n = len(frames)
        if len(streams) != n or n == 0:
            raise ValueError("one frame per listed stream")
        clocks = [float(t) for t in now_ms] if hasattr(now_ms, "__len__") else [float(now_ms)] * n
        if len(clocks) != n:
            raise ValueError("one clock per listed stream")
        per_record = hasattr(width, "__len__") or hasattr(height, "__len__")
        if per_record:
            widths = [int(v) for v in width] if hasattr(width, "__len__") else [int(width)] * n
            heights = [int(v) for v in height] if hasattr(height, "__len__") else [int(height)] * n
            if len(widths) != n or len(heights) != n:
                raise ValueError("one canvas width and height per listed stream")
        on_device = _is_torch(frames[0])
        recs = (VideoFrame * n)()
        keep = []
        for b, (k, f) in enumerate(zip(streams, frames)):
            if _is_torch(f) != on_device:
                raise ValueError("frames must be all numpy arrays or all torch CUDA tensors")
            ptr, pitch, f = _rgba_frame(f, on_device)
            keep.append(f)
            recs[b] = VideoFrame(ptr, int(k), f.shape[1], f.shape[0], pitch, clocks[b])
        ev = None if out is not None else (TrackerEvent * n)()
        dst = out.data_ptr() if out is not None else C.addressof(ev)
        if view is not None:
            widths = widths if per_record else [int(width)] * n
            heights = heights if per_record else [int(height)] * n
            crecs = (CanvasFrame * n)(*[CanvasFrame(recs[b], widths[b], heights[b]) for b in range(n)])
            views = _views(view, n)
            self._check(self._L.ht_tracker_feed_views(self._h, C.addressof(crecs), C.addressof(views), n, int(on_device), dst))
        elif per_record:
            crecs = (CanvasFrame * n)(*[CanvasFrame(recs[b], widths[b], heights[b]) for b in range(n)])
            self._check(self._L.ht_tracker_feed_canvases(self._h, C.addressof(crecs), n, int(on_device), dst))
        else:
            self._check(self._L.ht_tracker_feed(self._h, C.addressof(recs), n, int(on_device), width, height, dst))
        if out is not None:
            return None
        return [tracker_event_dict(e) for e in ev]

    def tracker_feed_yuv(self, streams, frames, now_ms, width, height, format="nv12", color="bt601", out=None, view=None):
        """tracker_feed on video in any of _lib.YUV_FORMATS (ht_tracker_feed_yuv): each frame is a tuple of 2-D planes
        for a planar format ((Y, UV) for NV12, (Y, U, V) for I420, uint16 planes for P010) or one (h, w, channels)
        array for a packed one (YUYV, UYVY, BGRA, BGR24, RGB24; _yuv_image), numpy arrays or torch tensors (CPU, or
        CUDA for every frame), whose row strides are the pitches.  A decoder's packed NV12 buffer `buf` of
        h + ceil(h/2) rows splits without a copy:
            frame = (buf[:h, :w], buf[h:, :2 * ((w + 1) // 2)])
        The conversion is the library's (DESIGN.md 2): format (a key of _lib.YUV_FORMATS) and color ("bt601",
        "bt709", "bt2020", each optionally "-full"; "bt601" for the packed RGB formats), one for all or one per
        record.  now_ms, width, height and view as for tracker_feed
        (every record has its own canvas here; with a view, ht_tracker_feed_yuv_views).  -> event dicts in record order; with a torch CUDA `out` tensor of
        len(streams)*144 bytes: asynchronous, nothing returned."""
        streams = list(streams)
        n = len(frames)
        if len(streams) != n or n == 0:
            raise ValueError("one frame per listed stream")
        clocks = [float(t) for t in now_ms] if hasattr(now_ms, "__len__") else [float(now_ms)] * n
        widths = [int(v) for v in _per_record(width, n, "canvas width")]
        heights = [int(v) for v in _per_record(height, n, "canvas height")]
        fmts, colors = _per_record(format, n, "format"), _per_record(color, n, "color")
        if len(clocks) != n:
            raise ValueError("one clock per listed stream")
        recs = (YuvFrame * n)()
        keep, where = [], set()
        for b, (k, f) in enumerate(zip(streams, frames)):
            img, on_device = _yuv_image(f, fmts[b], colors[b], keep)
            where.add(on_device)
            recs[b] = YuvFrame(img, int(k), widths[b], heights[b], 0, clocks[b])
        if len(where) != 1:
            raise ValueError("frames must be all host or all device memory")
        ev = None if out is not None else (TrackerEvent * n)()
        dst = out.data_ptr() if out is not None else C.addressof(ev)
        if view is not None:
            views = _views(view, n)
            self._check(self._L.ht_tracker_feed_yuv_views(self._h, C.addressof(recs), C.addressof(views), n, int(where.pop()),
                                                          dst))
        else:
            self._check(self._L.ht_tracker_feed_yuv(self._h, C.addressof(recs), n, int(where.pop()), dst))
        if out is not None:
            return None
        return [tracker_event_dict(e) for e in ev]

    def ingest_yuv(self, frames, width, height, format="nv12", color="bt601", out=None, view=None):
        """drawImage(video, 0, 0, width, height) of video frames (ht_ingest_yuv): frames, format and color as for
        tracker_feed_yuv (the frames may differ in size and format); view as for tracker_feed (ht_ingest_yuv_views).  -> numpy (n, height, width, 4); with a torch `out` tensor
        of that shape (CUDA or CPU) the result is written there."""
        n = len(frames)
        if n == 0:
            raise ValueError("no frames")
        fmts, colors = _per_record(format, n, "format"), _per_record(color, n, "color")
        imgs = (YuvImage * n)()
        keep, where = [], set()
        for b, f in enumerate(frames):
            imgs[b], on_device = _yuv_image(f, fmts[b], colors[b], keep)
            where.add(on_device)
        if len(where) != 1:
            raise ValueError("frames must be all host or all device memory")
        on_device = where.pop()
        if view is not None:
            views = _views(view, n)
            return self._ingest_into(out, n, width, height, lambda dst: self._L.ht_ingest_yuv_views(
                self._h, C.addressof(imgs), C.addressof(views), n, int(on_device), dst, width, height))
        if out is not None:
            if not out.is_contiguous() or tuple(out.shape) != (n, height, width, 4) or out.element_size() != 1:
                raise ValueError(f"out must be a contiguous uint8 tensor of shape {(n, height, width, 4)}")
            self._check(self._L.ht_ingest_yuv(self._h, C.addressof(imgs), n, int(on_device), out.data_ptr(), width, height))
            return out
        dst = np.zeros((n, height, width, 4), np.uint8)
        self._check(self._L.ht_ingest_yuv(self._h, C.addressof(imgs), n, int(on_device), dst.ctypes.data, width, height))
        return dst

    def _ingest_into(self, out, n, width, height, call):
        """call(destination address) writes n width x height canvases: into `out` (a contiguous torch uint8 tensor,
        CUDA or CPU), or into a new numpy array"""
        if out is not None:
            if not out.is_contiguous() or tuple(out.shape) != (n, height, width, 4) or out.element_size() != 1:
                raise ValueError(f"out must be a contiguous uint8 tensor of shape {(n, height, width, 4)}")
            self._check(call(out.data_ptr()))
            return out
        dst = np.zeros((n, height, width, 4), np.uint8)
        self._check(call(dst.ctypes.data))
        return dst

    def ingest(self, frames, width, height, out=None, view=None):
        """drawImage(video, 0, 0, width, height) for a batch (src/main.js:170).  numpy in -> numpy (n, height, width, 4)
        out; with a torch CUDA `out` tensor the result stays on the device.  With a view (as for tracker_feed;
        ht_ingest_views), frames is a list of (h, w, 4) frames of any sizes, all numpy arrays or all torch CUDA
        tensors, and `out` may also be a CPU tensor."""
        if view is not None:
            n = len(frames)
            if n == 0:
                raise ValueError("no frames")
            on_device = _is_torch(frames[0]) and frames[0].is_cuda
            recs = (VideoFrame * n)()
            keep = []
            for b, f in enumerate(frames):
                if (_is_torch(f) and f.is_cuda) != on_device:
                    raise ValueError("frames must be all numpy arrays or all torch CUDA tensors")
                ptr, pitch, a = _rgba_frame(f, on_device)
                keep.append(a)
                recs[b] = VideoFrame(ptr, 0, a.shape[1], a.shape[0], pitch, 0.0)
            views = _views(view, n)
            return self._ingest_into(out, n, width, height, lambda dst: self._L.ht_ingest_views(
                self._h, C.addressof(recs), C.addressof(views), n, int(on_device), dst, width, height))
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


def tracker_params(retryDetection=True, calcAngles=False, smoothing=True, fov=None, cameraOffset=11.5, headPosition=True,
                   edgecorrection=True, alpha=0.35, distance_to_screen=60.0):
    """ht_tracker_params from the reference's parameter names (src/main.js:39-55)"""
    head = HeadParams(int(bool(smoothing)), int(bool(headPosition)), int(bool(edgecorrection)), 0, alpha,
                      float(fov) if fov is not None else 0.0, cameraOffset, distance_to_screen)
    return TrackerParams(int(bool(retryDetection)), int(bool(calcAngles)), (C.c_int32 * 2)(), head)


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
