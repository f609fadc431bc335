"""Views of video frames (DESIGN.md 2, "Views"): a rotation, a mirror and a crop that the canvas draw applies, and the
map from canvas coordinates back to video pixel coordinates.

A view is a dict {"rotate": 0 | 90 | 180 | 270 (clockwise), "mirror": bool (after the rotation), "crop": (x, y, w, h)
of the oriented frame, or None for all of it}; None is the identity view.  Events are in canvas coordinates, as in
the reference; to_video, box_to_video and cs_to_video give the same points, boxes and tracked objects in the pixel
coordinates of the video as it sits in memory, e.g. to draw an overlay on the decoded frame.

Coordinates here are continuous: pixel (x, y) covers [x, x + 1) x [y, y + 1), so its centre is (x + 0.5, y + 0.5).
"""
import ctypes as C
import math

from . import framing
from ._lib import HT_REDACT_MOSAIC, HT_VIEW_MIRROR, FaceCrop, FaceRedact, TrackerEvent, VideoView, lib

# EXIF orientation tag (1..8) -> view orientation; a tag says how to turn the stored image to show it upright
EXIF_ORIENTATION = {1: 0, 2: 4, 3: 2, 4: 6, 5: 5, 6: 1, 7: 7, 8: 3}


def orientation(view):
    """the ht_video_view orientation (0..7) of a view dict"""
    if view is None:
        return 0
    rotate = view.get("rotate", 0)
    if rotate not in (0, 90, 180, 270):
        raise ValueError(f"rotate must be 0, 90, 180 or 270, not {rotate!r}")
    return rotate // 90 | (HT_VIEW_MIRROR if view.get("mirror", False) else 0)


def from_tag(rotate=0, flip=False):
    """the view of a rotation tag and a horizontal-flip bit (WebRTC rotation, RTP video orientation): rotate first,
    then flip"""
    return {"rotate": rotate, "mirror": bool(flip), "crop": None}


def from_exif(tag):
    """the view of an EXIF orientation tag 1..8"""
    o = EXIF_ORIENTATION[tag]
    return {"rotate": 90 * (o & 3), "mirror": bool(o & HT_VIEW_MIRROR), "crop": None}


def oriented_size(view, width, height):
    """(W', H') of the oriented frame of a width x height video"""
    return (height, width) if orientation(view) & 1 else (width, height)


def video_view(view):
    """a view dict -> ht_video_view (the library checks the crop against each frame)"""
    crop = None if view is None else view.get("crop")
    sx, sy, sw, sh = (0, 0, 0, 0) if crop is None else (int(v) for v in crop)
    if crop is not None and (sw < 1 or sh < 1):
        raise ValueError(f"crop {tuple(crop)} is empty")
    return VideoView(orientation(view), sx, sy, sw, sh)


def _rect(view, width, height):
    W, H = oriented_size(view, width, height)
    crop = None if view is None else view.get("crop")
    return (0, 0, W, H) if crop is None else tuple(crop)


def _oriented_to_video(o, width, height, x, y):
    """a continuous point of the oriented frame -> the video's"""
    W = height if o & 1 else width
    if o & HT_VIEW_MIRROR:
        x = W - x
    r = o & 3
    if r == 0:
        return x, y
    if r == 1:
        return y, height - x
    if r == 2:
        return width - x, height - y
    return width - y, x


def to_video(view, width, height, canvas_w, canvas_h, x, y):
    """a point (x, y) of a canvas_w x canvas_h canvas drawn from a width x height video through `view` -> the video's
    (x, y).  The canvas stretches the crop over the whole canvas, as the draw does."""
    sx, sy, sw, sh = _rect(view, width, height)
    return _oriented_to_video(orientation(view), width, height, sx + x * sw / canvas_w, sy + y * sh / canvas_h)


def box_to_video(view, width, height, canvas_w, canvas_h, x, y, w, h):
    """an axis-aligned canvas box (top-left x, y and size w, h; a "VJ" event) -> the video box (x, y, w, h) it covers"""
    a = to_video(view, width, height, canvas_w, canvas_h, x, y)
    b = to_video(view, width, height, canvas_w, canvas_h, x + w, y + h)
    return min(a[0], b[0]), min(a[1], b[1]), abs(b[0] - a[0]), abs(b[1] - a[1])


def cs_to_video(view, width, height, canvas_w, canvas_h, x, y, w, h, angle):
    """a tracked object of a "CS" event (centre x, y; width w and height h; angle in [0, pi), the direction of its
    height axis as src/camshift.js measures it: atan2(dy, dx) with y pointing down) -> the same object in the video:
    (x, y, w, h, angle) with the same meaning.
    The height axis keeps its length and turns with the view, so a 90 or 270 degree view turns the angle by a quarter
    turn (an upright object, angle pi/2, lies along the video's rows, angle 0) and a mirror negates it.  Width and
    height scale with the canvas-to-crop scale along their axes (exact when the scale is the same in x and y, or the
    object is axis-aligned)."""
    sx, sy, sw, sh = _rect(view, width, height)
    kx, ky = sw / canvas_w, sh / canvas_h
    o = orientation(view)
    cx, cy = to_video(view, width, height, canvas_w, canvas_h, x, y)

    def turn(dx, dy):
        """a canvas direction -> (video direction, its length after the crop scale)"""
        p0 = _oriented_to_video(o, width, height, 0.0, 0.0)
        p1 = _oriented_to_video(o, width, height, dx * kx, dy * ky)
        vx, vy = p1[0] - p0[0], p1[1] - p0[1]
        return (vx, vy), math.hypot(vx, vy)
    # the height axis: (cos a, sin a) on a y-down canvas (the reference's atan2 of canvas moments)
    (hx, hy), lh = turn(math.cos(angle), math.sin(angle))
    _, lw = turn(-math.sin(angle), math.cos(angle))
    a = math.atan2(hy, hx)
    if a < 0:
        a += math.pi
    if a >= math.pi:
        a -= math.pi
    return cx, cy, w * lw, h * lh, a


def crop_map(view, width, height, canvas_w, canvas_h, record, crop_w, crop_h, scale=1.0):
    """ht_face_crop_map: the exact fixed-point map (U0, V0, Ui, Vi, Uj, Vj) of a crop_w x crop_h face crop for a
    tracker record (a dict with detection "CS" / 2, x, y, width, height, angle, or an ht_tracker_event), on a
    canvas_w x canvas_h canvas drawn from a width x height video through `view`; crop pixel (i, j) samples video tap
    coordinates (U0 + i Ui + j Uj, V0 + i Vi + j Vj) / 65536 (tap u is pixel centre u + 0.5).  `record` may also be
    a framed box (a framing.py box dict or an ht_framed_box; ht_face_crop_map_framed): the map of a crop cut from it.
    -> None when the record makes no crop (or the box is not valid)."""
    vv = video_view(view)
    crop = FaceCrop(None, int(crop_w), int(crop_h), 0, 0, float(scale))
    out = (C.c_int64 * 6)()
    if framing.is_box(record):
        box = framing.as_struct(record)
        rc = lib().ht_face_crop_map_framed(C.addressof(box), int(canvas_w), int(canvas_h), int(width), int(height),
                                           C.addressof(vv), C.addressof(crop), out)
        if rc < 0:
            raise ValueError(f"ht_face_crop_map_framed rejected its arguments ({rc})")
        return tuple(out) if rc == 1 else None
    if isinstance(record, TrackerEvent):
        ev = record
    else:
        ev = TrackerEvent()
        det = record.get("detection", 0)
        ev.detection = {"VJ": 1, "CS": 2}.get(det, 0) if isinstance(det, str) else int(det)
        for k in ("x", "y", "width", "height", "angle"):
            setattr(ev, k, float(record[k]))
        ev.confidence = float(record.get("confidence", 1.0))
    rc = lib().ht_face_crop_map(C.addressof(ev), int(canvas_w), int(canvas_h), int(width), int(height), C.addressof(vv),
                                C.addressof(crop), out)
    if rc < 0:
        raise ValueError(f"ht_face_crop_map rejected its arguments ({rc})")
    return tuple(out) if rc == 1 else None


def _event(record):
    """an ht_tracker_event of a record dict (detection "VJ" / "CS" / 1 / 2, x, y, width, height, angle, confidence)"""
    if isinstance(record, TrackerEvent):
        return record
    ev = TrackerEvent()
    det = record.get("detection", 0)
    ev.detection = {"VJ": 1, "CS": 2}.get(det, 0) if isinstance(det, str) else int(det)
    for k in ("x", "y", "width", "height", "angle"):
        setattr(ev, k, float(record.get(k, 0.0)))
    ev.confidence = float(record.get("confidence", 1.0))
    return ev


def redact_rect(view, width, height, canvas_w, canvas_h, record, block=16, scale=1.25):
    """ht_face_redact_rect: the video pixels (x0, y0, x1, y1), half-open, that a face redaction with cells of `block`
    px and `scale` hides for a tracker record (a dict or an ht_tracker_event) on a canvas_w x canvas_h canvas drawn
    from a width x height video through `view`, exactly as the device computes them (DESIGN.md 2, "Face
    redaction").  -> None when the record is not a face tick or the region is empty."""
    vv = video_view(view)
    d = FaceRedact(HT_REDACT_MOSAIC, int(block), 0)
    d.scale = float(scale)
    out, ev = (C.c_int32 * 4)(), _event(record)
    rc = lib().ht_face_redact_rect(C.addressof(ev), int(canvas_w), int(canvas_h), int(width), int(height),
                                   C.addressof(vv), C.addressof(d), out)
    if rc < 0:
        raise ValueError(f"ht_face_redact_rect rejected its arguments ({rc})")
    return tuple(out) if rc == 1 else None


def crop_to_video(view, width, height, canvas_w, canvas_h, record, crop_w, crop_h, scale=1.0):
    """the 2x3 affine ((a, b, c), (d, e, f)) from continuous crop pixel coordinates (p, q) to the video's:
    x = a p + b q + c, y = d p + e q + f, exactly the map the device samples with (crop_map); e.g. to put landmarks
    found in the crop back onto the video; `record` may be a framed box, as for crop_map.  -> None when the record
    makes no crop."""
    m = crop_map(view, width, height, canvas_w, canvas_h, record, crop_w, crop_h, scale)
    if m is None:
        return None
    U0, V0, Ui, Vi, Uj, Vj = m
    # crop pixel centre p = i + 1/2 samples tap u = (U0 + i Ui + j Uj) / 65536, the video coordinate u + 1/2
    return ((Ui / 65536, Uj / 65536, (U0 - (Ui + Uj) / 2) / 65536 + 0.5),
            (Vi / 65536, Vj / 65536, (V0 - (Vi + Vj) / 2) / 65536 + 0.5))
