"""Host mirror of a tracker stream's framing (DESIGN.md 2, "Face crops", item 7; ht_tracker_set_framing): the filter
that glides a steady face-cam box instead of jumping with every camshift box.

The device runs it per stream during the tick (Context.tracker_set_framing, the "framing" key of TrackerSet) on an
ht_framed_box in device memory; this mirror replays it from the tick's records, operation for operation.  Python
floats are IEEE doubles and every operation here rounds once, as the library's (no contraction).

A box is a dict {cx, cy, width, height, canvas_w, canvas_h, updates, valid} as box_from_bytes decodes it; new_box() is
the box a framing starts with.
"""
import math

from . import _lib

# the wrappers' defaults: the C ABI takes explicit values
ALPHA = 0.25
DEAD_ZONE = 0.1

_S = (-1.66666666666666324348e-01, 8.33333333332248946124e-03, -1.98412698298579493134e-04, 2.75573137070700676789e-06,
      -2.50507602534068634195e-08, 1.58969099521155010221e-10)
_C = (4.16666666666666019037e-02, -1.38888888888741095749e-03, 2.48015872894767294178e-05, -2.75573143513906633035e-07,
      2.08757232129817482790e-09, -1.13596475577881948265e-11)


def stroke_sincos(t):
    """(sin t, cos t) as the library's stroke_sincos computes them (DESIGN.md 2, "Strokes"): fdlibm's kernels after a
    three-part Cody-Waite reduction by pi/2; a non-finite t is no rotation, (0, 1)"""
    if not math.isfinite(t):
        return 0.0, 1.0
    k = float(round(t * 6.36619772367581382433e-01))            # rint: ties to even, as Python's round
    r = t + -(k * 1.57079632673412561417e+00)
    r = r + -(k * 6.07710050630396597660e-11)
    r = r + -(k * 2.02226624879595063154e-21)
    z = r * r
    w = z * z
    S1, S2, S3, S4, S5, S6 = _S
    C1, C2, C3, C4, C5, C6 = _C
    sr = (S2 + z * (S3 + z * S4)) + (z * w) * (S5 + z * S6)
    sn = r + (z * r) * (S1 + z * sr)
    cr = z * (C1 + z * (C2 + z * C3)) + (w * w) * (C4 + z * (C5 + z * C6))
    hz = 0.5 * z
    one_hz = 1.0 + -hz
    cs = one_hz + (((1.0 + -one_hz) + -hz) + z * cr)
    q = int(k - 4.0 * math.floor(k * 0.25))
    return ((sn, cs), (cs, -sn), (-sn, -cs), (-cs, sn))[q]


def new_box():
    """the box a framing starts with: not valid, no updates"""
    return dict(cx=0.0, cy=0.0, width=0.0, height=0.0, canvas_w=0, canvas_h=0, updates=0, valid=0)


def crop_tick(record):
    """whether a tracker record (a dict with detection "CS" / 2, x, y, width, height) writes crops and moves a framed
    box: "CS" with width > 0 and height > 0 (and, as the crop map asks, no field non-finite or beyond 65536 px)"""
    det = record.get("detection", 0)
    det = {"VJ": 1, "CS": 2}.get(det, 0) if isinstance(det, str) else int(det)
    f = [float(record[k]) for k in ("x", "y", "width", "height")]
    return det == 2 and f[2] > 0.0 and f[3] > 0.0 and all(abs(v) <= 65536.0 for v in f)


def target(record):
    """(t_x, t_y, t_w, t_h) of a crop tick: the green rectangle's centre as the crop map places it, and the record's
    size"""
    x, y, w, h = (float(record[k]) for k in ("x", "y", "width", "height"))
    s, c = stroke_sincos(float(record["angle"]) + -1.5707963267948966)
    cx = float(math.trunc(-(w / 2))) + w * 0.5
    cy = float(math.trunc(-(h / 2))) + h * 0.5
    return x + (c * cx + -(s * cy)), y + (s * cx + c * cy), w, h


def _glide(v, t, size, alpha, dead_zone):
    band = dead_zone * size
    e = t + -v
    return v + alpha * (e + -math.copysign(band, e)) if abs(e) > band else v


def framing_step(box, record, canvas_w, canvas_h, alpha=ALPHA, dead_zone=DEAD_ZONE):
    """one tick of the framing: box (a dict, updated in place) after `record` on a canvas_w x canvas_h canvas.
    -> whether the tick was a crop tick (otherwise the box is unchanged)"""
    if not crop_tick(record):
        return False
    tx, ty, tw, th = target(record)
    b = box
    if (not b["valid"] or b["canvas_w"] != canvas_w or b["canvas_h"] != canvas_h or abs(tx + -b["cx"]) > b["width"] * 0.5
            or abs(ty + -b["cy"]) > b["height"] * 0.5):
        b.update(cx=tx, cy=ty, width=tw, height=th, canvas_w=int(canvas_w), canvas_h=int(canvas_h), valid=1)
    else:
        ow, oh = b["width"], b["height"]
        b.update(cx=_glide(b["cx"], tx, ow, alpha, dead_zone), cy=_glide(b["cy"], ty, oh, alpha, dead_zone),
                 width=_glide(ow, tw, ow, alpha, dead_zone), height=_glide(oh, th, oh, alpha, dead_zone))
    b["updates"] = (b["updates"] + 1) & 0xFFFFFFFF
    return True


def replay(records, canvas_w, canvas_h, alpha=ALPHA, dead_zone=DEAD_ZONE, box=None):
    """the box after each of `records` (one stream's ticks, each on a canvas_w x canvas_h canvas or on its own
    (canvas_w, canvas_h) when those are lists), from `box` (default new_box()) -> list of box dicts"""
    box = dict(box) if box is not None else new_box()
    out = []
    for i, r in enumerate(records):
        cw = canvas_w[i] if isinstance(canvas_w, (list, tuple)) else canvas_w
        ch = canvas_h[i] if isinstance(canvas_h, (list, tuple)) else canvas_h
        framing_step(box, r, cw, ch, alpha, dead_zone)
        out.append(dict(box))
    return out


def box_struct(box):
    """a box dict -> ht_framed_box"""
    return _lib.FramedBox(box["cx"], box["cy"], box["width"], box["height"], box["canvas_w"], box["canvas_h"],
                          box["updates"], box["valid"])


def box_to_bytes(box):
    """a box dict -> its FRAMED_BOX_BYTES bytes, as the device holds it"""
    return bytes(box_struct(box))


def box_from_bytes(b):
    """an ht_framed_box (FRAMED_BOX_BYTES bytes: numpy, bytes, or a torch tensor, copied to the host) -> box dict"""
    if hasattr(b, "detach"):
        b = b.detach().cpu().numpy()
    raw = bytes(memoryview(b).cast("B")) if not isinstance(b, (bytes, bytearray)) else bytes(b)
    if len(raw) != _lib.FRAMED_BOX_BYTES:
        raise ValueError(f"an ht_framed_box is {_lib.FRAMED_BOX_BYTES} bytes")
    s = _lib.FramedBox.from_buffer_copy(raw)
    return dict(cx=s.cx, cy=s.cy, width=s.width, height=s.height, canvas_w=s.canvas_w, canvas_h=s.canvas_h,
                updates=s.updates, valid=s.valid)


def is_box(record):
    """whether views.crop_map's `record` is a framed box (a box dict or an ht_framed_box) rather than a tracker record"""
    return isinstance(record, _lib.FramedBox) or (isinstance(record, dict) and "cx" in record and "valid" in record)


def as_struct(record):
    """a box dict or an ht_framed_box -> ht_framed_box"""
    return record if isinstance(record, _lib.FramedBox) else box_struct(record)
