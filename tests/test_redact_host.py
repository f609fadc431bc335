"""CPU: face redaction (DESIGN.md 2, "Face redaction") through the library's host build (ht_face_redact_rect,
ht_selftest_face_redact, ht_selftest_redact_hold), views.redact_rect and the independent C restatement
tests/redact_oracle.c:

  * the redacted rectangle agrees exactly three ways for every VJ and CS record of every golden, across canvas and
    video sizes, the 8 orientations with and without source rectangles, and scales from 0.01 to 16, and on the edge
    cases: boxes past the canvas, odd videos, a 1 x 1 video, a box over the whole video, empty regions;
  * the host build of k_face_redact's cell code and the restatement agree byte for byte on all 11 formats and RGBA8
    frames, both modes and several cell sizes, on random frames whose pitch padding and alpha come back unchanged;
  * numpy checks on hand-sized frames: the cell means, the grid anchored at (0, 0), the chroma spans of clipped cells,
    and that no sample belongs to two cells;
  * the hold over the lost-and-found sequence of reference_js_main.json;
  * the ABI, the record checks, and a spill-free k_face_redact."""
import ctypes as C
import json
import random
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib, views
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_framing_host import golden_sequences
from test_views_host import view_of

GOLDEN = Path(__file__).resolve().parent / "golden"
HALF_PI = 1.5707963267948966
# format -> (tight row bytes, rows) per plane of a w x h frame; -1 is an RGBA8 frame
FORMATS = {-1: "rgba", 0: "nv12", 1: "i420", 16: "nv21", 17: "i422", 18: "i444", 19: "yuyv", 20: "uyvy", 21: "p010",
           32: "bgra", 33: "bgr24", 34: "rgb24"}


def plane_shapes(fmt, w, h):
    cw, ch = (w + 1) // 2, (h + 1) // 2
    return {-1: [(4 * w, h)], 0: [(w, h), (2 * cw, ch)], 16: [(w, h), (2 * cw, ch)], 1: [(w, h), (cw, ch), (cw, ch)],
            17: [(w, h), (cw, h), (cw, h)], 18: [(w, h)] * 3, 19: [(4 * cw, h)], 20: [(4 * cw, h)],
            21: [(2 * w, h), (4 * cw, ch)], 32: [(4 * w, h)], 33: [(3 * w, h)], 34: [(3 * w, h)]}[fmt]


@pytest.fixture(scope="module")
def ro(tmp_path_factory):
    """tests/redact_oracle.c built into a temporary directory, without contraction"""
    lib = tmp_path_factory.mktemp("redact_oracle") / "libredact_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(lib),
                           str(Path(__file__).with_name("redact_oracle.c")), "-lm"])
    L = C.CDLL(str(lib))
    L.hro_rect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double,
                           C.c_void_p]
    L.hro_hold.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.hro_redact.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_selftest_face_redact.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]
    st.ht_selftest_redact_hold.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    st.ht_face_redact_rect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return st


def event(r):
    e = _lib.TrackerEvent()
    det = r["detection"]
    e.detection = {"VJ": 1, "CS": 2}.get(det, det) if isinstance(det, str) else int(det)
    e.x, e.y, e.width, e.height = r["x"], r["y"], r["width"], r["height"]
    e.angle, e.confidence = r.get("angle", 0.0), r.get("confidence", 1.0)
    return e


def rec_array(r):
    e = event(r)
    return (C.c_double * 7)(e.detection, e.x, e.y, e.width, e.height, e.angle, e.confidence)


def redaction(mode=1, block=16, scale=1.25, hold=0, fill_rgb=(0, 0, 0), fill_yuv=(16, 128, 128)):
    d = _lib.FaceRedact(mode, block, hold)
    d.fill_rgb[:], d.fill_yuv[:], d.scale = list(fill_rgb), list(fill_yuv), scale
    return d


def resolved(o, w, h, crop):
    """the oriented frame's source rectangle {sx, sy, sw, sh} of a view"""
    W, H = (h, w) if o & 1 else (w, h)
    return crop if crop[2] else (0, 0, W, H)


def three_rects(lib, ro, r, cw, ch, w, h, o, crop, B, scale):
    """the rectangle from ht_face_redact_rect, views.redact_rect and the restatement; all three must agree"""
    e, d, v = event(r), redaction(block=B, scale=scale), view_of(o, crop)
    out = (C.c_int32 * 4)()
    rc = lib.ht_face_redact_rect(C.addressof(e), cw, ch, w, h, C.addressof(v), C.addressof(d), out)
    vd = {"rotate": 90 * (o & 3), "mirror": bool(o & 4), "crop": crop if crop[2] else None}
    py = views.redact_rect(vd, w, h, cw, ch, r, B, scale)
    oo = (C.c_int32 * 4)()
    oc = ro.hro_rect(rec_array(r), cw, ch, w, h, o, (C.c_int32 * 4)(*resolved(o, w, h, crop)), B, scale, oo)
    a = tuple(out) if rc == 1 else None
    assert rc in (0, 1) and a == py == (tuple(oo) if oc else None), (r, cw, ch, w, h, o, crop, B, scale, a, py, tuple(oo))
    return a


def golden_records():
    out = []
    for _, seq in golden_sequences():
        out += [r for r in seq if r["detection"] in (1, 2)]
    return out


def test_rect_agrees_three_ways_on_every_golden_record(lib, ro):
    rng = random.Random(5)
    canvases = [(320, 240), (160, 120), (300, 260), (97, 61)]
    videos = [(640, 480), (1280, 720), (321, 241), (57, 33), (1, 1)]
    scales = [0.01, 0.5, 1.0, 1.25, 2.0, 16.0]
    nonempty = 0
    for r in golden_records():
        for _ in range(6):
            cw, ch = rng.choice(canvases)
            w, h = rng.choice(videos)
            o = rng.randrange(8)
            W, H = (h, w) if o & 1 else (w, h)
            crop = (0, 0, 0, 0)
            if rng.random() < 0.5 and W > 1 and H > 1:
                sw, sh = rng.randint(1, W), rng.randint(1, H)
                crop = (rng.randint(0, W - sw), rng.randint(0, H - sh), sw, sh)
            nonempty += three_rects(lib, ro, r, cw, ch, w, h, o, crop, rng.choice([2, 4, 16, 34, 128]),
                                    rng.choice(scales)) is not None
    assert nonempty > 500


def test_rect_edge_cases(lib, ro):
    cs = dict(detection="CS", x=160.0, y=120.0, width=40.0, height=60.0, angle=HALF_PI)
    # a box over the whole video: every cell, clipped to the video
    assert three_rects(lib, ro, dict(cs, width=400.0, height=400.0), 320, 240, 641, 481, 0, (0, 0, 0, 0), 16, 1.0) == \
        (0, 0, 641, 481)
    # past the canvas's edges: clipped, then whole cells
    r = three_rects(lib, ro, dict(cs, x=-5.0, y=235.0), 320, 240, 640, 480, 0, (0, 0, 0, 0), 16, 1.0)
    assert r[0] == 0 and r[3] == 480 and r[2] % 16 == 0 and r[1] % 16 == 0
    # wholly outside the canvas: empty
    assert three_rects(lib, ro, dict(cs, x=-500.0), 320, 240, 640, 480, 0, (0, 0, 0, 0), 16, 1.0) is None
    assert three_rects(lib, ro, dict(cs, y=5000.0), 320, 240, 640, 480, 5, (0, 0, 0, 0), 16, 1.0) is None
    # a 1 x 1 video, odd videos, every orientation
    for o in range(8):
        assert three_rects(lib, ro, cs, 320, 240, 1, 1, o, (0, 0, 0, 0), 2, 1.0) == (0, 0, 1, 1)
        r = three_rects(lib, ro, cs, 320, 240, 333, 211, o, (0, 0, 0, 0), 8, 1.0)
        assert r[0] % 8 == 0 and r[1] % 8 == 0 and (r[2] % 8 == 0 or r[2] in (333, 211)) and r[2] > r[0]
    # not a face tick: IDLE, WB, confidence 0, a lost CS, a non-finite or huge box
    for bad in (dict(cs, detection=0), dict(cs, detection=3), dict(cs, confidence=0.0), dict(cs, width=0.0),
                dict(cs, height=-1.0), dict(cs, x=float("nan")), dict(cs, y=70000.0)):
        assert three_rects(lib, ro, bad, 320, 240, 640, 480, 0, (0, 0, 0, 0), 16, 1.0) is None
    # a NaN angle is unrotated, as the strokes draw it; a VJ box is upright from its corner
    assert three_rects(lib, ro, dict(cs, angle=float("nan")), 320, 240, 320, 240, 0, (0, 0, 0, 0), 2, 1.0) == \
        (140, 90, 180, 150)
    assert three_rects(lib, ro, dict(cs, detection="VJ", angle=0.0), 320, 240, 320, 240, 0, (0, 0, 0, 0), 2, 1.0) == \
        (160, 120, 200, 180)
    # a view's source rectangle: the cells stay on the video's grid and are clipped to the rectangle
    r = three_rects(lib, ro, dict(cs, width=400.0, height=400.0), 320, 240, 640, 480, 0, (13, 7, 301, 203), 16, 1.0)
    assert r == (13, 7, 314, 210)


def test_rect_rejections(lib):
    e, v, out = event(dict(detection=2, x=10.0, y=10.0, width=5.0, height=5.0)), view_of(0), (C.c_int32 * 4)()
    for d in (redaction(block=3), redaction(block=0), redaction(block=130), redaction(hold=-1), redaction(hold=65536),
              redaction(scale=0.0), redaction(scale=16.5), redaction(scale=float("nan"))):
        assert lib.ht_face_redact_rect(C.addressof(e), 32, 32, 32, 32, C.addressof(v), C.addressof(d), out) == _lib.HT_ERR_ARG
    for field in ("pad0", "pad1", "pad_"):
        d = redaction()
        setattr(d, field, 1)
        assert lib.ht_face_redact_rect(C.addressof(e), 32, 32, 32, 32, C.addressof(v), C.addressof(d), out) == _lib.HT_ERR_ARG
    d = redaction()
    assert lib.ht_face_redact_rect(C.addressof(e), 0, 32, 32, 32, C.addressof(v), C.addressof(d), out) == _lib.HT_ERR_SIZE
    assert lib.ht_face_redact_rect(C.addressof(e), 32, 32, 32, 16385, C.addressof(v), C.addressof(d), out) == _lib.HT_ERR_SIZE
    assert lib.ht_face_redact_rect(C.addressof(e), 32, 32, 32, 32, C.addressof(view_of(8)), C.addressof(d), out) == \
        _lib.HT_ERR_ARG
    assert lib.ht_face_redact_rect(None, 32, 32, 32, 32, None, C.addressof(d), out) == _lib.HT_ERR_ARG
    assert lib.ht_face_redact_rect(C.addressof(e), 32, 32, 32, 32, None, C.addressof(d), out) == 1   # NULL view: whole


# ---- the cells ----------------------------------------------------------------------------------------------------------

class Frame:
    """a random frame of a format: each plane a padded byte array (random padding), pitch = row bytes + pad"""

    def __init__(self, rng, fmt, w, h):
        self.fmt, self.w, self.h = fmt, w, h
        self.bufs, self.pitch, self.rows = [], [], []
        for bytes_, rows in plane_shapes(fmt, w, h):
            pad = int(rng.integers(0, 5)) * 2
            self.bufs.append(rng.integers(0, 256, (rows, bytes_ + pad), dtype=np.uint8))
            self.pitch.append(bytes_ + pad)
            self.rows.append(bytes_)

    def copy(self):
        c = Frame.__new__(Frame)
        c.__dict__ = dict(self.__dict__, bufs=[b.copy() for b in self.bufs])
        return c

    def ptrs(self):
        p = [b.ctypes.data for b in self.bufs] + [0] * (3 - len(self.bufs))
        return (C.c_void_p * 3)(*p), (C.c_int32 * 3)(*(self.pitch + [0] * (3 - len(self.pitch))))

    def api(self):
        """(ht_yuv_image, None) or (None, ht_video_frame)"""
        if self.fmt == -1:
            return None, _lib.VideoFrame(self.bufs[0].ctypes.data, 0, self.w, self.h, self.pitch[0], 0.0)
        p, q = self.ptrs()
        img = _lib.YuvImage()
        img.planes[:] = list(p)
        img.pitch[:] = list(q)
        img.width, img.height, img.format = self.w, self.h, self.fmt
        img.color = 0
        return img, None

    def padding(self):
        return [b[:, n:].copy() for b, n in zip(self.bufs, self.rows)]


def lib_redact(lib, fr, r, cw, ch, o, crop, d, hold=None):
    img, rgba = fr.api()
    v, e = view_of(o, crop), event(r)
    return lib.ht_selftest_face_redact(C.addressof(e), cw, ch, C.addressof(img) if img else None,
                                       C.addressof(rgba) if rgba else None, C.addressof(v), C.addressof(d),
                                       None if hold is None else C.addressof(hold))


def oracle_redact(ro, fr, rect, d):
    p, q = fr.ptrs()
    assert ro.hro_redact(fr.fmt, p, q, (C.c_int32 * 4)(*rect), d.mode, d.block, C.addressof(d.fill_rgb),
                         C.addressof(d.fill_yuv)) == 1


@pytest.mark.parametrize("fmt", sorted(FORMATS), ids=[FORMATS[f] for f in sorted(FORMATS)])
def test_cells_agree_byte_for_byte_on_every_format(lib, ro, fmt):
    rng = np.random.default_rng(100 + fmt)
    prng = random.Random(fmt)
    cases = 0
    for w, h in ((64, 48), (97, 61), (33, 17), (2, 2)):
        for mode in (1, 2):
            for B in (2, 6, 16, 128):
                o = prng.randrange(8)
                W, H = (h, w) if o & 1 else (w, h)
                crop = (0, 0, 0, 0)
                if prng.random() < 0.5 and W > 2 and H > 2:
                    crop = (1, 1, W - 2, H - 1)
                cw, ch = prng.choice([(40, 30), (64, 48), (17, 11)])
                r = dict(detection=prng.choice([1, 2]), x=prng.uniform(0, cw), y=prng.uniform(0, ch),
                         width=prng.uniform(2, cw), height=prng.uniform(2, ch), angle=prng.uniform(0, 3.2))
                d = redaction(mode, B, prng.choice([0.5, 1.25, 3.0]), 0, [prng.randrange(256) for _ in range(3)],
                              [prng.randrange(256) for _ in range(3)])
                fr = Frame(rng, fmt, w, h)
                ours, want, pad = fr.copy(), fr.copy(), fr.padding()
                rc = lib_redact(lib, ours, r, cw, ch, o, crop, d)
                rect = three_rects(lib, ro, r, cw, ch, w, h, o, crop if crop[2] else (0, 0, 0, 0), B, d.scale)
                assert rc == (rect is not None)
                if rect is not None:
                    oracle_redact(ro, want, rect, d)
                    cases += 1
                for a, b in zip(ours.bufs, want.bufs):
                    assert np.array_equal(a, b), (fmt, w, h, mode, B, o, crop, rect)
                assert all(np.array_equal(a, b) for a, b in zip(ours.padding(), pad))       # pitch padding untouched
                if fmt in (-1, 32):                                                             # alpha untouched
                    assert np.array_equal(ours.bufs[0][:, 3:4 * w:4], fr.bufs[0][:, 3:4 * w:4])
                if rect is not None and mode == 2 and fmt == 21:                              # P010 fill: v << 8
                    y = ours.bufs[0][:, :2 * w].view("<u2")
                    assert y[rect[1], rect[0]] == d.fill_yuv[0] << 8
    assert cases > 15


def test_cell_means_grid_and_chroma_spans_by_hand(lib):
    """I420 31 x 21, cells of 4 over video rectangle [5, 27) x [3, 18) from a 1:1 canvas: numpy's cell means"""
    rng = np.random.default_rng(3)
    fr = Frame(rng, 1, 31, 21)
    ours = fr.copy()
    r = dict(detection=1, x=5.0, y=3.0, width=22.0, height=15.0)
    assert lib_redact(lib, ours, r, 31, 21, 0, (0, 0, 0, 0), redaction(block=4, scale=1.0)) == 1
    Y, U, V = (b[:, :n].astype(np.int64) for b, n in zip(fr.bufs, fr.rows))
    want = [Y.copy(), U.copy(), V.copy()]
    x0, y0, x1, y1 = 4, 0, 28, 20                # the cells the rectangle meets: grid lines at multiples of 4
    owner = [np.zeros(a.shape, np.int64) for a in want]
    cell = 0
    for cy in range(y0, y1, 4):
        for cx in range(x0, x1, 4):
            cell += 1
            X0, Y0, X1, Y1 = cx, cy, min(cx + 4, 31), min(cy + 4, 21)
            for k, (a, s) in enumerate(zip((Y, U, V), (0, 1, 1))):
                i0, i1, j0, j1 = X0 >> s, ((X1 - 1) >> s) + 1, Y0 >> s, ((Y1 - 1) >> s) + 1
                blk = a[j0:j1, i0:i1]
                want[k][j0:j1, i0:i1] = (blk.sum() + blk.size // 2) // blk.size
                assert (owner[k][j0:j1, i0:i1] == 0).all()       # no sample belongs to two cells
                owner[k][j0:j1, i0:i1] = cell
    for k in range(3):
        assert np.array_equal(ours.bufs[k][:, :fr.rows[k]], want[k]), k
    # the grid is the video's: the same face one pixel to the right covers the same cells
    other = fr.copy()
    assert lib_redact(lib, other, dict(r, x=6.0, width=21.0), 31, 21, 0, (0, 0, 0, 0), redaction(block=4, scale=1.0)) == 1
    assert all(np.array_equal(a, b) for a, b in zip(other.bufs, ours.bufs))
    # a clipped cell at an odd edge (a source rectangle from x = 3) covers the chroma sample of pixels 2 and 3
    clip = fr.copy()
    assert lib_redact(lib, clip, dict(r, x=0.0, width=6.0), 28, 21, 0, (3, 0, 28, 21),
                      redaction(mode=2, block=4, scale=1.0, fill_yuv=(1, 2, 3))) == 1
    assert (clip.bufs[0][:20, 3:12] == 1).all() and (clip.bufs[0][:, :3] == fr.bufs[0][:, :3]).all()
    assert (clip.bufs[0][20:] == fr.bufs[0][20:]).all() and (clip.bufs[0][:, 12:] == fr.bufs[0][:, 12:]).all()
    assert (clip.bufs[1][:10, 1:6] == 2).all() and (clip.bufs[1][:, 0] == fr.bufs[1][:, 0]).all()
    assert (clip.bufs[2][:10, 1:6] == 3).all() and (clip.bufs[2][10:] == fr.bufs[2][10:]).all()


# ---- the hold -----------------------------------------------------------------------------------------------------------

def main_golden_records():
    """reference_js_main.json's "default" case as tracker records: WB ticks, VJ ticks without a face, and its CS
    facetrackingEvents (the lost one with width 0)"""
    case = json.loads((GOLDEN / "reference_js_main.json").read_text())["cases"][0]
    out = []
    for s in case["steps"]:
        ev = [e for e in s["events"] if e["type"] == "facetrackingEvent"]
        if ev:
            e = ev[0]
            out.append(dict(detection=2, x=e["x"], y=e["y"], width=e["width"], height=e["height"], angle=e["angle"],
                            confidence=1.0))
        elif s["status"] == "whitebalance":
            out.append(dict(detection=3, x=0.0, y=0.0, width=0.0, height=0.0, angle=0.0, confidence=-10000.0))
        else:
            out.append(dict(detection=1, x=0.0, y=0.0, width=0.0, height=0.0, angle=0.0, confidence=-10000.0))
    return out


def hold_run(lib, ro, recs, hold, canvases=None):
    """(redacts, box) per tick from the library's host build and the restatement, which must agree"""
    n = lib.ht_selftest_redact_hold_bytes()
    assert n == 56
    ls, os_ = (C.c_char * n)(), (C.c_char * n)()
    out = []
    for t, r in enumerate(recs):
        cw, ch = canvases[t] if canvases else (320, 240)
        e = event(r)
        a = lib.ht_selftest_redact_hold(ls, hold, C.addressof(e), cw, ch)
        b = ro.hro_hold(os_, hold, rec_array(r), cw, ch)
        assert a == b and bytes(ls) == bytes(os_), (t, r)
        box = np.frombuffer(bytes(ls)[:40], np.float64)
        out.append((a, tuple(box)))
    return out


def test_hold_over_the_main_golden_lost_and_found(lib, ro):
    recs = main_golden_records()
    lost = next(t for t, r in enumerate(recs) if r["detection"] == 2 and r["width"] == 0)
    found = [t for t, r in enumerate(recs) if r["detection"] == 2 and r["width"] > 0]
    assert found[0] == 16 and lost == 28 and found[found.index(27) + 1] == 32
    last = recs[27]
    for hold in (0, 3, 10):
        run = hold_run(lib, ro, recs, hold)
        on = [t for t, (a, _) in enumerate(run) if a]
        assert on == [t for t in range(len(recs)) if t in found or 28 <= t < 28 + min(hold, 4)], hold
        for t in range(28, 28 + min(hold, 4)):     # the gap redacts the last face box
            assert run[t][1] == (last["x"], last["y"], last["width"], last["height"], last["angle"])
    # an IDLE tick and a canvas-size change end the hold
    idle = dict(recs[0], detection=0)
    run = hold_run(lib, ro, recs[:28] + [idle] + recs[28:31], 10)
    assert [a for a, _ in run[28:]] == [0, 0, 0, 0]
    canv = [(320, 240)] * 28 + [(160, 120)] * 3
    run = hold_run(lib, ro, recs[:31], 10, canv)
    assert [a for a, _ in run[28:]] == [0, 0, 0]


def test_held_ticks_redact_the_stored_box_through_their_own_view(lib, ro):
    rng = np.random.default_rng(9)
    face = dict(detection=2, x=30.0, y=20.0, width=12.0, height=16.0, angle=1.2, confidence=1.0)
    lost = dict(face, width=0.0, height=0.0)
    hold = (C.c_char * 56)()
    d = redaction(mode=2, block=4, scale=1.0, hold=2, fill_rgb=(9, 8, 7))
    fr = Frame(rng, -1, 64, 48)
    assert lib_redact(lib, fr.copy(), face, 64, 48, 0, (0, 0, 0, 0), d, hold) == 1
    for o in (3, 6):                                # the next two ticks: lost, on other views
        ours, want = fr.copy(), fr.copy()
        assert lib_redact(lib, ours, lost, 64, 48, o, (0, 0, 0, 0), d, hold) == 1
        rect = three_rects(lib, ro, face, 64, 48, 64, 48, o, (0, 0, 0, 0), 4, 1.0)
        oracle_redact(ro, want, rect, d)
        assert np.array_equal(ours.bufs[0], want.bufs[0])
    assert lib_redact(lib, fr.copy(), lost, 64, 48, 0, (0, 0, 0, 0), d, hold) == 0   # the hold is spent


# ---- ABI and build ------------------------------------------------------------------------------------------------------

def test_abi_layout():
    R = _lib.FaceRedact
    assert C.sizeof(R) == 32
    assert [getattr(R, f).offset for f in ("mode", "block", "hold", "fill_rgb", "pad0", "fill_yuv", "pad1", "pad_",
                                           "scale")] == [0, 4, 8, 12, 15, 16, 19, 20, 24]
    hdr = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    for name, v in (("HT_REDACT_OFF", 0), ("HT_REDACT_MOSAIC", 1), ("HT_REDACT_FILL", 2)):
        assert re.search(rf"#define {name} {v}\b", hdr) and getattr(_lib, name) == v
    for f in ("ht_tracker_set_redact", "ht_face_redact_rect"):
        assert f in _lib.EXPORTS and f in hdr


def test_k_face_redact_does_not_spill(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    m = re.search(r"Compiling entry function '\w*k_face_redact\w*'.*?\n.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill "
                  r"stores, (\d+) bytes spill loads", out)
    assert m and m.groups() == ("0", "0", "0"), out[-2000:]
