"""CPU: camshift on faces that move - out of the canvas at every edge and corner, left and up by non-integer steps,
in jumps wider than the search window, towards the camera and away to a few pixels - against the reference.

The motion corpus is built here by code (tests/test_gpu_track_motion.py imports it): a face on a background that
shares few of its colour bins, moved along scripted paths that scale with the canvas, tracked from rectangles that
start on the face, partly outside the canvas or wholly outside it.  These inputs reach the parts of meanShift and
camShift (src/camshift.js:222-312) that a face staying near where it started never does:

* search windows with x or y < 0 (wadx = max(x, 0) clips them, vx counts from the clipped origin), windows reaching
  past W or H, and empty ones (x >= W, or a width of 0 after a lost face): m00 = 0, NaN shifts that `>> 0` turns into
  0, width and height 0;
* leftward and upward shifts, where `(xc - w/2) >> 0` truncates toward zero, not down;
* calls that stop at the ten-pass cap without converging, and the clamps of :253-254 and :308-309;
* windows narrower than 4 pixels, wider than 128 and shorter than 16 rows, which k_track splits into partial vector
  groups, several column blocks, or fewer rows than its warps.

tests/golden/reference_js_motion.json (tools/make_goldens_motion.py) holds what the unmodified camshift.js returns on
the corpus at 160x120 and 162x122; the oracle must replay it bit for bit.  The oracle's per-pass trace then shows that
the corpus takes each of the paths above at every canvas size the GPU test runs.
"""
import hashlib
import json
import math
from functools import lru_cache
from pathlib import Path

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth

GOLD_PATH = Path(__file__).resolve().parent / "golden" / "reference_js_motion.json"
T = 36                                      # frames per clip
SIZES = [(160, 120), (320, 240), (333, 251), (640, 480), (1280, 720)]


# ------------------------------------------------------------------------------------------------------------------
# frames

def _tint(t):
    """synth.frame's skin tint of a grey template: red >= green >= blue, so blue >> 4 <= 9"""
    t = t.astype(np.int32)
    return np.stack([t, (t * 200) >> 8, (t * 150) >> 8], axis=-1).astype(np.uint8)


@lru_cache(maxsize=64)
def _face(side):
    return _tint(synth.shim_resize(synth.face_template(), side, side))


@lru_cache(maxsize=4)
def background(W, H, specks=True):
    """Blue noise (blue >> 4 >= 10, so no bin of the face) with one pixel in 400 in a face colour: the face's bins are
    rarely all its own, so their weights min(model / current, 1) are fractions and mass centres fall between pixels.
    Without the specks, a window that the face has left holds no weight at all."""
    rng = np.random.Generator(np.random.PCG64(0x5EED + 7919 * W + H))
    out = np.empty((H, W, 4), np.uint8)
    out[..., 0] = rng.integers(0, 64, (H, W))
    out[..., 1] = rng.integers(64, 128, (H, W))
    out[..., 2] = rng.integers(160, 256, (H, W))
    out[..., 3] = 255
    speck = (rng.integers(0, 400, (H, W)) == 0) & specks
    out[speck, :3] = _tint(rng.integers(40, 256, int(speck.sum())))
    out.setflags(write=False)
    return out


def paste(out, x, y, side):
    """The face with its top-left corner at (x, y), clipped to the canvas on every side."""
    H, W = out.shape[:2]
    f = _face(side)
    x0, y0, x1, y1 = max(x, 0), max(y, 0), min(x + side, W), min(y + side, H)
    if x1 > x0 and y1 > y0:
        out[y0:y1, x0:x1, :3] = f[y0 - y:y1 - y, x0 - x:x1 - x]


# Scripted paths: t -> (centre x / W, centre y / H, side / H), or None (no face).  Steps are in canvas fractions, so a
# path moves by a non-integer number of pixels per frame at every size.
def _lin(a, b, t, t0, t1):
    u = min(max((t - t0) / (t1 - t0), 0.0), 1.0)
    return a + (b - a) * u


PATHS = {
    # out of the canvas at every edge, then the calls go on with the face gone
    "exit_left": lambda t: (_lin(0.5, -0.35, t, 4, 28), 0.5, 0.3),
    "exit_right": lambda t: (_lin(0.45, 1.35, t, 4, 28), 0.52, 0.3),
    "exit_top": lambda t: (0.48, _lin(0.5, -0.3, t, 4, 26), 0.32),
    "exit_bottom": lambda t: (0.53, _lin(0.45, 1.3, t, 4, 26), 0.32),
    "exit_corner": lambda t: (_lin(0.5, -0.3, t, 2, 30), _lin(0.5, -0.35, t, 2, 30), 0.28),
    # slow drift left and up, 0.37 % of the width and 0.53 % of the height per frame
    "drift": lambda t: (0.62 - 0.0037 * t, 0.6 - 0.0053 * t, 0.27),
    # jumps of more than a window: left, down-right, up-left, right, each held for a few frames
    "jump": lambda t: ([(0.72, 0.5), (0.3, 0.42), (0.62, 0.7), (0.25, 0.3), (0.7, 0.45), (0.4, 0.62)][t // 6]
                       + (0.22,)),
    # towards the camera, then away until the face is a few pixels
    "zoom": lambda t: (0.5 - 0.002 * t, 0.5 + 0.0013 * t,
                       _lin(0.18, 0.75, t, 0, 12) if t < 12 else _lin(0.75, 0.02, t, 12, 34)),
    # out at the right, gone, back in from the left
    "reenter": lambda t: None if 18 <= t < 24 else
    ((_lin(0.5, 1.3, t, 2, 18), 0.5, 0.3) if t < 18 else (_lin(-0.2, 0.4, t, 24, 34), 0.46, 0.3)),
}


# For headtrackr.Tracker (tests/test_gpu_track_motion.py): the face holds still at the centre while the whitebalance
# gate fills and the head diagonal settles, walks off the canvas across one edge or corner - through the 11-pixel
# margin where headposition corrects the face box - stays away, and comes back to the centre.  On a background without
# specks of face colour, so that the tracker loses the face once it has left (and does not settle on specks).
def _walk(ex, ey):
    return lambda t: (None if 52 <= t < 58 else (0.5, 0.5, 0.3) if t < 28 or t >= 58 else
                      (_lin(0.5, ex, t, 28, 52), _lin(0.5, ey, t, 28, 52), 0.3))


LIFE_PATHS = {"walk_left": _walk(-0.4, 0.5), "walk_right": _walk(1.4, 0.5), "walk_top": _walk(0.5, -0.4),
              "walk_bottom": _walk(0.5, 1.4), "walk_corner": _walk(-0.4, -0.4)}
LIFE_T = 70


def face_box(path, t, W, H):
    """-> (x, y, side) of the face in frame t (top-left corner, may lie outside the canvas), or None"""
    p = (PATHS[path] if path in PATHS else LIFE_PATHS[path])(t)
    if p is None:
        return None
    cx, cy, s = p
    side = max(2, int(round(s * H)))
    return int(math.floor(cx * W - side / 2)), int(math.floor(cy * H - side / 2)), side


def frame(path, t, W, H):
    out = background(W, H, path in PATHS).copy()
    box = face_box(path, t, W, H)
    if box is not None:
        paste(out, *box)
    return out


# Tracked rectangles: the face of frame 0, or one that starts partly or wholly outside the canvas.  All within +-2 W / H:
# far outside that, wadx + sw would overflow in the reference too.
def init_rect(kind, path, W, H):
    x, y, s = face_box(path, 0, W, H)
    return {
        "face": (x, y, s, s),
        "neg": (x - s, y - s, 2 * s, 2 * s),                     # x, y < 0 when the face is near the top-left
        "corner": (-s // 2, -s // 3, s, s),                       # x, y < 0: the top-left corner of the canvas
        "past": (W - s // 3, H - s // 4, s, s),                   # x + w > W, y + h > H
        "sliver": (W - 3, H - 2, s, s),                           # a window 3 pixels wide and 2 rows high
        "right": (W + 3, y, s, s),                                # x >= W: the first window is empty
        "far": (-2 * W + s, -H, s, 2 * H),                        # wholly outside, above and to the left
    }[kind]


# (name, path, init rect kind)
CASES = [(p, p, "face") for p in PATHS] + [
    ("corner_init", "exit_corner", "corner"),
    ("neg_init", "drift", "neg"),
    ("past_init", "exit_bottom", "past"),
    ("sliver_init", "exit_right", "sliver"),
    ("right_init", "drift", "right"),
    ("far_init", "zoom", "far"),
]
CASE = {c[0]: c for c in CASES}


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------------------------
# the oracle on the corpus

def oracle_run(name, W, H, calc, n_calls, frames=None):
    """-> per frame, per call: (TrackTrace, track object, search window before the call, search window after)"""
    _, path, kind = CASE[name]
    ot = oracle.CamshiftTracker(calc_angles=calc)
    ot.init_tracker(frame(path, 0, W, H) if frames is None else frames[0], *init_rect(kind, path, W, H))
    out = []
    for t in range(T):
        f = frame(path, t, W, H) if frames is None else frames[t]
        calls = []
        for _ in range(n_calls):
            before = ot.search_window()
            tr = ot.track(f)
            calls.append((tr, ot.track_obj(), before, ot.search_window()))
        out.append(calls)
    return out


def load_golden():
    return json.loads(GOLD_PATH.read_text())


# ------------------------------------------------------------------------------------------------------------------
# replay of the reference's results

def replay(lib, case):
    """The case through an oracle library (oracle.lib(), or a mutant of it): -> per frame, per call, (obj, window)"""
    import ctypes as C
    W, H = case["W"], case["H"]
    t = oracle.binding.Tracker()
    p = C.POINTER(C.c_uint8)
    f0 = np.ascontiguousarray(frame(case["path"], 0, W, H))
    if lib.hto_tracker_init(C.byref(t), f0.ctypes.data_as(p), W, H, *case["rect"], int(case["calc_angles"])) != 0:
        raise ValueError("empty rectangle")
    out = []
    for n in range(T):
        f = np.ascontiguousarray(frame(case["path"], n, W, H))
        calls = []
        for _ in range(case["n_calls"]):
            lib.hto_tracker_track(C.byref(t), f.ctypes.data_as(p), W, H, None)
            calls.append(([t.tx, t.ty, t.tw, t.th, t.angle], [t.sx, t.sy, t.sw, t.sh]))
        out.append(calls)
    return out


def same_angle(a, b):
    return (a != a and b != b) or a == b


def first_difference(case, got):
    """-> None when `got` (replay's result) equals the golden case bit for bit, else where it first differs"""
    for n, (calls, want) in enumerate(zip(got, case["frames"])):
        for c, ((obj, win), w) in enumerate(zip(calls, want)):
            if obj[:4] != w["obj"][:4] or win != w["window"] or not same_angle(obj[4], w["obj"][4]):
                return (n, c, obj, win, w)
    return None


def case_id(case):
    return f"{case['name']}-{case['W']}x{case['H']}-{'angles' if case['calc_angles'] else 'noangles'}-x{case['n_calls']}"


_GOLD = load_golden() if GOLD_PATH.exists() else {"frames": [], "cases": []}


def test_corpus_frames_match_the_golden():
    """The corpus builds the frames the golden was made from (their hashes), and the golden covers every case."""
    assert _GOLD["T"] == T
    for size in _GOLD["frames"]:
        W, H = size["W"], size["H"]
        assert set(size["sha256"]) == set(PATHS)
        for path, hashes in size["sha256"].items():
            assert [sha(frame(path, t, W, H)) for t in range(T)] == hashes, (path, W, H)
    for case in _GOLD["cases"]:
        _, path, kind = CASE[case["name"]]
        assert (case["path"], case["rect_kind"]) == (path, kind)
        assert tuple(case["rect"]) == init_rect(kind, path, case["W"], case["H"])
    assert {c["name"] for c in _GOLD["cases"]} == set(CASE)
    assert {(c["W"] % 4 != 0) for c in _GOLD["cases"]} == {False, True}
    assert {c["calc_angles"] for c in _GOLD["cases"]} == {False, True}
    assert {c["n_calls"] for c in _GOLD["cases"]} == {1, 3}


@pytest.mark.parametrize("case", _GOLD["cases"], ids=case_id)
def test_oracle_replays_the_reference(case):
    """Every call: x, y, width, height and the search window equal the reference's, the angle bit for bit (or both
    NaN)."""
    assert first_difference(case, replay(oracle.lib(), case)) is None


# ------------------------------------------------------------------------------------------------------------------
# mutants of the oracle that the replay must reject

ORACLE_SRC = Path(oracle.__file__).resolve().parent / "ht_oracle.c"
_TRACK = "int hto_tracker_track("
MUTANTS = {
    # the shift rounded down instead of truncated toward zero (src/camshift.js:295-296)
    "floor_shift": [(_TRACK, "static int32_t mut_floor(double v) { return v == v ? (int32_t)floor(v) : 0; }\n" + _TRACK),
                    ("t->sx += js_to_int32(x - t->sw / 2.0);", "t->sx += mut_floor(x - t->sw / 2.0);"),
                    ("t->sy += js_to_int32(y - t->sh / 2.0);", "t->sy += mut_floor(y - t->sh / 2.0);")],
    # eleven mean-shift passes instead of ten (:277)
    "eleven_passes": [("const int iters = 10;", "const int iters = 11;")],
    # the window's origin not clipped to the canvas (:286-287); pixels left of or above the canvas weigh 0
    "no_origin_clip": [("int wadx = imax(t->sx, 0);", "int wadx = t->sx;"),
                       ("int wady = imax(t->sy, 0);", "int wady = t->sy;"),
                       ("double val = a[j];", "double val = (i >= 0 && j >= 0) ? a[j] : 0.0;")],
    # no clamp of the search window to [0, W] x [0, H] after mean-shift (:308-309)
    "no_window_clamp": [("t->sx = imax(0, imin(t->sx, W));", ""), ("t->sy = imax(0, imin(t->sy, H));", "")],
}


def build_mutant(name, tmp_path):
    import ctypes as C
    import shutil
    import subprocess
    src = ORACLE_SRC.read_text()
    for old, new in MUTANTS[name]:
        assert src.count(old) == 1, (name, old)
        src = src.replace(old, new)
    d = tmp_path / name
    d.mkdir()
    (d / "ht_oracle.c").write_text(src)
    shutil.copy(ORACLE_SRC.with_name("ht_oracle.h"), d / "ht_oracle.h")
    so = d / "libmutant.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=c11", "-D_GNU_SOURCE",
                           "-shared", "-o", str(so), str(d / "ht_oracle.c"), "-lm"])
    L = C.CDLL(str(so))
    ref = oracle.lib()
    for fn in ("hto_tracker_init", "hto_tracker_track"):
        getattr(L, fn).argtypes = getattr(ref, fn).argtypes
    return L


@pytest.mark.parametrize("name", list(MUTANTS))
def test_replay_rejects_oracle_mutants(name, tmp_path):
    """Each mutation of the oracle's camshift changes at least one call of the golden."""
    L = build_mutant(name, tmp_path)
    killed = [case_id(c) for c in _GOLD["cases"] if first_difference(c, replay(L, c)) is not None]
    assert killed, name


# ------------------------------------------------------------------------------------------------------------------
# the corpus takes every path, at every size the GPU test runs

def bins_of(rgba):
    r, g, b = (rgba[..., i].astype(np.int64) >> 4 for i in range(3))
    return 256 * r + 16 * g + b


def coverage(W, H):
    """Per path of meanShift / camShift, how many passes (or calls) of the corpus take it, from the oracle's trace.
    The shifts of passes that moved left or up (or not at all) are re-derived from the window's moments (numpy, fp64)
    to count those whose truncation toward zero differs from rounding down."""
    c = dict.fromkeys(("clipped_negative", "clipped_right_bottom", "empty", "m00_zero", "trunc_not_floor",
                       "not_converged", "size_zero", "width_below_4", "width_above_128", "height_below_16",
                       "origin_unaligned"), 0)
    for name, path, kind in CASES:
        for calc in (False, True):
            for n_calls in (1, 3):
                frames = [frame(path, t, W, H) for t in range(T)]
                ot = oracle.CamshiftTracker(calc_angles=calc)
                ot.init_tracker(frames[0], *init_rect(kind, path, W, H))
                model = np.frombuffer(bytes(ot.t.model_hist), np.uint32)
                for f in frames:
                    pdf = None
                    for _ in range(n_calls):
                        sx, sy, sw, sh = ot.search_window()
                        tr = ot.track(f)
                        o = ot.track_obj()
                        for i in range(tr.n_iter):
                            x0, y0 = max(sx, 0), max(sy, 0)
                            x1, y1 = min(x0 + sw, W), min(y0 + sh, H)
                            c["clipped_negative"] += sx < 0 or sy < 0
                            c["clipped_right_bottom"] += sx + sw > W or sy + sh > H
                            c["empty"] += x1 <= x0 or y1 <= y0
                            c["width_below_4"] += 0 < x1 - x0 < 4 and y1 > y0
                            c["width_above_128"] += x1 - x0 > 128 and y1 > y0
                            c["height_below_16"] += 0 < y1 - y0 < 16 and x1 > x0
                            c["origin_unaligned"] += x0 % 4 != 0 and x1 > x0 and y1 > y0
                            dx, dy = tr.wx[i] - sx, tr.wy[i] - sy
                            if (dx <= 0 or dy <= 0) and x1 > x0 and y1 > y0:
                                if pdf is None:
                                    pdf = oracle.weights(model, oracle.histogram(f))[bins_of(f)]
                                win = pdf[y0:y1, x0:x1]
                                m00 = win.sum()
                                if m00 > 0:
                                    vx = (win.sum(axis=0) @ np.arange(x1 - x0)) / m00 - sw / 2
                                    vy = (win.sum(axis=1) @ np.arange(y1 - y0)) / m00 - sh / 2
                                    c["trunc_not_floor"] += any(v < 0 and abs(v - round(v)) > 1e-6 and math.floor(v) != d
                                                                for v, d in ((vx, dx), (vy, dy)))
                            sx, sy = tr.wx[i], tr.wy[i]
                        c["m00_zero"] += tr.m00 == 0
                        c["not_converged"] += tr.n_iter == 10 and tr.converged == 0
                        c["size_zero"] += o["width"] == 0 or o["height"] == 0
    return c


@pytest.mark.parametrize("W,H", SIZES)
def test_corpus_takes_every_path(W, H):
    c = coverage(W, H)
    assert all(v > 0 for v in c.values()), c
