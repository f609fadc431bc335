"""CPU: a stream's best shot (DESIGN.md 2, "Best shots") three ways - the library's host build (ht_best_shot_score,
ht_selftest_best_shot_step / _end), headtrackr_b200.bestshot and the independent C restatement tests/best_shot_oracle.c:

  * the score agrees exactly on the candidates of every golden CS box, cut by the host build of k_face_crop's per-crop
    code (ht_selftest_face_crop_rgba) across canvas and video sizes, orientations, source rectangles and scales
    0.01-16, and on random images with alpha holes and edges at 3x3, 3x2048, 2048x3 and odd sizes; the 2048x2048
    checkerboard reaches the bound 2046^2 1020^2 < 2^43;
  * the state agrees byte for byte over begin, improve, ties, the ends (a lost face, an IDLE or VJ tick, import), one
    and two images, setting anew, the golden CS sequences and random sequences;
  * the ABI's sizes and offsets, the two new span kinds of the overlap rule in both directions against a brute force,
    and spill-free new kernels that leave k_face_crop's own copy of face_crop_tile alone."""
import ctypes as C
import itertools
import math
import random
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import _lib, bestshot
from headtrackr_b200.framing import crop_tick
from test_cascade_host import CSRC, st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_face_crop_host import golden_cs_boxes, lib_crop_rgba, smooth_frame
from test_framing_host import golden_sequences
from test_output_overlap_host import random_stream
from test_output_overlap_host import spans as spans_before

FRAMING, BEST_IMAGE, BEST_STATE = 4, 5, 6        # the overlap rule's kinds after the four of test_output_overlap_host


@pytest.fixture(scope="module")
def bo(tmp_path_factory):
    """tests/best_shot_oracle.c built into a temporary directory, without contraction"""
    so = tmp_path_factory.mktemp("best_shot_oracle") / "libbest_shot_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(so),
                           str(Path(__file__).with_name("best_shot_oracle.c")), "-lm"])
    L = C.CDLL(str(so))
    L.hbo_score.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.hbo_score.restype = C.c_uint64
    L.hbo_step.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_double, C.c_int, C.c_int]
    L.hbo_end.argtypes = [C.c_void_p]
    L.hbo_end.restype = None
    return L


@pytest.fixture(scope="module")
def lib(st):  # noqa: F811
    st.ht_best_shot_score.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    st.ht_selftest_best_shot_step.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_double, C.c_int, C.c_int]
    st.ht_selftest_best_shot_end.argtypes = [C.c_void_p]
    st.ht_selftest_best_shot_end.restype = None
    st.ht_selftest_face_crop_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    st.ht_selftest_tick_writes_best.argtypes = [C.c_int] + [C.c_void_p] * 8
    return st


def event(det, x, y, w, h, angle):
    e = _lib.TrackerEvent()
    e.detection, e.confidence, e.x, e.y, e.width, e.height, e.angle = det, 1.0, x, y, w, h, angle
    return e


def scores(lib, bo, img, pitch=None):
    """the score of an (h, w, 4) uint8 image (optionally inside rows of `pitch` bytes) three ways, asserted equal"""
    h, w = img.shape[:2]
    pitch = pitch or 4 * w
    buf = np.zeros((h, pitch), np.uint8)
    buf[:, :4 * w] = img.reshape(h, 4 * w)
    out = C.c_uint64()
    assert lib.ht_best_shot_score(buf.ctypes.data, w, h, pitch, C.byref(out)) == 0
    o = bo.hbo_score(buf.ctypes.data, w, h, pitch)
    p = bestshot.score(img)
    assert out.value == o == p, (img.shape, out.value, o, p)
    return p


# ---- the score -------------------------------------------------------------------------------------------------------

def test_golden_candidates_score_alike(lib, bo):
    boxes = golden_cs_boxes()
    assert len(boxes) > 20
    rng = random.Random(7)
    scored = holes = 0
    cases = [((160, 120), (320, 240), 0, (0, 0, 0, 0)), ((320, 240), (320, 240), 0, (0, 0, 0, 0)),
             ((320, 240), (640, 480), 3, (0, 0, 0, 0)), ((640, 480), (1280, 720), 5, (40, 100, 640, 960)),
             ((320, 240), (321, 243), 6, (0, 0, 0, 0))]
    for n, (x, y, w, h, a) in enumerate(boxes):
        (cw, ch), (vw, vh), o, rect = cases[n % len(cases)]
        k = cw / 320.0
        frame = smooth_frame(vw, vh, seed=n)
        for scale in (0.01, 1.0, 1.25, rng.choice([0.5, 2.0, 4.0]), 16.0):
            Sw, Sh = rng.choice([(24, 20), (3, 3), (33, 17), (64, 64), (65, 18)])
            rc, buf, pitch = lib_crop_rgba(lib, event(2, x * k, y * k, w * k, h * k, a), cw, ch, frame, o, rect,
                                           Sw, Sh, scale)
            assert rc == int(crop_tick(dict(detection=2, x=x, y=y, width=w, height=h)))
            if rc == 0:                              # a golden box of width or height 0 makes no candidate
                continue
            img = buf.reshape(Sh, pitch)[:, :4 * Sw].reshape(Sh, Sw, 4)
            scores(lib, bo, img, pitch)
            scored += 1
            holes += bool((img[..., 3] < 255).any())
    assert scored > 100 and holes > 10           # faces near and past the video's edges leave alpha holes


@pytest.mark.parametrize("w,h", [(3, 3), (3, 2048), (2048, 3), (5, 7), (17, 33), (64, 16), (65, 17), (127, 3)])
def test_random_images_with_holes_score_alike(lib, bo, w, h):
    rng = np.random.default_rng(w * 4096 + h)
    for trial in range(6):
        img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        img[..., 3] = np.where(rng.random((h, w)) < [0.0, 0.02, 0.3, 0.9, 1.0, 0.1][trial], 255,
                               rng.choice([0, 254], (h, w))).astype(np.uint8) if trial else 255
        if trial == 5:
            img[..., :3] = np.where(rng.random((h, w, 1)) < 0.5, 0, 255)     # hard edges
        s = scores(lib, bo, img, pitch=4 * w + 4 * (trial % 3))
        if trial == 0:
            assert s > 0
        if (img[..., 3] < 255).all():
            assert s == 0


def test_edges_and_alpha_rule(lib, bo):
    img = np.zeros((5, 5, 4), np.uint8)
    img[..., 3] = 255
    img[2, 2, :3] = 100                          # one bright pixel: L = 4 g at the centre, -g at its four neighbours
    g = 100
    assert scores(lib, bo, img) == (4 * g) ** 2 + 4 * g * g
    img[2, 3, 3] = 254                           # a hole on a neighbour drops the centre's term and its own
    assert scores(lib, bo, img) == 3 * g * g
    img[..., :3] = 200                           # a flat image scores 0
    img[..., 3] = 255
    assert scores(lib, bo, img) == 0
    img[0, :, :3] = 0                            # the border row is read only as a neighbour
    assert scores(lib, bo, img) == 3 * 200 ** 2


def test_checkerboard_reaches_the_bound(lib, bo):
    n = 2048
    img = np.zeros((n, n, 4), np.uint8)
    img[..., 3] = 255
    img[(np.add.outer(np.arange(n), np.arange(n)) & 1) == 1, :3] = 255
    s = scores(lib, bo, img)
    assert s == (n - 2) ** 2 * 1020 ** 2 and s < 2 ** 43


def test_score_rejections(lib):
    img = np.zeros((4, 4, 4), np.uint8)
    out = C.c_uint64()
    assert lib.ht_best_shot_score(None, 4, 4, 16, C.byref(out)) == _lib.HT_ERR_ARG
    assert lib.ht_best_shot_score(img.ctypes.data, 4, 4, 16, None) == _lib.HT_ERR_ARG
    assert lib.ht_best_shot_score(img.ctypes.data, 4, 4, 12, C.byref(out)) == _lib.HT_ERR_ARG
    for w, h in ((2, 4), (4, 2), (2049, 4), (4, 2049)):
        assert lib.ht_best_shot_score(img.ctypes.data, w, h, 0, C.byref(out)) == _lib.HT_ERR_SIZE
    assert lib.ht_best_shot_score(img.ctypes.data, 4, 4, 0, C.byref(out)) == 0 and out.value == 0


# ---- the state -------------------------------------------------------------------------------------------------------

class Three:
    """one best shot's state three ways: the library's host build, bestshot.py and the C restatement"""

    def __init__(self, lib, bo, two=True):
        self.lib, self.bo, self.two = lib, bo, two
        self.ls, self.os, self.py = _lib.BestShotState(), (C.c_char * 96)(), bestshot.new_state()

    def step(self, r, score, now_ms=0.0, cw=320, ch=240):
        e = event(r["detection"], r["x"], r["y"], r["width"], r["height"], r["angle"])
        a = self.lib.ht_selftest_best_shot_step(C.addressof(self.ls), int(self.two), score, C.addressof(e), now_ms, cw, ch)
        b = bestshot.step(self.py, r, score, now_ms, cw, ch, self.two)
        c = self.bo.hbo_step(self.os, int(self.two), score,
                             (C.c_double * 6)(*(r[k] for k in ("detection", "x", "y", "width", "height", "angle"))),
                             now_ms, cw, ch)
        assert a == int(b) == c, (r, score, a, b, c)
        self.check()
        return a

    def end(self):
        self.lib.ht_selftest_best_shot_end(C.addressof(self.ls))
        bestshot.end(self.py)
        self.bo.hbo_end(self.os)
        self.check()

    def reset(self):
        self.ls, self.os, self.py = _lib.BestShotState(), (C.c_char * 96)(), bestshot.new_state()

    def check(self):
        lb = bytes(self.ls)
        assert lb == bestshot.state_to_bytes(self.py) == bytes(self.os), (bestshot.state_from_bytes(lb), self.py)
        assert bestshot.state_to_bytes(bestshot.state_from_bytes(lb)) == lb

    @property
    def s(self):
        return dict(self.py)


def cs(x=100.0, y=80.0, w=40.0, h=48.0, angle=math.nan):
    return dict(detection=2, x=x, y=y, width=w, height=h, angle=angle)


IDLE = dict(detection=0, x=0.0, y=0.0, width=0.0, height=0.0, angle=0.0)
VJ = dict(detection=1, x=90.0, y=70.0, width=44.0, height=44.0, angle=0.0)
LOST = cs(w=0.0, h=0.0)


def test_begin_improve_ties_and_ends(lib, bo):
    t = Three(lib, bo)
    assert t.s["track"] == t.s["ended"] == 0
    assert t.step(cs(), 0, now_ms=10.0) == 1                 # a track's first tick is its best, even at score 0
    s = t.s
    assert (s["track"], s["ended"], s["ticks"], s["best_tick"], s["buffer"], s["flags"]) == (1, 0, 1, 0, 0, 3)
    assert s["now_ms"] == 10.0 and (s["canvas_w"], s["canvas_h"]) == (320, 240)
    assert t.step(cs(x=101.0), 50, now_ms=20.0) == 1          # strictly greater: improves
    assert t.s["best_tick"] == 1 and t.s["x"] == 101.0 and t.s["flags"] == bestshot.IMPROVED
    assert t.step(cs(x=102.0), 50, now_ms=30.0) == 0          # a tie: the earliest tick keeps it
    assert t.s["best_tick"] == 1 and t.s["x"] == 101.0 and t.s["score"] == 50 and t.s["flags"] == 0
    assert t.step(cs(x=103.0), 40, now_ms=40.0) == 0
    assert t.s["score"] == 40 and t.s["best_score"] == 50 and t.s["ticks"] == 4
    assert t.step(LOST, 999) == 0                             # the CS tick that loses the face ends the track
    assert (t.s["ended"], t.s["flags"], t.s["ticks"], t.s["best_score"]) == (1, bestshot.ENDED, 4, 50)
    assert t.step(IDLE, 0) == 0 and t.s["flags"] == 0 and t.s["ended"] == 1   # nothing open: nothing ends
    assert t.step(VJ, 0) == 0 and t.s["flags"] == 0
    assert t.step(cs(), 7, now_ms=50.0) == 1                  # track 2 writes the other image
    assert (t.s["track"], t.s["buffer"], t.s["best_tick"], t.s["best_score"], t.s["flags"]) == (2, 1, 0, 7, 3)
    assert t.step(IDLE, 0) == 0 and t.s["flags"] == bestshot.ENDED and t.s["ended"] == 2   # a tick after stop
    assert t.step(cs(), 7) == 1 and t.s["buffer"] == 0 and t.s["track"] == 3
    assert t.step(VJ, 0) == 0 and t.s["ended"] == 3           # any tick that is not a crop tick ends it


def test_import_ends_an_open_track(lib, bo):
    t = Three(lib, bo)
    t.end()
    assert t.s == bestshot.new_state()                        # nothing open: nothing changes
    t.step(cs(), 5)
    t.step(cs(), 9)
    t.end()
    assert (t.s["ended"], t.s["track"], t.s["flags"], t.s["best_score"]) == (1, 1, bestshot.ENDED, 9)
    t.end()
    assert t.s["ended"] == 1 and t.s["flags"] == bestshot.ENDED
    assert t.step(cs(), 1) == 1 and t.s["track"] == 2 and t.s["buffer"] == 1 and t.s["flags"] == 3


def test_one_image_and_setting_anew(lib, bo):
    t = Three(lib, bo, two=False)
    for track in range(1, 6):
        assert t.step(cs(), track) == 1 and t.s["buffer"] == 0 and t.s["track"] == track
        t.step(IDLE, 0)
    t.reset()                                                 # setting the best shot again zeroes the state
    assert t.step(cs(), 3) == 1 and t.s["track"] == 1 and t.s["buffer"] == 0


def test_golden_sequences_agree(lib, bo):
    rng = random.Random(11)
    seqs = golden_sequences()
    assert len(seqs) >= 3
    writes = 0
    for two in (True, False):
        for name, seq in seqs:
            t = Three(lib, bo, two)
            for n, r in enumerate(seq):
                writes += t.step(r, rng.choice([0, 1, rng.randrange(1 << 43)]), now_ms=1000.0 + 33.0 * n)
                if rng.random() < 0.1:
                    t.step(IDLE, 0)
    assert writes > 50


def test_random_sequences_agree(lib, bo):
    rng = random.Random(5)
    tracks = 0
    for run in range(200):
        t = Three(lib, bo, two=run % 3 != 0)
        for n in range(rng.randint(1, 60)):
            u = rng.random()
            if u < 0.55:
                r = cs(rng.uniform(-10, 330), rng.uniform(-10, 250), rng.choice([0.0, -1.0, 1.0, rng.uniform(1, 200)]),
                       rng.choice([rng.uniform(1, 200), 0.0, math.nan]), rng.choice([math.nan, rng.uniform(-4, 4)]))
                if rng.random() < 0.05:
                    r["x"] = rng.choice([65536.0, 65537.0, math.inf])
            else:
                r = rng.choice([IDLE, VJ, LOST, dict(IDLE, detection=3)])
            t.step(r, rng.choice([0, 1, 2, 2, rng.randrange(1 << 43)]), now_ms=rng.uniform(0, 1e12),
                   cw=rng.choice([320, 160]), ch=rng.choice([240, 120]))
            if rng.random() < 0.03:
                t.end()
        tracks += t.s["track"]
    assert tracks > 300


# ---- ABI ---------------------------------------------------------------------------------------------------------------

def test_abi_sizes_offsets_and_symbols(bo):
    header = (CSRC.parent.parent / "include" / "headtrackr_b200.h").read_text()
    assert "#define HT_BEST_SHOT_STATE_BYTES 96" in header and "} ht_best_shot;           /* 48 bytes */" in header
    assert "int ht_tracker_set_best_shot(ht_ctx *ctx, int first, int n, const ht_best_shot *shots);" in header
    assert "int ht_best_shot_score(const uint8_t *rgba, int w, int h, int pitch, uint64_t *out);" in header
    for name, v in (("BEGAN", 1), ("IMPROVED", 2), ("ENDED", 4)):
        assert f"#define HT_BEST_{name} {v}" in header
    S = _lib.BestShotState
    assert C.sizeof(S) == bo.hbo_state_bytes() == _lib.BEST_SHOT_STATE_BYTES == 96
    assert [getattr(S, f).offset for f in ("best_score", "score", "x", "y", "width", "height", "angle", "now_ms",
                                           "canvas_w", "canvas_h", "track", "ended", "ticks", "best_tick", "buffer",
                                           "flags")] == [0, 8, 16, 24, 32, 40, 48, 56, 64, 68, 72, 76, 80, 84, 88, 92]
    B = _lib.BestShot
    assert C.sizeof(B) == 48 and [getattr(B, f).offset for f in ("rgba", "state", "width", "height", "pitch", "pad_",
                                                                  "scale")] == [0, 16, 24, 28, 32, 36, 40]
    L = _lib.lib()
    for s in ("ht_tracker_set_best_shot", "ht_best_shot_score"):
        assert hasattr(L, s) and s in _lib.EXPORTS
    assert L.ht_tracker_set_best_shot(None, 0, 1, (_lib.BestShot * 1)()) == _lib.HT_ERR_ARG
    img, out = np.zeros((3, 3, 4), np.uint8), C.c_uint64(1)
    assert L.ht_best_shot_score(img.ctypes.data, 3, 3, 0, C.byref(out)) == 0 and out.value == 0


# ---- the overlap rule ------------------------------------------------------------------------------------------------

def spans(stream):
    out = spans_before(stream)
    if stream.get("box"):
        out.append((FRAMING, stream["box"], stream["box"] + _lib.FRAMED_BOX_BYTES))
    b = stream.get("best")
    if b:
        pitch = b.pitch or 4 * b.width
        for p in b.rgba:
            if p:
                out.append((BEST_IMAGE, p, p + (b.height - 1) * pitch + 4 * b.width))
        out.append((BEST_STATE, b.state, b.state + _lib.BEST_SHOT_STATE_BYTES))
    return out


def brute(streams):
    flat = [(k, s, set(range(a, b))) for s, x in enumerate(streams) for k, a, b in spans(x)]
    return [((k0, s0), (k1, s1)) for (k0, s0, b0), (k1, s1, b1) in itertools.combinations(flat, 2) if b0 & b1]


def verdict(lib, streams):
    n = len(streams)
    dbg, crops, yuv = (_lib.DebugCanvas * n)(), (_lib.FaceCrop * n)(), (_lib.FaceCropYuv * n)()
    tensors, cams, boxes, shots = (_lib.FaceTensor * n)(), (C.c_void_p * n)(), (C.c_void_p * n)(), (_lib.BestShot * n)()
    clash = (C.c_int32 * 4)()
    for s, x in enumerate(streams):
        for arr, key in ((dbg, "debug"), (crops, "crop"), (yuv, "yuv"), (tensors, "tensor"), (shots, "best")):
            if x.get(key):
                arr[s] = x[key]
        cams[s], boxes[s] = x.get("camera"), x.get("box")
    hit = lib.ht_selftest_tick_writes_best(n, dbg, crops, yuv, tensors, cams, boxes, shots, clash)
    return hit, ((clash[0], clash[1]), (clash[2], clash[3]))


def random_best(rng, space):
    at = lambda align=1: rng.randrange(64, space, align)   # noqa: E731
    w, h = rng.randint(3, 6), rng.randint(3, 5)
    pitch = rng.choice([0, 4 * w + 4 * rng.randint(0, 3)])
    return _lib.BestShot((C.c_void_p * 2)(at(4), at(4) if rng.random() < 0.6 else None), at(8), w, h, pitch, 0, 1.0)


def test_random_layouts_with_best_shots_equal_the_brute_force(lib):
    rng = random.Random(2027)
    kinds, verdicts = set(), [0, 0]
    for trial in range(2500):
        space = rng.choice([2048, 8192, 32768])
        streams = []
        for _ in range(rng.randint(1, 4)):
            x = random_stream(rng, space)
            if rng.random() < 0.3:
                x["box"] = rng.randrange(64, space, 8)
            if rng.random() < 0.6:
                x["best"] = random_best(rng, space)
            streams.append(x)
        hit, pair = verdict(lib, streams)
        pairs = brute(streams)
        assert hit == (len(pairs) > 0), (hit, pairs)
        if hit:
            assert pair in pairs or pair[::-1] in pairs, (pair, pairs)
        verdicts[hit] += 1
        kinds |= {tuple(sorted((a[0], b[0]))) for a, b in pairs}
    for k in range(7):                                       # each new kind clashed with every kind, itself included
        assert tuple(sorted((k, BEST_IMAGE))) in kinds and tuple(sorted((k, BEST_STATE))) in kinds, (k, kinds)
    assert min(verdicts) > 200, verdicts


def test_hand_cases(lib):
    base = 1 << 20
    shot = lambda a, b, st, w=4, h=3, pitch=0: _lib.BestShot((C.c_void_p * 2)(a, b), st, w, h, pitch, 0, 1.0)  # noqa: E731
    one = dict(best=shot(base, base + 48, base + 4096))
    assert verdict(lib, [one])[0] == 0                                           # two images back to back
    assert verdict(lib, [dict(best=shot(base, base + 44, base + 4096))])[0] == 1   # sharing the last byte
    assert verdict(lib, [dict(best=shot(base, base + 44, base + 4096))])[1] == ((BEST_IMAGE, 0), (BEST_IMAGE, 0))
    # a state inside an image's row padding is a clash: the span runs over the rows
    assert verdict(lib, [dict(best=shot(base, None, base + 20, pitch=32))])[0] == 1
    # a crop on the other stream's state, and a state on another stream's crop, in both orders
    crop = _lib.FaceCrop(base + 4096 + 8, 2, 2, 0, 0, 1.0)
    hit, pair = verdict(lib, [one, dict(crop=crop)])
    assert hit and sorted(pair) == [(1, 1), (BEST_STATE, 0)]
    hit, pair = verdict(lib, [dict(crop=crop), one])
    assert hit and sorted(pair) == [(1, 0), (BEST_STATE, 1)]
    cam = dict(camera=base + 32)
    hit, pair = verdict(lib, [cam, one])
    assert hit and sorted(pair) == [(3, 0), (BEST_IMAGE, 1)]


# ---- registers, spills and k_face_crop's own copy --------------------------------------------------------------------

def test_new_kernels_do_not_spill(tmp_path):
    out = subprocess.run([_lib.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                          "-Xptxas", "-v", "-Xcompiler", "-fPIC", "-c", "-o", str(tmp_path / "ht_api.o"),
                          str(CSRC / "ht_api.cu")], capture_output=True, text=True, check=True).stderr
    spills, regs, cur = {}, {}, None
    for line in out.splitlines():
        m = re.search(r"(?:Compiling entry function '|Function properties for )(\w+)", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            spills[cur] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            regs[cur] = int(m.group(1))
    for name in ("k_best_score", "k_best_write", "best_tile_gray", "face_crop_tile"):
        hits = {k: v for k, v in spills.items() if name in k}
        assert hits and all(v == (0, 0) for v in hits.values()), (name, hits)
    # k_best_write calls its own instantiation of face_crop_tile, so k_face_crop's stays as it was
    assert any("face_crop_tileILi0ELi1E" in k for k in spills) and any("face_crop_tileILi0ELi0E" in k for k in spills)
    best = {k: v for k, v in regs.items() if "k_best_score" in k or "k_best_write" in k}
    assert len(best) == 2 and all(v <= 128 for v in best.values()), best
