"""GPU parity of detection across canvas geometries (tests/test_detect_geometry_host.py's GEOMETRIES), against the oracle.

The host emulation pins the planner's layout and the kernels' per-thread arithmetic at these sizes; what it replaces by
loops is checked here: k_gray's chunking and its 16-bit histogram counters, k_resample's tiles, k_cascade's TMA /
cp.async staging, survivor masks and barriers, waves, k_group, and the plan and tensor-map caches of one context.
Each test makes its own Context (the session one stops at 1280x720) and closes it.
"""
import ctypes as C
import math

import numpy as np
import pytest

import oracle
from headtrackr_b200 import synth
from test_detect_geometry_host import (GEOMETRIES, HIST_FACES, HIST_H, HIST_W, REJECTED, arena_words, flat_face,
                                       geometry_frame, largest_cta_bin)

pytestmark = pytest.mark.gpu

BATCH = 5                    # two quads, the second one partial
LARGE_PX = 1_500_000         # above this a batch repeats 3 distinct frames (the oracle takes seconds per frame)
_FRAMES, _WANT = {}, {}


def distinct(W, H):
    """how many distinct frames a W x H batch holds; frame i of the batch is distinct frame i % distinct(W, H)"""
    return 3 if W * H > LARGE_PX else BATCH


def frames_of(W, H):
    """BATCH frames of W x H: faces, and one noise frame (the last distinct one)"""
    if (W, H) not in _FRAMES:
        uniq = distinct(W, H)
        fr = [geometry_frame(i, W, H, kind="noise" if i == min(3, uniq - 1) else "faces") for i in range(uniq)]
        _FRAMES[(W, H)] = np.stack([fr[i % uniq] for i in range(BATCH)])
    return _FRAMES[(W, H)]


def want(W, H, interval, i):
    """(grouped list at min_neighbors 1, raw list) of frame i, from the oracle, once per distinct frame"""
    key = (W, H, interval, i % distinct(W, H))
    if key not in _WANT:
        _WANT[key] = oracle.detect(frames_of(W, H)[i], _blob(), interval, want_raw=True)
    return _WANT[key]


def _blob():
    return synth.load_cascade_blob()


def tup(d):
    return (d["x"], d["y"], d["width"], d["height"], d["confidence"], d.get("neighbors", d.get("neighbor")))


def context(W, H, n=BATCH):
    from headtrackr_b200 import Context
    # result lists as long as the raw lists: the min_neighbors 0 output is the whole raw list
    return Context(max_width=W, max_height=H, max_frames=n, max_raw_per_frame=16384, max_rects_per_frame=16384)


def plane(c, frame, slot, q, W, H):
    """ht_debug_plane with a buffer as large as the frame (Context.debug_plane's stops at 2048x2048)"""
    w, h = C.c_int32(), C.c_int32()
    buf = np.zeros(W * H, np.uint8)
    c._check(c._L.ht_debug_plane(c._h, frame, slot, q, buf.ctypes.data, buf.size, C.addressof(w), C.addressof(h)))
    return buf[: w.value * h.value].reshape(h.value, w.value).copy()


def raw_lists(c, n):
    out = []
    for f in range(n):
        r, cnt = c.debug_raw(f, cap=16384)
        assert cnt == len(r), (f, cnt)
        out.append(r)
    return out


CASES = [(W, H, iv) for W, H, ivs, _ in GEOMETRIES for iv in ivs]


@pytest.mark.parametrize("W,H,interval", CASES)
def test_detect_equals_the_oracle(blob, W, H, interval):
    """Grouped lists and raw lists of a 5-frame batch, from host and from device memory; every pyramid plane of frame
    1 (byte lane 1 of the first quad); the min_neighbors 0 output equals the raw list."""
    import torch
    frames = frames_of(W, H)
    c = context(W, H)
    try:
        n_faces = 0
        for src in (frames, torch.from_numpy(frames).cuda()):
            got = c.detect(src, interval, 1)
            assert c.last_warning is None
            raw = raw_lists(c, BATCH)
            for i in range(BATCH):
                grouped, want_raw = want(W, H, interval, i)
                assert raw[i] == want_raw, (i, "raw")
                assert [tup(d) for d in got[i]] == grouped, (i, "grouped")
                n_faces += len(grouped)
        assert n_faces >= 1                                 # parity must not be vacuous
        gray = oracle.grayscale(frames[1])
        pyr = oracle.Pyramid(gray, interval)
        g = pyr.geom
        info = c.plan_info(W, H, interval)
        assert info["w"] == list(g.w[: g.n_slots]) and info["h"] == list(g.h[: g.n_slots])
        for s in range(g.n_slots):
            for q in range(4 if s >= 2 * g.next else 1):
                assert np.array_equal(plane(c, 1, s, q, W, H), pyr.plane(s, q)), (s, q)
        raw0 = c.detect(frames, interval, 0)
        assert c.last_warning is None
        for i in range(BATCH):
            assert [tup(d) for d in raw0[i]] == want(W, H, interval, i)[1], (i, "min_neighbors 0")
    finally:
        c.close()


def test_rejected_geometries_launch_nothing():
    """Every rejected size returns HT_ERR_SIZE with the planner's reason and launches no kernel."""
    from headtrackr_b200._lib import HT_ERR_SIZE, HtError
    def is_reason(msg, why):                                # msg: the whole message after "error -3: "
        if why == "small":
            return msg.startswith("frame too small: pyramid level ")
        return msg == {"bilinear": "frame too large for 32-bit bilinear numerators", "dim": "frame too large"}[why]

    for W, H, interval, why in REJECTED:
        c = context(W, H, 1)
        try:
            f = np.zeros((H, W, 4), np.uint8)
            before = c.launch_count
            for call in (lambda: c.detect(f, interval, 1),
                         lambda: c.detect_track(f, interval, 1, calc_angles=False, n_calls=1)):
                with pytest.raises(HtError) as e:
                    call()
                assert e.value.code == HT_ERR_SIZE, (W, H, interval)
                assert is_reason(str(e.value).split(f"error {HT_ERR_SIZE}: ", 1)[1], why), (W, H, interval, str(e.value))
            assert c.launch_count == before, (W, H, interval)
        finally:
            c.close()


VARIANTS = {
    "no_tma": ({"HT_TMA": "0"}, 0),
    "wave4_pipe": ({"HT_WAVE": "4", "HT_DETECT_PIPE": "1"}, 0),
    "wave8_pipe": ({"HT_WAVE": "8", "HT_DETECT_PIPE": "1"}, 0),
    "forced_ties": ({}, 3),
}
VARIANT_N = 9                # three waves of 4 / two of 8, the last one partial


@pytest.mark.parametrize("W,H", [(1920, 1080), (2560, 1440), (16000, 200)])
def test_variants_give_the_same_raw_lists(blob, W, H, monkeypatch):
    frames = np.stack([frames_of(W, H)[i % BATCH] for i in range(VARIANT_N)])
    c = context(W, H, VARIANT_N)
    try:
        c.detect(frames, 5, 1)
        base = raw_lists(c, VARIANT_N)
    finally:
        c.close()
    for i in range(BATCH):
        assert base[i] == want(W, H, 5, i)[1], i
    for name, (env, exact) in VARIANTS.items():
        with monkeypatch.context() as m:
            for k, v in env.items():
                m.setenv(k, v)
            c = context(W, H, VARIANT_N)
        try:
            if exact:
                c.debug_set_exactness(exact)
            c.detect(frames, 5, 1)
            assert raw_lists(c, VARIANT_N) == base, name
        finally:
            c.close()


@pytest.mark.parametrize("tma", ["1", "0"])
def test_one_context_alternating_geometries(blob, tma, monkeypatch):
    """A, B, A, C, B in one context equals a fresh context per call.  The context runs waves of one quad (HT_WAVE=4), so
    its arena reservation is one quad's stride: A's first call allocates it, C's is larger and reallocates it (a new
    arena pointer for the tensor-map cache), and the calls after C re-use C's arena."""
    monkeypatch.setenv("HT_TMA", tma)
    A, B, Cg = (1000, 100), (321, 241), (1920, 1080)
    reserve = {g: 4 * -(-arena_words(oracle.geometry(*g, 5)) // 64) * 64 for g in (A, B, Cg)}   # bytes of one wave
    assert reserve[Cg] > reserve[A] > reserve[B]
    fresh = {}
    for W, H in (A, B, Cg):
        c = context(W, H)
        try:
            got = c.detect(frames_of(W, H), 5, 1)
            fresh[(W, H)] = (got, raw_lists(c, BATCH))
        finally:
            c.close()
    monkeypatch.setenv("HT_WAVE", "4")
    c = context(1920, 1080)
    try:
        for W, H in (A, B, A, Cg, B):
            got = c.detect(frames_of(W, H), 5, 1)
            assert (got, raw_lists(c, BATCH)) == fresh[(W, H)], (W, H)
        for i in range(BATCH):
            assert fresh[B][1][i] == want(*B, 5, i)[1] and fresh[Cg][1][i] == want(*Cg, 5, i)[1]
    finally:
        c.close()


def oracle_detect_track(f, blob, interval, calc_angles, n_calls):
    """oracle.detect_track plus the tracker's search window -> (found, (x, y, width, height), angle, window)"""
    L = oracle.lib()
    f = np.ascontiguousarray(f)
    t = oracle.Tracker()
    found = C.c_int()
    L.hto_detect_track(f.ctypes.data_as(C.POINTER(C.c_uint8)), f.shape[1], f.shape[0], blob, len(blob), interval, 1,
                       int(calc_angles), n_calls, C.byref(t), C.byref(found))
    return found.value, (t.tx, t.ty, t.tw, t.th), t.angle, (t.sx, t.sy, t.sw, t.sh)


def assert_track(found, obj, win, want, what):
    assert found == want[0], what
    assert (obj["x"], obj["y"], obj["width"], obj["height"]) == want[1], what
    assert abs(obj["angle"] - want[2]) <= 1e-4 or (math.isnan(obj["angle"]) and math.isnan(want[2])), what
    assert win == want[3], what


@pytest.mark.parametrize("calc_angles", [False, True])
@pytest.mark.parametrize("W,H,interval", [(1920, 1080, 5), (2560, 1440, 5), (81, 81, 5)])
def test_detect_track_equals_the_oracle(blob, W, H, interval, calc_angles):
    frames = frames_of(W, H)
    c = context(W, H)
    try:
        dets, found, objs, wins = c.detect_track(frames, interval, 1, calc_angles=calc_angles, n_calls=3)
        for i in range(BATCH):
            w = oracle_detect_track(frames[i], blob, interval, calc_angles, 3)
            assert [tup(d) for d in dets[i]] == want(W, H, interval, i)[0], i
            assert_track(found[i], objs[i], wins[i], w, i)
        assert any(found)
    finally:
        c.close()


# ---- k_gray's 16-bit histogram counters ----

def test_histogram_counters_at_their_limit(blob):
    """8 x SM-count frames of 301x598, one colour but for a face (tests/test_detect_geometry_host.py, HIST_*).  Each
    launch has 2 x SM-count quads, so the SM count alone would give k_gray 2 chunks per quad, and one CTA would count
    about 90,000 background pixels; the (w*h + 59999) / 60000 rule makes it 3, and one CTA counts 60,003 pixels in the
    background bin, which the tracked model holds.  The host test shows that the oracle's result changes when that
    count loses 65,536, so the tracker equals the oracle only if no counter wraps."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    quads = 2 * sms
    n = 4 * quads
    g = oracle.geometry(HIST_W, HIST_H, 5)
    wave = max(4, min((2048 << 20) // (-(-arena_words(g) // 64) * 64), 1 << 20) & ~3)   # run_detect's default wave
    assert wave >= n                                        # one k_gray launch over all the quads
    chunks_sm = max(1, min(HIST_H, -(-4 * sms // quads)))
    chunks = max(chunks_sm, (HIST_W * HIST_H + 59999) // 60000)
    assert chunks_sm == 2 and chunks == 3
    uniq = [flat_face(*fc) for fc in HIST_FACES]
    assert max(largest_cta_bin(f, chunks) for f in uniq) > 60000
    assert min(largest_cta_bin(f, chunks_sm) for f in uniq) > 65536      # what the SM count alone would give
    # device frames: ht_detect_track detects the whole batch in one part (host frames are cut into parts)
    dev = torch.from_numpy(np.stack(uniq)).cuda()[torch.arange(n, device="cuda") % len(uniq)].contiguous()
    from headtrackr_b200 import Context
    c = Context(max_width=HIST_W, max_height=HIST_H, max_frames=n)
    try:
        for calc_angles in (False, True):
            want_t = [oracle_detect_track(f, blob, 5, calc_angles, 3) for f in uniq]
            assert all(w[0] == 1 for w in want_t)
            dets, found, objs, wins = c.detect_track(dev, 5, 1, calc_angles=calc_angles, n_calls=3)
            for i in range(n):
                assert_track(found[i], objs[i], wins[i], want_t[i % len(uniq)], (calc_angles, i))
    finally:
        c.close()
