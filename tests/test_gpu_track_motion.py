"""GPU parity of k_track and of headtrackr.Tracker on moving faces (the corpus of tests/test_track_motion_host.py): faces
that leave the canvas at every edge and corner, drift left and up, jump, approach and recede, and re-enter; tracked
rectangles that start partly or wholly outside the canvas.

* Every case, with calcAngles on and off, runs as one stream of a context per configuration - the default, every
  cluster size, 128 and 512 threads, the window memo off, zero-weight marking forced, the serial moments forced -
  at 160x120 up to 1280x720 and at 333x251 (W % 4 != 0: the scalar path), with one and with three track() calls per
  frame.  Every launch's result equals the oracle's: x, y, width, height and the search window exactly, the angle
  within 1e-4 or both NaN.
* The passes k_track runs per stream and launch (HT_TRACK_TRACE, memo off) equal the oracle's mean-shift passes, so
  a kernel that ran too many or too few passes but ended on the same window is caught.
* One launch of 270 streams - every case at nine phase offsets, in permuted slots - runs the longest-chain-first
  tiers with edge and empty-window streams beside heavy ones.
* headtrackr.Tracker (TrackerSet, step and feed) on faces that walk off the canvas and come back equals the Python
  mirror main.Tracker over the oracle, event for event: the face is lost by leaving, "redetecting", then "found"
  again, and the device's head events go through every edge-correction branch of headposition.
"""
import math

import numpy as np
import pytest

from test_host_main import check_events
from test_track_motion_host import (CASE, CASES, LIFE_PATHS, LIFE_T, PATHS, SIZES, T, face_box, frame, init_rect,
                                    oracle_run)

pytestmark = pytest.mark.gpu

STREAMS = [(name, calc) for name, _, _ in CASES for calc in (False, True)]

CONFIGS = {
    "default": {},
    "cluster1": {"HT_TRACK_CLUSTER": "1"},
    "cluster2": {"HT_TRACK_CLUSTER": "2"},
    "cluster4": {"HT_TRACK_CLUSTER": "4"},
    "cluster8": {"HT_TRACK_CLUSTER": "8"},
    "cluster16": {"HT_TRACK_CLUSTER": "16"},
    "nt128": {"HT_TRACK_NT": "128"},
    "nt512": {"HT_TRACK_NT": "512"},
    "nomemo": {"HT_TRACK_MEMO": "0"},
    "mask": {"HT_TRACK_MASK": "1,0"},
    "serial": {},                   # ht_debug_set_exactness(4): every pass sums in the reference's order
}

_WANT, _DEV = {}, {}


def want(W, H, n_calls, phase=0):
    """Per stream, per frame: (obj, window, passes) after the frame's n_calls calls, from the oracle."""
    key = (W, H, n_calls, phase)
    if key not in _WANT:
        out = []
        for name, calc in STREAMS:
            path = CASE[name][1]
            frames = [frame(path, (phase + t) % T, W, H) for t in range(T)]
            run = oracle_run(name, W, H, calc, n_calls, frames)
            out.append([(calls[-1][1], calls[-1][3], sum(c[0].n_iter for c in calls)) for calls in run])
        _WANT[key] = out
    return _WANT[key]


def device_clips(W, H):
    """{path: (T, H, W, 4) uint8 CUDA tensor}"""
    import torch
    if (W, H) not in _DEV:
        _DEV.clear()
        _DEV[(W, H)] = {p: torch.from_numpy(np.stack([frame(p, t, W, H) for t in range(T)])).cuda() for p in PATHS}
    return _DEV[(W, H)]


def batch(clips, streams, t):
    """frame t of every stream's clip -> (n, H, W, 4) CUDA tensor; streams: [(name, phase)]"""
    import torch
    b = torch.stack([clips[CASE[name][1]][(phase + t) % T] for name, phase in streams]).contiguous()
    torch.cuda.synchronize()                          # the library runs on its own stream
    return b


def init_streams(c, clips, W, H, streams, calcs, slots):
    """track_init of every stream on its clip's first frame, one call per calcAngles value"""
    for calc in (False, True):
        ks = [k for k in range(len(streams)) if calcs[k] == calc]
        if not ks:
            continue
        f0 = batch(clips, [streams[k] for k in ks], 0)
        rects = [init_rect(CASE[streams[k][0]][2], CASE[streams[k][0]][1], W, H) for k in ks]
        c.track_init(f0, rects, slots=[slots[k] for k in ks], calc_angles=calc)


def assert_call(obj, win, w, what):
    o, ww, _ = w
    assert (obj["x"], obj["y"], obj["width"], obj["height"]) == (o["x"], o["y"], o["width"], o["height"]), (what, obj, o)
    assert abs(obj["angle"] - o["angle"]) <= 1e-4 or (math.isnan(obj["angle"]) and math.isnan(o["angle"])), what
    assert win == ww, (what, win, ww)


@pytest.mark.parametrize("n_calls", [1, 3])
@pytest.mark.parametrize("W,H", SIZES)
@pytest.mark.parametrize("config", list(CONFIGS))
def test_motion_corpus_matches_oracle(config, W, H, n_calls, monkeypatch):
    from headtrackr_b200 import Context
    for k, v in CONFIGS[config].items():
        monkeypatch.setenv(k, v)
    clips = device_clips(W, H)
    wants = want(W, H, n_calls)
    n = len(STREAMS)
    streams = [(name, 0) for name, _ in STREAMS]
    c = Context(max_width=W, max_height=H, max_frames=n)
    try:
        if config == "serial":
            c.debug_set_exactness(4)
        init_streams(c, clips, W, H, streams, [calc for _, calc in STREAMS], list(range(n)))
        c.debug_track_stats(reset=True)
        for t in range(T):
            objs, wins = c.track(batch(clips, streams, t), n_calls=n_calls)
            for k in range(n):
                assert_call(objs[k], wins[k], wants[k][t], (STREAMS[k], config, t))
        st = c.debug_track_stats(reset=True)
        assert st["calls"] == n * n_calls * T
        if config == "serial":
            assert st["serial_passes"] >= st["passes"] > 0
    finally:
        c.close()


@pytest.mark.parametrize("n_calls", [1, 3])
@pytest.mark.parametrize("W,H", [(160, 120), (333, 251), (1280, 720)])
def test_passes_per_launch_equal_the_oracles(W, H, n_calls, monkeypatch):
    """One k_track pass sums one window, as one iteration of meanShift's loop does (the reference's second Moments()
    of a converged window is part of that iteration): with the memo off, each stream's passes per launch equal the
    oracle's n_iter summed over the launch's calls, and the context's totals are their sums."""
    from headtrackr_b200 import Context
    monkeypatch.setenv("HT_TRACK_TRACE", "1")
    monkeypatch.setenv("HT_TRACK_MEMO", "0")
    clips = device_clips(W, H)
    wants = want(W, H, n_calls)
    n = len(STREAMS)
    streams = [(name, 0) for name, _ in STREAMS]
    c = Context(max_width=W, max_height=H, max_frames=n)
    try:
        init_streams(c, clips, W, H, streams, [calc for _, calc in STREAMS], list(range(n)))
        c.debug_track_stats(reset=True)
        total = 0
        for t in range(T):
            objs, wins = c.track(batch(clips, streams, t), n_calls=n_calls)
            passes = c.debug_track_trace(n)[:, 3]
            for k in range(n):
                assert_call(objs[k], wins[k], wants[k][t], (STREAMS[k], t))
                assert int(passes[k]) == wants[k][t][2], (STREAMS[k], t, int(passes[k]), wants[k][t][2])
            total += sum(wants[k][t][2] for k in range(n))
        st = c.debug_track_stats(reset=True)
        assert st["passes"] == total and st["memo_hits"] == 0 and st["calls"] == n * n_calls * T
    finally:
        c.close()


def test_tiered_launch_of_every_clip_at_nine_phases():
    """270 streams in permuted slots of a 300-slot context: every case with calcAngles on and off, each starting at
    one of nine phases of its clip (the clip wraps around, one more jump).  The launch orders them longest chain
    first and runs the heavy ones in tiers; every stream equals the oracle on every frame."""
    from headtrackr_b200 import Context
    W, H, P = 320, 240, 9
    clips = device_clips(W, H)
    streams, calcs, wants = [], [], []
    for phase in range(P):
        w = want(W, H, 1, phase=phase * 4)
        for (name, calc), ws in zip(STREAMS, w):
            streams.append((name, phase * 4))
            calcs.append(calc)
            wants.append(ws)
    n = len(streams)
    assert n >= 256
    slots = [int(s) for s in np.random.default_rng(3).permutation(300)[:n]]
    c = Context(max_width=W, max_height=H, max_frames=300)
    try:
        init_streams(c, clips, W, H, streams, calcs, slots)
        for t in range(T):
            objs, wins = c.track(batch(clips, streams, t), slots=slots)
            for k in range(n):
                assert_call(objs[k], wins[k], wants[k][t], (streams[k], calcs[k], t))
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------------------------
# headtrackr.Tracker

LW, LH = 320, 240
MS = 35.0
MARGIN = 11                          # src/headposition.js:102


def edge_branch(face, W, H):
    """The branch of headposition.track's edge correction (src/headposition.js:100-157) for a face (x, y, w, h)"""
    x, y, w, h = face
    left, right = x - w / 2 < MARGIN, W - (x + w / 2) < MARGIN
    top, bottom = y - h / 2 < MARGIN, H - (y + h / 2) < MARGIN
    if (top or bottom) and (left or right):
        return "corner"
    if top:
        return "top"
    if bottom:
        return "bottom"
    if left:
        return "left"
    if right:
        return "right"
    return "none"


def host_lifecycle(blob, path):
    """main.Tracker over the oracle on a walk clip: per frame, the events (time stripped) and the status"""
    from headtrackr_b200 import Canvas, main
    from test_host_logic import OracleBackend
    video, canvas = Canvas(frame(path, 0, LW, LH)), Canvas(np.zeros((LH, LW, 4), np.uint8))
    clock = [1.0e12]
    ht = main.Tracker(dict(ui=False), backend=OracleBackend(blob), clock=lambda: clock[0])
    log = []
    for typ in ("headtrackrStatus", "facetrackingEvent", "headtrackingEvent"):
        ht.addEventListener(typ, log.append)
    ht.init(video, canvas, False)
    out = []
    for t in range(LIFE_T):
        video.pixels = frame(path, t, LW, LH)
        clock[0] += MS
        n0 = len(log)
        if t == 0:
            assert ht.start() is True
        else:
            ht.step()
        out.append(([{k: v for k, v in e.items() if k != "time"} for e in log[n0:]], ht.status))
    return out


_HOST = {}
EDGE = {"walk_left": "left", "walk_right": "right", "walk_top": "top", "walk_bottom": "bottom", "walk_corner": "corner"}


def inside(box):
    """the face lies wholly on the canvas"""
    return box is not None and box[0] >= 0 and box[1] >= 0 and box[0] + box[2] <= LW and box[1] + box[2] <= LH


@pytest.mark.parametrize("entry", ["step", "feed"])
def test_tracker_follows_faces_off_the_canvas_and_back(blob, entry):
    """TrackerSet, one stream per walk clip: on a 320x240 canvas (step), or from 640x480 video - every pixel
    replicated 2 x 2, which drawImage maps back onto the canvas exactly - (feed).  Every event and status equals
    main.Tracker over the oracle; head events to 1e-9 (check_events)."""
    from headtrackr_b200 import Context
    from headtrackr_b200.streams import TrackerSet
    paths = list(LIFE_PATHS)
    for p in paths:
        if p not in _HOST:
            _HOST[p] = host_lifecycle(blob, p)
    c = Context(max_width=LW, max_height=LH, max_frames=len(paths))
    try:
        ts = TrackerSet(c, len(paths), {})
        log = [[] for _ in paths]
        ts.addEventListener(lambda k, e: log[k].append(e))
        branches = {p: set() for p in paths}
        lost_by_leaving = {p: False for p in paths}
        refound = {p: False for p in paths}
        for t in range(LIFE_T):
            marks = [len(x) for x in log]
            if t == 0:
                ts.start()
            frames = [frame(p, t, LW, LH) for p in paths]
            now = 1.0e12 + MS * (t + 1)
            if entry == "step":
                recs = ts.step(np.stack(frames), now_ms=now)
            else:
                big = {k: np.ascontiguousarray(np.repeat(np.repeat(f, 2, axis=0), 2, axis=1))
                       for k, f in enumerate(frames)}
                recs = ts.feed(big, now_ms=now, width=LW, height=LH)
            for k, p in enumerate(paths):
                got = [{kk: v for kk, v in e.items() if kk != "time"} for e in log[k][marks[k]:]]
                want_events, want_status = _HOST[p][t]
                check_events(got, want_events)
                assert ts.status[k] == want_status, (p, t, ts.status[k], want_status)
                if recs[k]["head"]["valid"]:
                    branches[p].add(edge_branch(recs[k]["head"]["face"], LW, LH))
                statuses = [e["status"] for e in got if e["type"] == "headtrackrStatus"]
                if "redetecting" in statuses and not inside(face_box(p, t, LW, LH)):
                    lost_by_leaving[p] = True
                if "found" in statuses and lost_by_leaving[p]:
                    refound[p] = True
        for p in paths:
            assert lost_by_leaving[p] and refound[p], p
        for p in paths:
            assert {"none", EDGE[p]} <= branches[p], (p, branches[p])
    finally:
        c.close()
