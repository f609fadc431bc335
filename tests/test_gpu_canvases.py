"""GPU: per-stream Tracker parameters (ht_tracker_set_params) and a canvas per record (ht_tracker_feed_canvases) -
streams of one context behaving as independent `new headtrackr.Tracker(params)` + `init(video, canvas)` objects:

  * one TrackerSet replays every case of the reference's own src/main.js runs (reference_js_lifecycle.json,
    reference_js_main.json at 160x120, reference_js_params.json at 200x150 and 120x160) from frame 0, each stream with
    its case's parameters and canvas, all in the same ht_tracker_feed_canvases calls; the 160x120 cases also through
    ht_tracker_step with per-stream parameters;
  * off the replication lattice: synth videos onto canvases of four sizes in one call equal, record for record, one
    single-stream context per stream doing ht_ingest + ht_tracker_step with that stream's canvas and parameters;
  * max_frames records on max_frames distinct canvas sizes;
  * rejections enqueue nothing; ht_tracker_config after per-stream parameters sets every stream again."""
import ctypes as C
import json
import math
import sys
from pathlib import Path

import numpy as np
import pytest

import test_gpu_tracker
from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.context import tracker_params
from headtrackr_b200.streams import TrackerSet
from test_gpu_feed import equal_records, to_device, video
from test_host_lifecycle import GOLD_L, case_spec, strip_time
from test_host_lifecycle import make_frame as frame_160
from test_host_main import GOLD_M, check_events, same

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD_P = json.loads((Path(__file__).resolve().parent / "golden" / "reference_js_params.json").read_text())
LIFE = {c["name"]: c for c in GOLD_L["cases"]}
MAIN = {c["name"]: c for c in GOLD_M["cases"]}
PAR = {c["name"]: c for c in GOLD_P["cases"]}
W0, H0 = GOLD_L["width"], GOLD_L["height"]


def canvas_of(case):
    return (case.get("width", W0), case.get("height", H0))


def make_frame(case, kind, t):
    if "width" not in case:
        return frame_160(kind, t)
    import make_goldens_params as pg
    return pg.make_frame(kind, t, case["width"], case["height"])


def black(w, h):
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 3] = 255
    return f


def spec_of(case):
    s, ms = case_spec(case)
    return s, case.get("ms_per_frame", ms)


# (golden case, first frame) per stream; ("idle", canvas) = never started, ("black", canvas) = black frames only
STREAMS = ([(c, 0) for c in GOLD_L["cases"]] + [(c, 0) for c in GOLD_M["cases"]] + [(c, 0) for c in GOLD_P["cases"]]
           + [(LIFE["no_retry"], 4), (MAIN["no_smoothing_fov"], 6), (PAR["angles_200x150"], 3),
              (PAR["portrait_120x160"], 5), (PAR["no_head_200x150"], 2), ("idle", (200, 150)), ("black", (120, 160))])


def same_angle(g, w):
    """NaN where the reference has NaN (a face lost with calcAngles on); else equal up to the summation order of the
    moments (1e-9 relative, as check_events compares every field)"""
    return (math.isnan(g) and math.isnan(w)) or same(g, w)


@pytest.mark.parametrize("io", ["numpy-host", "torch-device"])
def test_one_context_replays_every_case_with_its_params_and_canvas(io):
    n = len(STREAMS)
    params = [s[0]["params"] if isinstance(s[0], dict) else {} for s in STREAMS]
    canvases = [canvas_of(s[0]) if isinstance(s[0], dict) else s[1] for s in STREAMS]
    assert len({repr(sorted(p.items())) for p in params}) >= 5 and len(set(canvases)) == 3
    rng = np.random.default_rng(13)
    c = Context(max_width=200, max_height=160, max_frames=32)
    try:
        ts = TrackerSet(c, n, params, device_events=(io == "torch-device"))
        log = [[] for _ in range(n)]
        ts.addEventListener(lambda k, e: log[k].append(e))
        specs = [spec_of(s[0]) if isinstance(s[0], dict) else (None, 1000.0) for s in STREAMS]
        pos = [0] * n
        offset = [1.0e12 + 7919.0 * k for k in range(n)]
        angles_nan = 0
        multi_size_calls = 0

        def finished(k):
            return not isinstance(STREAMS[k][0], dict) or pos[k] - STREAMS[k][1] >= len(specs[k][0])

        call = 0
        while not all(finished(k) for k in range(n)) or call < 12:
            chosen = [k for k in range(n) if rng.random() < 0.6] or [int(rng.integers(n))]
            rng.shuffle(chosen)
            listed, vids, clocks, marks = [], {}, {}, {}
            for k in chosen:
                s, first = STREAMS[k]
                marks[k] = len(log[k])
                f = black(*canvases[k])
                if s == "black" and pos[k] == 0:
                    ts.start(k)
                j = pos[k] - first if isinstance(s, dict) else -1
                if isinstance(s, dict) and 0 <= j < len(specs[k][0]):
                    action, kind, tt = specs[k][0][j]
                    if action == "start":
                        ts.start(k)
                    if action == "stop":
                        ts.stop(k)                     # this stream's timer does not fire on a stop step
                        continue
                    f = make_frame(s, kind, tt)
                listed.append(k)
                clocks[k] = offset[k] + specs[k][1] * (pos[k] + 1)
                vids[k] = video(f, 1 + k % 3, k == 1)
            got_recs = {}
            if listed:
                if io == "torch-device":
                    import torch
                    vids = {k: to_device(v) for k, v in vids.items()}
                    torch.cuda.synchronize()           # the library runs on its own stream
                got_recs = ts.feed(vids, now_ms=clocks, width={k: canvases[k][0] for k in listed},
                                   height={k: canvases[k][1] for k in listed})
                assert list(got_recs) == listed
                multi_size_calls += len({canvases[k] for k in listed}) == 3
            for k in chosen:
                s, first = STREAMS[k]
                rec = got_recs.get(k)
                got = strip_time(log[k][marks[k]:])
                j = pos[k] - first if isinstance(s, dict) else -1
                if not isinstance(s, dict) or j < 0:
                    assert got == [] and not rec["running"] and rec["detection"] == "", (k, call, got, rec)
                elif j < len(specs[k][0]):
                    want = s["steps"][j]
                    check_events(got, want["events"])
                    for g, w in zip(got, want["events"]):
                        if w["type"] == "facetrackingEvent":
                            assert same_angle(g["angle"], w["angle"]), (k, call, g, w)
                            angles_nan += math.isnan(w["angle"])
                    assert ts.status[k] == want["status"], (k, call, ts.status[k], want["status"])
                    if "fov" in want:                  # (reference_js_main.json records getFOV() once per case)
                        assert same(ts.getFOV(k), want["fov"]), (k, call)
                    if j == len(specs[k][0]) - 1:      # the case's closing stop()
                        m = len(log[k])
                        ts.stop(k)
                        check_events(strip_time(log[k][m:]), s["stop_events"])
                        assert same(ts.getFOV(k), s["fov"])
                pos[k] += 1
            call += 1
            assert call < 2000
        assert angles_nan >= 4 and multi_size_calls > 10     # lost faces with calcAngles; calls with every size
        for k, (s, _) in enumerate(STREAMS):
            if not isinstance(s, dict):
                assert log[k] == [] and ts.status[k] == ""
    finally:
        c.close()


def test_tracker_step_with_per_stream_params(monkeypatch):
    """the 160x120 cases of every parameter set in one ht_tracker_step batch, each stream with its own parameters"""
    params, streams = [], []
    for name, (p, ss) in test_gpu_tracker.BATCHES.items():
        for s in (ss if name == "default" else ss[:2]):   # (16 streams: the context's max_frames)
            params.append(p)
            streams.append(s)
    assert len({repr(sorted(p.items())) for p in params}) == 3
    monkeypatch.setitem(test_gpu_tracker.BATCHES, "per_stream", (params, streams))
    test_gpu_tracker.replay("per_stream", "host")


def solo_contexts(n, cw, ch, kw):
    solo = []
    for k in range(n):
        c = Context(max_width=cw, max_height=ch, max_frames=1)
        solo.append(c)
        c.tracker_config(**kw[k])
        c.tracker_reset(0, 1)
        c.tracker_start(0, 1)
    return solo


def run_against_solo(videos, canvas_at, kw, ticks, max_w, max_h, seed):
    """feed_canvases on one context vs ingest + tracker_step on one context per stream -> (records, cs streams)"""
    n = len(videos)
    rng = np.random.default_rng(seed)
    one = Context(max_width=max_w, max_height=max_h, max_frames=n)
    solo = solo_contexts(n, max_w, max_h, kw)
    try:
        one.tracker_config()
        one.tracker_set_params(0, kw)
        one.tracker_reset(0, n)
        one.tracker_start(0, n)
        clock = [1.0e12 + 333.0 * k for k in range(n)]
        cs, modes = set(), set()
        for tick in range(ticks):
            ks = [k for k in range(n) if rng.random() < 0.8] or [0]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 20.0 + 5.0 * (k % 3)
            sizes = [canvas_at(k, tick) for k in ks]
            got = one.tracker_feed(ks, [videos[k] for k in ks], [clock[k] for k in ks], [s[0] for s in sizes],
                                   [s[1] for s in sizes])
            for k, (cw, ch), rec in zip(ks, sizes, got):
                canvas = solo[k].ingest(np.ascontiguousarray(videos[k]), cw, ch)
                want = solo[k].tracker_step(canvas, clock[k])[0]
                assert equal_records(rec, want), (tick, k, (cw, ch), rec, want)
                modes.add(rec["detection"])
                if rec["detection"] == "CS":
                    cs.add(k)
        return cs, modes
    finally:
        one.close()
        for c in solo:
            c.close()


def test_mixed_canvases_equal_one_context_per_stream_off_the_lattice():
    sizes = [(640, 480), (480, 640), (1280, 720), (333, 251), (200, 150), (640, 480), (480, 640), (320, 240)]
    videos = [synth.frame(300 + i, w, h, n_faces=1) for i, (w, h) in enumerate(sizes)]
    pad = np.full((251, 340, 4), 0xAB, np.uint8)                    # one row-padded video
    pad[:, :333] = videos[3]
    videos[3] = pad[:, :333]
    canv = [(320, 240), (240, 320), (320, 240), (200, 150), (200, 150), (160, 120), (240, 320), None]
    kw = [tracker_kw(calcAngles=True, cameraOffset=5.0), tracker_kw(calcAngles=True, fov=60.0),
          tracker_kw(calcAngles=True, smoothing=False), tracker_kw(retryDetection=False),
          tracker_kw(calcAngles=True, headPosition=False), tracker_kw(fov=45.0, cameraOffset=8.0),
          tracker_kw(calcAngles=True), tracker_kw(calcAngles=True, cameraOffset=2.0)]

    def canvas_at(k, tick):                      # stream 7's canvas changes between ticks
        if canv[k] is not None:
            return canv[k]
        return ((320, 240), (200, 150), (160, 120), (240, 320))[(tick // 7) % 4]

    cs, modes = run_against_solo(videos, canvas_at, kw, 45, 320, 320, 11)
    assert {"WB", "VJ", "CS"} <= modes
    assert len([k for k in cs if kw[k]["calcAngles"]]) >= 2, cs


def tracker_kw(**p):
    base = dict(retryDetection=True, calcAngles=False, smoothing=True, fov=None, cameraOffset=11.5, headPosition=True)
    base.update(p)
    return base


def test_max_frames_records_on_max_frames_canvas_sizes():
    sizes = [(160, 120), (161, 121), (163, 97), (120, 160), (200, 150), (101, 89)]
    videos = [synth.frame(400 + i, 320, 240, n_faces=1) for i in range(len(sizes))]
    kw = [tracker_kw(calcAngles=bool(k % 2)) for k in range(len(sizes))]
    cs, modes = run_against_solo(videos, lambda k, tick: sizes[k], kw, 30, 200, 160, 17)
    assert {"WB", "VJ"} <= modes


def canvases_raw(c, recs, on_device):
    arr = (_lib.CanvasFrame * max(1, len(recs)))(*recs)
    out = (_lib.TrackerEvent * max(1, len(recs)))()
    return c._L.ht_tracker_feed_canvases(c._h, C.addressof(arr), len(recs), on_device, C.addressof(out))


def set_params_raw(c, first, plist):
    arr = (_lib.TrackerParams * max(1, len(plist)))(*plist)
    return c._L.ht_tracker_set_params(c._h, first, len(plist), C.addressof(arr) if plist is not None else None)


def test_rejections_enqueue_nothing():
    MAXF, MW, MH = 4, 240, 240
    f = synth.frame(1, 320, 240, n_faces=1)

    def rec(stream=0, cw=160, ch=120):
        return _lib.CanvasFrame(_lib.VideoFrame(f.ctypes.data, stream, 320, 240, 0, 1.0e12), cw, ch)

    good = tracker_params(calcAngles=True, fov=50.0)
    bad_alpha = tracker_params(alpha=1.5)
    bad_dist = tracker_params(distance_to_screen=0.0)
    c = Context(max_width=MW, max_height=MH, max_frames=MAXF)
    ref = Context(max_width=MW, max_height=MH, max_frames=MAXF)
    try:
        assert canvases_raw(c, [rec()], 0) == HT_ERR_STATE                # lifecycle not configured
        assert set_params_raw(c, 0, [good]) == HT_ERR_STATE
        for x in (c, ref):
            x.tracker_config()
            x.tracker_reset(0, MAXF)
            x.tracker_start(0, MAXF)
        param_cases = [(-1, [good]), (0, []), (3, [good, good]), (MAXF, [good]),
                       (0, [good, bad_alpha]), (1, [bad_dist])]
        for i, (first, plist) in enumerate(param_cases):
            rc = set_params_raw(c, first, plist)
            assert rc == HT_ERR_ARG, (i, rc, c._L.ht_last_error(c._h))
        assert c._L.ht_tracker_set_params(c._h, 0, 1, None) == HT_ERR_ARG
        feed_cases = [
            (HT_ERR_SIZE, [rec(0, 0, 120)], 0, 0),
            (HT_ERR_SIZE, [rec(0), rec(1, 160, 0)], 0, 1),
            (HT_ERR_SIZE, [rec(0), rec(1, MW + 1, 120)], 0, 1),         # above max_width
            (HT_ERR_SIZE, [rec(0), rec(1, 200, 150), rec(2, 20, 20)], 0, 2),   # too small for the pyramid
            (HT_ERR_ARG, [rec(0), rec(1, 200, 150), rec(0, 120, 160)], 0, 2),  # a stream listed twice
            (HT_ERR_ARG, [rec(0), rec(1, 200, 150)], 1, None),           # host pixels, frames_on_device = 1
        ]
        for i, (code, recs, on_dev, idx) in enumerate(feed_cases):
            rc = canvases_raw(c, recs, on_dev)
            msg = c._L.ht_last_error(c._h).decode()
            assert rc == code, (i, rc, msg)
            if idx is not None:
                assert msg.startswith(f"record {idx}:"), (i, msg)
        sizes = [(160, 120), (200, 150), (120, 160), (240, 180)]
        for tick in range(3):
            ks = [2, 0, 3] if tick != 1 else [1, 3]
            a = c.tracker_feed(ks, [f] * len(ks), 1.0e12 + 40.0 * tick, [sizes[k][0] for k in ks], [sizes[k][1] for k in ks])
            b = ref.tracker_feed(ks, [f] * len(ks), 1.0e12 + 40.0 * tick, [sizes[k][0] for k in ks], [sizes[k][1] for k in ks])
            assert equal_records(a, b) and all(r["detection"] == "WB" for r in a), (a, b)
    finally:
        c.close()
        ref.close()
    # the rejected parameter records left every stream's parameters as they were: run to CS against a context that
    # never saw them
    videos = [synth.frame(500 + k, 320, 240, n_faces=1) for k in range(MAXF)]
    cs, _ = run_params_after_rejections(videos)
    assert cs


def run_params_after_rejections(videos):
    n = len(videos)
    a = Context(max_width=160, max_height=120, max_frames=n)
    b = Context(max_width=160, max_height=120, max_frames=n)
    try:
        for x in (a, b):
            x.tracker_config()
        assert set_params_raw(a, 0, [tracker_params(calcAngles=True, fov=50.0), tracker_params(alpha=2.0)]) == HT_ERR_ARG
        assert set_params_raw(a, n - 1, [tracker_params(calcAngles=True)] * 2) == HT_ERR_ARG
        for x in (a, b):
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
        cs = set()
        for tick in range(30):
            now = 1.0e12 + 35.0 * tick
            ra = a.tracker_feed(list(range(n)), videos, now, 160, 120)
            rb = b.tracker_feed(list(range(n)), videos, now, 160, 120)
            assert equal_records(ra, rb), tick
            cs |= {k for k, r in enumerate(ra) if r["detection"] == "CS"}
        return cs, None
    finally:
        a.close()
        b.close()


def test_config_after_per_stream_params_sets_every_stream():
    n = 4
    videos = [synth.frame(600 + k, 320, 240, n_faces=1) for k in range(n)]
    uniform = tracker_kw(calcAngles=True, cameraOffset=4.0, fov=52.0)
    a = Context(max_width=200, max_height=150, max_frames=n)
    b = Context(max_width=200, max_height=150, max_frames=n)
    try:
        a.tracker_config()
        a.tracker_set_params(0, [tracker_kw(retryDetection=False), tracker_kw(calcAngles=True, fov=70.0),
                                 tracker_kw(smoothing=False, headPosition=False), tracker_kw(cameraOffset=20.0)])
        a.tracker_config(**uniform)
        b.tracker_config(**uniform)
        for x in (a, b):
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
        sizes = [(200, 150), (160, 120), (200, 150), (120, 150)]
        cs = set()
        for tick in range(40):
            now = 1.0e12 + 35.0 * tick
            ra = a.tracker_feed(list(range(n)), videos, now, [s[0] for s in sizes], [s[1] for s in sizes])
            rb = b.tracker_feed(list(range(n)), videos, now, [s[0] for s in sizes], [s[1] for s in sizes])
            assert equal_records(ra, rb), tick
            cs |= {k for k, r in enumerate(ra) if r["detection"] == "CS"}
        assert cs
    finally:
        a.close()
        b.close()
