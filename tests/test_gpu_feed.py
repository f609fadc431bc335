"""GPU: ht_tracker_feed / TrackerSet.feed - headtrackr.Tracker per stream on the device, each stream ticked from its own
video frame (any size, optionally row-padded), on its own clock, only when its timer fires.

  * every case of the reference's own src/main.js runs (tests/golden/reference_js_lifecycle.json and
    reference_js_main.json) replayed in the stream mixes of test_gpu_tracker.py, each stream's video its golden frame
    replicated k x k per pixel (which draws back onto the golden's canvas exactly, test_feed_host.py), each call listing
    a seeded random subset of the streams in shuffled order;
  * off the replication lattice: synth videos of four sizes fed onto a 320x240 canvas equal, record for record,
    ht_ingest + ht_tracker_step of the same ticks on one context per stream;
  * every rejection, each a single call on well-formed memory, leaves the context as it was."""
import ctypes as C
import math

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE, HtError
from headtrackr_b200.streams import TrackerSet
from test_gpu_tracker import BATCHES, H, W, black
from test_host_lifecycle import case_spec, make_frame, strip_time
from test_host_main import check_events, same

pytestmark = pytest.mark.gpu

FACTORS = (1, 2, 3, 4)
PADDED = 1                         # this stream's video is a row-padded view


def video(frame, k, pad):
    """frame replicated k x k per pixel; pad: rows padded by 5 pixels of 0xAB (pitch > 4 * width)"""
    v = np.repeat(np.repeat(frame, k, axis=0), k, axis=1)
    if not pad:
        return np.ascontiguousarray(v)
    buf = np.full((v.shape[0], v.shape[1] + 5, 4), 0xAB, np.uint8)
    buf[:, :v.shape[1]] = v
    return buf[:, :v.shape[1]]


def to_device(v):
    import torch
    if v.strides[0] == 4 * v.shape[1]:
        return torch.from_numpy(np.ascontiguousarray(v)).cuda()
    base = v.base if v.base is not None else v
    while base.base is not None:
        base = base.base
    t = torch.from_numpy(np.ascontiguousarray(base)).cuda()      # keep the padding: a strided view of the tensor
    return t[:, :v.shape[1]]


def replay(batch, io, seed=7):
    """io: "numpy-host" / "torch-device" / "torch-host" (frames - records), or "mixed": step and feed calls alternate"""
    params, streams = BATCHES[batch]
    n = len(streams)
    frames_dev = io.startswith("torch") or io == "mixed"
    rng = np.random.default_rng(seed)
    c = Context(max_width=W, max_height=H, max_frames=16)
    try:
        ts = TrackerSet(c, n, params, device_events=(io == "torch-device"))
        log = [[] for _ in range(n)]
        ts.addEventListener(lambda k, e: log[k].append(e))
        specs = [case_spec(s[0]) if isinstance(s, tuple) else (None, 1000.0) for s in streams]
        pos = [0] * n                                  # ticks of each stream's own timer so far
        offset = [1.0e12 + 7919.0 * k for k in range(n)]

        def clock(k):                                  # the golden's clock: ms per frame of the case, per stream
            if io == "mixed":                          # step takes one clock: 1000 ms per frame for every stream
                return 1.0e12 + 1000.0 * (pos[k] + 1)
            return offset[k] + specs[k][1] * (pos[k] + 1)

        def finished(k):
            s = streams[k]
            return isinstance(s, tuple) and pos[k] - s[1] >= len(specs[k][0])

        listed_total = [0] * n
        call = 0
        while not all(finished(k) or not isinstance(streams[k], tuple) for k in range(n)) or call < 12:
            use_step = io == "mixed" and call % 2 == 0
            if use_step or io == "mixed":
                chosen = list(range(n))
            else:
                chosen = [k for k in range(n) if rng.random() < 0.6] or [int(rng.integers(n))]
            rng.shuffle(chosen)
            listed, vids, clocks, marks, stops = [], {}, {}, {}, []
            for k in chosen:
                s = streams[k]
                marks[k] = len(log[k])
                f = black()
                if s == "black" and pos[k] == 0:
                    ts.start(k)
                j = pos[k] - s[1] if isinstance(s, tuple) else -1
                if isinstance(s, tuple) and 0 <= j < len(specs[k][0]):
                    action, kind, tt = specs[k][0][j]
                    if action == "start":
                        ts.start(k)
                    if action == "stop":
                        ts.stop(k)                     # this stream's timer does not fire on a stop step
                        stops.append(k)
                        if not use_step:
                            continue
                    else:
                        f = make_frame(kind, tt)
                listed.append(k)
                clocks[k] = clock(k)
                vids[k] = f if use_step else video(f, FACTORS[k % 4], k == PADDED)
            if use_step:
                batch_frames = np.stack([vids[k] for k in range(n)])
                if frames_dev:
                    import torch
                    batch_frames = torch.from_numpy(batch_frames).cuda()
                    torch.cuda.synchronize()
                got_recs = dict(enumerate(ts.step(batch_frames, now_ms=clocks[0])))
            elif listed:
                if frames_dev:
                    import torch
                    vids = {k: to_device(v) for k, v in vids.items()}
                    torch.cuda.synchronize()           # the library runs on its own stream
                got_recs = ts.feed(vids, now_ms=clocks, width=W, height=H)
                assert list(got_recs) == listed
            else:
                got_recs = {}
            for k in chosen:
                s = streams[k]
                rec = got_recs.get(k)
                got = strip_time(log[k][marks[k]:])
                if rec is not None:
                    listed_total[k] += 1
                j = pos[k] - s[1] if isinstance(s, tuple) else -1
                if not isinstance(s, tuple) or j < 0:
                    assert got == [] and not rec["running"] and rec["detection"] == "", (k, call, got, rec)
                elif j < len(specs[k][0]):
                    want = s[0]["steps"][j]
                    check_events(got, want["events"])
                    for g, w in zip(got, want["events"]):
                        if w["type"] == "facetrackingEvent":
                            assert abs(g["angle"] - w["angle"]) <= 1e-12
                    assert ts.status[k] == want["status"], (k, call, ts.status[k], want["status"])
                    if "fov" in want:
                        assert same(ts.getFOV(k), want["fov"]), (k, call)
                    if j == len(specs[k][0]) - 1:      # the case's closing stop()
                        m = len(log[k])
                        ts.stop(k)
                        check_events(strip_time(log[k][m:]), s[0]["stop_events"])
                        assert same(ts.getFOV(k), s[0]["fov"])
                pos[k] += 1
            call += 1
            assert call < 2000
        for k, s in enumerate(streams):
            if s is None:
                assert log[k] == [] and ts.status[k] == "" and listed_total[k] > 0
        return c
    except BaseException:
        c.close()
        raise


@pytest.mark.parametrize("io", ["numpy-host", "torch-device", "torch-host", "mixed"])
@pytest.mark.parametrize("batch", list(BATCHES))
def test_tracker_feed_replays_main_js_from_frame_0(batch, io):
    c = replay(batch, io)
    c.close()


def equal_records(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(equal_records(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(equal_records(x, y) for x, y in zip(a, b))
    if isinstance(a, float) and math.isnan(a):
        return isinstance(b, float) and math.isnan(b)
    return a == b


def test_feed_equals_ingest_plus_step_off_the_lattice():
    CW, CH = 320, 240
    sizes = [(640, 480), (1280, 720), (333, 251), (200, 150)] * 2
    videos = [synth.frame(200 + i, w, h, n_faces=1) for i, (w, h) in enumerate(sizes)]
    pad = np.full((251, 340, 4), 0xAB, np.uint8)                    # one row-padded video
    pad[:, :333] = videos[2]
    videos[2] = pad[:, :333]
    n = len(videos)
    rng = np.random.default_rng(11)
    one = Context(max_width=CW, max_height=CH, max_frames=n)
    solo = [Context(max_width=CW, max_height=CH, max_frames=1) for _ in range(n)]
    try:
        one.tracker_config()
        one.tracker_reset(0, n)
        one.tracker_start(0, n)
        for c in solo:
            c.tracker_config()
            c.tracker_reset(0, 1)
            c.tracker_start(0, 1)
        clock = [1.0e12 + 333.0 * k for k in range(n)]
        modes = set()
        cs_streams = set()
        for tick in range(40):
            ks = [k for k in range(n) if rng.random() < 0.75] or [0]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 20.0 + 5.0 * (k % 3)
            got = one.tracker_feed(ks, [videos[k] for k in ks], [clock[k] for k in ks], CW, CH)
            for k, rec in zip(ks, got):
                canvas = solo[k].ingest(np.ascontiguousarray(videos[k]), CW, CH)
                want = solo[k].tracker_step(canvas, clock[k])[0]
                assert equal_records(rec, want), (tick, k, rec, want)
                modes.add(rec["detection"])
                if rec["detection"] == "CS":
                    cs_streams.add(k)
        assert cs_streams, modes
        assert {"WB", "VJ"} <= modes
    finally:
        one.close()
        for c in solo:
            c.close()


def feed_raw(c, recs, on_device, cw, ch):
    arr = (_lib.VideoFrame * max(1, len(recs)))(*recs)
    out = (_lib.TrackerEvent * max(1, len(recs)))()
    return c._L.ht_tracker_feed(c._h, C.addressof(arr), len(recs), on_device, cw, ch, C.addressof(out)), list(out)


def test_feed_rejections_enqueue_nothing():
    import torch
    MAXF = 4
    f = synth.frame(1, W, H, n_faces=1)
    p = f.ctypes.data

    def rec(stream=0, ptr=None, w=W, h=H, pitch=0):
        return _lib.VideoFrame(p if ptr is None else ptr, stream, w, h, pitch, 1.0e12)

    c = Context(max_width=W, max_height=H, max_frames=MAXF)
    ref = Context(max_width=W, max_height=H, max_frames=MAXF)
    try:
        assert feed_raw(c, [rec()], 0, W, H)[0] == HT_ERR_STATE          # lifecycle not configured
        for x in (c, ref):
            x.tracker_config()
            x.tracker_reset(0, MAXF)
            x.tracker_start(0, MAXF)
        dev = torch.from_numpy(f).cuda()
        torch.cuda.synchronize()
        cases = [
            (HT_ERR_ARG, [], 0, W, H),                                       # n = 0
            (HT_ERR_ARG, [rec(k) for k in range(MAXF)] + [rec(0)], 0, W, H),  # n > max_frames
            (HT_ERR_ARG, [rec(-1)], 0, W, H),
            (HT_ERR_ARG, [rec(MAXF)], 0, W, H),
            (HT_ERR_ARG, [rec(1), rec(2), rec(1)], 0, W, H),                  # listed twice
            (HT_ERR_ARG, [rec(0), rec(1, ptr=0)], 0, W, H),                   # NULL pixels
            (HT_ERR_ARG, [rec(0, ptr=p + 2)], 0, W, H),                       # pointer not a multiple of 4
            (HT_ERR_ARG, [rec(0, pitch=4 * W + 2)], 0, W, H),                 # pitch not a multiple of 4
            (HT_ERR_ARG, [rec(0, w=W // 2, h=H // 2, pitch=4 * (W // 2) - 4)], 0, W, H),   # pitch below 4 * width
            (HT_ERR_SIZE, [rec(0, w=0)], 0, W, H),
            (HT_ERR_SIZE, [rec(0, w=1, h=16385, pitch=4 * W)], 0, W, H),
            (HT_ERR_SIZE, [rec(0)], 0, W + 1, H),                             # canvas above max_width
            (HT_ERR_SIZE, [rec(0)], 0, 20, 20),                               # too small for the pyramid
            (HT_ERR_SIZE, [rec(0)], 0, 0, H),
            (HT_ERR_ARG, [rec(0)], 1, W, H),                                  # host pixels, frames_on_device = 1
            (HT_ERR_ARG, [rec(0, ptr=dev.data_ptr())], 0, W, H),              # device pixels, frames_on_device = 0
        ]
        for i, (code, recs, on_dev, cw, ch) in enumerate(cases):
            rc = feed_raw(c, recs, on_dev, cw, ch)[0]
            assert rc == code, (i, rc, c._L.ht_last_error(c._h))
            assert c._L.ht_last_error(c._h)
        # nothing was enqueued: the rejected context ticks exactly like one that never saw those calls
        for tick in range(3):
            ks = [2, 0] if tick != 1 else [3]
            vids = [f] * len(ks) if tick != 2 else [dev] * len(ks)
            if tick == 2:
                torch.cuda.synchronize()
            a = c.tracker_feed(ks, vids, 1.0e12 + 40.0 * tick, W, H)
            b = ref.tracker_feed(ks, vids, 1.0e12 + 40.0 * tick, W, H)
            assert equal_records(a, b) and all(r["detection"] == "WB" for r in a), (a, b)
        with pytest.raises(HtError) as e:
            c.tracker_feed([0], [f], 0.0, W, H + 8)
        assert e.value.code == HT_ERR_SIZE
    finally:
        c.close()
        ref.close()
