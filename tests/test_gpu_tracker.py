"""GPU: ht_tracker_step / TrackerSet - headtrackr.Tracker per stream on the device from its first frame - replaying
every case of the reference's own src/main.js runs (tests/golden/reference_js_lifecycle.json and
reference_js_main.json) from frame 0, stop() included, in mixed batches: streams started on different frames, one never
started, one that only ever sees black frames, so that IDLE, STARTING, WB, VJ and CS streams share frame quads."""
import numpy as np
import pytest

from headtrackr_b200 import Context
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE, HtError
from headtrackr_b200.streams import TrackerSet
from test_host_lifecycle import GOLD_L, case_spec, make_frame, strip_time
from test_host_main import GOLD_M, check_events, same

pytestmark = pytest.mark.gpu

W, H = GOLD_L["width"], GOLD_L["height"]
LIFE = {c["name"]: c for c in GOLD_L["cases"]}
MAIN = {c["name"]: c for c in GOLD_M["cases"]}
# one batch per parameter set: (golden case, first frame) per stream; None = never started, "black" = black frames only
BATCHES = {
    "default": ({}, [(LIFE["starter_black"], 0), (LIFE["wb_unstable"], 0), (LIFE["hints"], 0), (MAIN["default"], 0),
                     (LIFE["starter_black"], 3), (LIFE["hints"], 2), (MAIN["default"], 5), (LIFE["wb_unstable"], 7),
                     None, "black"]),
    "no_retry": ({"retryDetection": False}, [(LIFE["no_retry"], 0), (LIFE["no_retry"], 4), None, "black"]),
    "no_smoothing_fov": (MAIN["no_smoothing_fov"]["params"],
                         [(MAIN["no_smoothing_fov"], 0), (MAIN["no_smoothing_fov"], 6), None, "black"]),
}
# one clock for the whole batch: 1000 ms per frame makes "hints" of the hints case and changes no other case (their
# detection phases are shorter than 5 s)
MS = 1000.0


def black():
    f = np.zeros((H, W, 4), np.uint8)
    f[..., 3] = 255
    return f


def replay(batch, io):
    params, streams = BATCHES[batch]
    n = len(streams)
    c = Context(max_width=W, max_height=H, max_frames=16)
    try:
        ts = TrackerSet(c, n, params, device_events=(io == "torch"))
        log = [[] for _ in range(n)]
        ts.addEventListener(lambda k, e: log[k].append(e))
        specs = [case_spec(s[0])[0] if isinstance(s, tuple) else None for s in streams]
        T = max(s[1] + len(sp) for s, sp in zip(streams, specs) if sp) + 2
        modes_seen = set()
        for t in range(T):
            frames, marks = [], []
            for k, s in enumerate(streams):
                marks.append(len(log[k]))
                f = black()
                if s == "black" and t == 0:
                    ts.start(k)
                if isinstance(s, tuple) and 0 <= t - s[1] < len(specs[k]):
                    action, kind, tt = specs[k][t - s[1]]
                    if action == "start":
                        ts.start(k)
                    if action == "stop":
                        ts.stop(k)                        # this stream's frame is not looked at on a stop step
                    else:
                        f = make_frame(kind, tt)
                frames.append(f)
            batch_frames = np.stack(frames)
            if io == "torch":
                import torch
                batch_frames = torch.from_numpy(batch_frames).cuda()
                torch.cuda.synchronize()                  # the library runs on its own stream
            recs = ts.step(batch_frames, now_ms=1.0e12 + MS * t)
            for k, s in enumerate(streams):
                got = strip_time(log[k][marks[k]:])
                modes_seen.add(recs[k]["detection"])
                if not isinstance(s, tuple) or not (0 <= t - s[1] < len(specs[k])):
                    if not (isinstance(s, tuple) and t - s[1] >= len(specs[k])):
                        assert got == [] and not recs[k]["running"], (k, t, got)   # idle / starter on black frames
                    continue
                want = s[0]["steps"][t - s[1]]
                check_events(got, want["events"])
                for g, w in zip(got, want["events"]):
                    if w["type"] == "facetrackingEvent":
                        assert abs(g["angle"] - w["angle"]) <= 1e-12
                assert ts.status[k] == want["status"], (k, t, ts.status[k], want["status"])
                if "fov" in want:
                    assert same(ts.getFOV(k), want["fov"]), (k, t)
                if t - s[1] == len(specs[k]) - 1:           # the case's closing stop()
                    m = len(log[k])
                    ts.stop(k)
                    check_events(strip_time(log[k][m:]), s[0]["stop_events"])
                    assert same(ts.getFOV(k), s[0]["fov"])
        assert {"WB", "VJ", "CS", ""} <= modes_seen
        for k, s in enumerate(streams):
            if s is None or s == "black":
                assert log[k] == [] and ts.status[k] == ""
        # the facetrackr-only entry points share the tracker slots: refused while the lifecycle is on, usable after
        with pytest.raises(HtError) as e:
            c.stream_step(np.stack([black()] * 2), 5, 1)
        assert e.value.code == HT_ERR_STATE
        c.tracker_config(enable=False)
        ev = c.stream_step(np.stack([black()] * 2), 5, 1)
        assert ev[0]["detection"] == "VJ" and ev[1]["detection"] == "VJ"
        with pytest.raises(HtError) as e:
            c.tracker_step(np.stack([black()] * 2), 0.0)
        assert e.value.code == HT_ERR_STATE
    finally:
        c.close()


@pytest.mark.parametrize("io", ["host", "torch"])
@pytest.mark.parametrize("batch", list(BATCHES))
def test_tracker_step_replays_main_js_from_frame_0(batch, io):
    replay(batch, io)


def test_stream_ranges_past_int_max_are_refused():
    """A stream range whose end overflows int is outside [0, max_frames) like any other: ht_stream_reset and
    ht_tracker_reset / start / stop refuse it, and the tracker states stay as they were."""
    c = Context(max_width=W, max_height=H, max_frames=4)
    try:
        c.tracker_config()
        c.tracker_reset(0, 4)
        c.tracker_start(0, 2)
        states = c.tracker_export(list(range(4)))
        for fn in ("ht_stream_reset", "ht_tracker_reset", "ht_tracker_start", "ht_tracker_stop"):
            for first, n in ((2**31 - 1, 1), (1, 2**31 - 1), (3, 2), (-1, 1), (0, 0)):
                assert getattr(c._L, fn)(c._h, first, n) == HT_ERR_ARG, (fn, first, n)
                assert c._L.ht_last_error(c._h).decode() == "stream range outside [0,4)", (fn, first, n)
        assert np.array_equal(c.tracker_export(list(range(4))), states)
    finally:
        c.close()
