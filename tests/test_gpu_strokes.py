"""GPU: main.js's strokes drawn on each stream's debug canvas by k_debug_strokes (ht_tracker_set_debug_strokes,
TrackerSet's "debugStrokes"), against the C restatement tests/stroke_oracle.c applied to the device's own records (the
raster is a function of the record; the device's angle may differ from the oracle's in its last bits):

  * every case of reference_js_debug.json through TrackerSet.step and TrackerSet.feed with strokes on: after every
    tick each debug canvas is the twin context's (strokes off) back-projection composite, then the restated strokes
    of the tick's debug_calls; records are byte-identical to the twin's;
  * one ht_tracker_feed_canvases call per tick over three canvas sizes, debug canvases smaller, larger and row-padded,
    carved out of one sentinel-filled buffer: only the clipped back-projection and the strokes are written;
  * 1024 streams of 640x480 in random subsets, half with calcAngles on;
  * the flag's lifetime across config, set_debug, set_params, stop, start, reset and import, the launch count, and
    rejections that leave every setting in force."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet, debug_calls
from test_debug_host import GOLD_D, debug_canvas, make_frame
from test_gpu_debug import black, carve, run
from test_gpu_feed import equal_records, to_device, video
from test_strokes_host import oracle_calls, so  # noqa: F401  (fixture: the C restatement)

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]


def torch():
    import torch as t
    return t


def expect(so, exp, twin, rec, cw, ch):  # noqa: F811
    """one tick of a stream on the host copy `exp` ((Dh, Dw, 4) uint8): the twin's back-projection on a CS tick
    (min(cw, Dw) x min(ch, Dh) of its canvas `twin`), then the restated strokes of the record's debug_calls"""
    if rec["detection"] == "CS":
        h, w = min(ch, exp.shape[0]), min(cw, exp.shape[1])
        exp[:h, :w] = twin[:h, :w]
    flat = np.ascontiguousarray(exp)
    oracle_calls(so, debug_calls(rec), flat, exp.shape[1], exp.shape[0], 4 * exp.shape[1])
    exp[...] = flat


def host(t):
    return t.cpu().numpy()


def stroked(d):
    """a pixel that is not grey: the back-projection is (v, v, v, 255), the strokes are blue or green"""
    return bool(((d[..., 0] != d[..., 1]) | (d[..., 1] != d[..., 2])).any())


@pytest.mark.parametrize("path", ["step", "feed"])
def test_golden_replay(so, path):  # noqa: F811
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    try:
        dbg = [T.from_numpy(debug_canvas(case)).cuda() for case in cases]
        twin = [d.clone() for d in dbg]
        exp = [host(d) for d in dbg]
        ts = TrackerSet(c, n, [dict(case["params"], debug=dbg[k], debugStrokes=True) for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], debug=twin[k]) for k, case in enumerate(cases)])
        T.cuda.synchronize()
        clock = 1.0e12
        n_stroked = rotated = nan = 0
        for i in range(max(len(case["steps"]) for case in cases)):
            clock += 35.0
            frames, listed = [], []
            for k, case in enumerate(cases):
                f = black(W0, H0)
                if i < len(case["steps"]):
                    s = case["steps"][i]
                    f = make_frame(*s["frame"])
                    if s["action"] == "start":
                        ts.start(k), tr.start(k)
                    elif s["action"] == "stop":
                        ts.stop(k), tr.stop(k)
                    if s["action"] != "stop":
                        listed.append(k)
                elif i == len(case["steps"]):
                    ts.stop(k), tr.stop(k)
                frames.append(f)
            if path == "step":
                batch = T.from_numpy(np.stack(frames)).cuda()
                T.cuda.synchronize()
                recs = ts.step(batch, clock)
                assert equal_records(recs, tr.step(batch, clock)), i
                ticked = dict(enumerate(recs))
            elif listed:
                vids = {k: to_device(video(frames[k], 1 + k % 3, k == 1)) for k in listed}
                T.cuda.synchronize()
                ticked = ts.feed(vids, clock, W0, H0)
                assert equal_records(list(ticked.values()), list(tr.feed(vids, clock, W0, H0).values())), i
            else:
                ticked = {}
            for k, rec in ticked.items():
                expect(so, exp[k], host(twin[k]), rec, W0, H0)
                calls = debug_calls(rec)
                n_stroked += bool(calls)
                rot = [x[1] for x in calls if x[0] == "rotate"]
                rotated += bool(rot) and rot[0] == rot[0] and abs(rot[0]) > 1e-3
                nan += bool(rot) and rot[0] != rot[0]
            for k in range(n):
                assert np.array_equal(host(dbg[k]), exp[k]), (cases[k]["name"], i)
        assert n_stroked > 50 and rotated > 0 and nan > 0
    finally:
        c.close()
        ref.close()


def test_mixed_canvases_write_only_backprojection_and_strokes(so):  # noqa: F811
    """one ht_tracker_feed_canvases call per tick: 160x120, 200x150 and 120x160 canvases; debug canvases smaller,
    larger, narrower and taller, row-padded, carved out of one buffer of sentinel bytes; stream 3 has no canvas but
    strokes on, stream 4 a canvas and strokes off"""
    T = torch()
    import make_goldens_params as pg
    canv = [(160, 120), (200, 150), (120, 160), (160, 120), (200, 150), (120, 160)]
    spec = [(100, 80, 400), (240, 180, 960), (120, 160, 4 * 120 + 36), None, (200, 150, 800), (64, 200, 4 * 64 + 4)]
    offs, off = [], 64
    for s in spec:
        offs.append(off)
        if s:
            off += s[2] * s[1] + 64
    buf = T.full((off + 64,), 0x5A, dtype=T.uint8, device="cuda")
    tbuf = buf.clone()
    exp = host(buf).copy()
    views = [carve(buf, o, *s) if s else None for o, s in zip(offs, spec)]
    tviews = [carve(tbuf, o, *s) if s else None for o, s in zip(offs, spec)]
    ctx = Context(max_width=200, max_height=160, max_frames=8)
    ref = Context(max_width=200, max_height=160, max_frames=8)
    try:
        for x, v in ((ctx, views), (ref, tviews)):
            x.tracker_config()
            x.tracker_reset(0, 6)
            x.tracker_start(0, 6)
            x.tracker_set_debug(0, v)
        ctx.tracker_set_debug_strokes(0, [1, 1, 1, 1, 0, 1])
        T.cuda.synchronize()
        rng = np.random.default_rng(5)
        drawn = set()
        for tick in range(40):
            ks = [k for k in range(6) if rng.random() < 0.85] or [0]
            rng.shuffle(ks)
            frames = {k: pg.make_frame("face", tick, *canv[k]) for k in ks}
            vids = [to_device(video(frames[k], 1 + k % 2, k == 2)) for k in ks]
            T.cuda.synchronize()
            args = (ks, vids, 1.0e12 + 35.0 * tick, [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            recs = ctx.tracker_feed(*args)
            assert equal_records(recs, ref.tracker_feed(*args)), tick
            tb = host(tbuf)
            for k, rec in zip(ks, recs):
                if not spec[k]:
                    continue
                dw, dh, pitch = spec[k]
                e = np.lib.stride_tricks.as_strided(exp[offs[k]:], (dh, dw, 4), (pitch, 4, 1))
                t = np.lib.stride_tricks.as_strided(tb[offs[k]:], (dh, dw, 4), (pitch, 4, 1))
                if k == 4:                                   # strokes off: the back-projection only
                    if rec["detection"] == "CS":
                        h, w = min(canv[k][1], dh), min(canv[k][0], dw)
                        e[:h, :w] = t[:h, :w]
                    continue
                patch = e.copy()
                expect(so, patch, t, rec, *canv[k])
                e[...] = patch
                if debug_calls(rec):
                    drawn.add(k)
            assert np.array_equal(host(buf), exp), tick
        assert drawn == {0, 1, 2, 5}
        assert (host(buf) == 0x5A).any()
    finally:
        ctx.close()
        ref.close()


def test_1024_streams_640x480_random_subsets(so):  # noqa: F811
    T = torch()
    n, W, H = 1024, 640, 480
    rng = np.random.default_rng(29)
    frames = [T.from_numpy(synth.frame(900 + i, W, H, n_faces=1)).cuda() for i in range(16)]
    dbg = T.zeros((n, H, W, 4), dtype=T.uint8, device="cuda")
    twin = T.zeros_like(dbg)
    ctx = Context(max_width=W, max_height=H, max_frames=n)
    ref = Context(max_width=W, max_height=H, max_frames=n)
    try:
        angles = [dict(calcAngles=bool(k % 2)) for k in range(n)]
        for x, d in ((ctx, dbg), (ref, twin)):
            x.tracker_config()
            x.tracker_set_params(0, [dict(retryDetection=True, calcAngles=a["calcAngles"], smoothing=True, fov=None,
                                          cameraOffset=11.5, headPosition=True) for a in angles])
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
            x.tracker_set_debug(0, [d[k] for k in range(n)])
        ctx.tracker_set_debug_strokes(0, [1] * n)
        T.cuda.synchronize()
        follow = {}                                          # stream -> its expected canvas, once picked
        clock = [1.0e12 + 17.0 * k for k in range(n)]
        checked = rotated = 0
        for tick in range(32):
            ks = [k for k in range(n) if rng.random() < 0.85]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            args = (ks, [frames[k % 16] for k in ks], [clock[k] for k in ks], W, H)
            recs = ctx.tracker_feed(*args)
            assert equal_records(recs, ref.tracker_feed(*args)), tick
            for k, rec in zip(ks, recs):
                if k in follow:
                    expect(so, follow[k], host(twin[k]), rec, W, H)
                    checked += bool(debug_calls(rec))
                    rotated += rec["detection"] == "CS" and k % 2 == 1 and abs(rec["angle"] - np.pi / 2) > 1e-3
            for k in follow:
                assert np.array_equal(host(dbg[k]), follow[k]), (tick, k)
            if len(follow) < 96:                             # 8 more streams followed from the next tick on
                for k in rng.choice([k for k in range(n) if k not in follow], 8, replace=False):
                    follow[int(k)] = host(dbg[int(k)]).copy()
        assert checked > 200 and rotated > 0
    finally:
        ctx.close()
        ref.close()


# ---- lifetime, launches, rejections ---------------------------------------------------------------------------------

def test_lifetime():
    T = torch()
    import make_goldens_params as pg
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        d = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
        ctx.tracker_set_debug_strokes(0, [1])               # before the canvas: the flag is the stream's
        ctx.tracker_set_debug(0, [d])
        T.cuda.synchronize()
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]

        def green(t):
            """one CS tick on a cleared canvas; -> whether a stroke was drawn on the back-projection"""
            d.zero_()
            T.cuda.synchronize()
            recs = run(ctx, 1, t)
            T.cuda.synchronize()
            assert recs[0]["detection"] == "CS"
            return stroked(d)

        assert green(30)
        ctx.tracker_set_params(0, [dict(calcAngles=True)])
        assert green(31)                                     # set_params keeps it
        ctx.tracker_set_debug(0, [None])
        ctx.tracker_set_debug(0, [d])
        assert green(32)                                     # set_debug keeps it
        snap = ctx.tracker_export([0])
        ctx.tracker_stop(0, 1)
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        ctx.tracker_import([0], snap)
        assert green(33)                                     # stop / reset / start / import keep it
        ctx.tracker_set_debug_strokes(0, [0])
        assert not green(34)
        ctx.tracker_set_debug_strokes(0, [1])
        ctx.tracker_config()                                 # clears canvases and flags
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        ctx.tracker_set_debug(0, [d])
        run(ctx, 22, 40)
        assert not green(62)
        ts_ctx = Context(max_width=W0, max_height=H0, max_frames=2)
        try:
            e = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
            ts = TrackerSet(ts_ctx, 2, [dict(debug=e, debugStrokes=True), {}])
            ts.start()
            for t in range(22):
                ts.feed({0: pg.make_frame("face", t, W0, H0)}, 1.0e12 + 35.0 * t, W0, H0)
            T.cuda.synchronize()
            assert ts.current[0]["detection"] == "CS" and stroked(e)
            ts.set_params(0, {"debug": e})                   # no "debugStrokes" key: off
            e.zero_()
            T.cuda.synchronize()
            ts.feed({0: pg.make_frame("face", 22, W0, H0)}, 1.0e12 + 35.0 * 22, W0, H0)
            T.cuda.synchronize()
            assert ts.current[0]["detection"] == "CS" and not stroked(e)
        finally:
            ts_ctx.close()
    finally:
        ctx.close()


def test_launch_count():
    """no stroking stream (flag without canvas, canvas without flag): the launches of a context without strokes; one
    stream with both: one more per tick"""
    T = torch()
    a = Context(max_width=W0, max_height=H0, max_frames=4)
    b = Context(max_width=W0, max_height=H0, max_frames=4)
    try:
        for x in (a, b):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        d = [T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda") for _ in range(2)]
        a.tracker_set_debug(2, d)
        b.tracker_set_debug(2, d[:1] + [T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")])
        b.tracker_set_debug_strokes(0, [1, 1, 0, 0])        # streams 0, 1: a flag but no canvas
        for t in range(40):
            if t == 10:
                b.tracker_set_debug_strokes(3, [1])
            if t == 25:
                b.tracker_set_debug_strokes(3, [0])
            la, lb = a.launch_count, b.launch_count
            ra, rb = run(a, 1, t, 4), run(b, 1, t, 4)
            assert equal_records(ra, rb)
            assert b.launch_count - lb == a.launch_count - la + (1 if 10 <= t < 25 else 0), t
    finally:
        a.close()
        b.close()


def set_raw(c, first, flags, n=None):
    arr = (C.c_int32 * max(1, len(flags)))(*flags)
    return c._L.ht_tracker_set_debug_strokes(c._h, first, len(flags) if n is None else n, arr)


def test_rejections_leave_the_settings_in_force():
    T = torch()
    mf = 3
    c = Context(max_width=W0, max_height=H0, max_frames=mf)
    try:
        assert set_raw(c, 0, [1]) == HT_ERR_STATE
        c.tracker_config()
        c.tracker_reset(0, mf)
        c.tracker_start(0, mf)
        d = [T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda") for _ in range(mf)]
        c.tracker_set_debug(0, d)
        c.tracker_set_debug_strokes(0, [1, 0, 1])
        for code, first, flags, n in [(HT_ERR_ARG, -1, [0], None), (HT_ERR_ARG, 0, [0], 0), (HT_ERR_ARG, 0, [0], -2),
                                      (HT_ERR_ARG, 2, [0, 0], None), (HT_ERR_ARG, 0, [0, 2, 0], None),
                                      (HT_ERR_ARG, 0, [0, 0, -1], None), (HT_ERR_ARG, 3, [0], None)]:
            assert set_raw(c, first, flags, n) == code, (first, flags, n)
        assert c._L.ht_tracker_set_debug_strokes(c._h, 0, 1, None) == HT_ERR_ARG
        T.cuda.synchronize()
        recs = run(c, 24, 0, mf)
        T.cuda.synchronize()
        assert [r["detection"] for r in recs] == ["CS"] * mf
        assert [stroked(x) for x in d] == [True, False, True]
    finally:
        c.close()
