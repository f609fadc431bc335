"""GPU: the debug canvas of each headtrackr.Tracker stream (ht_tracker_set_debug, `params.debug`):

  * every case of the reference's own src/main.js runs with a debug canvas (reference_js_debug.json) through
    TrackerSet.step and TrackerSet.feed (k x k videos): after every tick the debug canvas hashes as the reference's,
    and debug_calls are the calls main.js made; records are byte-identical to a context without debug canvases;
  * one ht_tracker_feed_canvases call per tick over three canvas sizes with debug canvases that are smaller, larger,
    row-padded, carved out of one sentinel-filled buffer: only the clipped back-projection of CS entries is written;
  * 256 streams of 640x480 in random shuffled subsets: every CS entry's debug canvas is numpy's (here torch's fp64)
    floor(255 * min(m / c, 1)) of the stream's model and the drawn canvas's histogram, clipped; nothing else changes;
  * lifetime across ht_tracker_config / reset / stop / start / set_params, the launch count, and rejections."""
import ctypes as C
import hashlib
import sys
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, debug_canvas, make_frame, same_calls
from test_gpu_feed import equal_records, to_device, video

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
W0, H0 = GOLD_D["width"], GOLD_D["height"]


def torch():
    import torch as t
    return t


def sha_t(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def black(w, h):
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 3] = 255
    return f


def backproj(model, canvas):
    """getBackProjectionImg of a (h, w, 4) uint8 CUDA canvas under a 4096-bin model histogram, in fp64 on the device"""
    T = torch()
    c = canvas.to(T.int64)
    b = ((c[..., 0] >> 4) << 8) | ((c[..., 1] >> 4) << 4) | (c[..., 2] >> 4)
    cur = T.bincount(b.flatten(), minlength=4096).to(T.float64)
    m = T.as_tensor(model.astype(np.float64), device="cuda")
    p = T.where(cur == 0, T.zeros_like(cur), T.minimum(m / T.where(cur == 0, T.ones_like(cur), cur), T.ones_like(cur)))
    v = T.floor(255 * p).to(T.uint8)[b]
    return T.stack([v, v, v, T.full_like(v, 255)], dim=-1)


def put(dst, img):
    h, w = min(img.shape[0], dst.shape[0]), min(img.shape[1], dst.shape[1])
    dst[:h, :w] = img[:h, :w]


# ---- the reference's runs -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("path", ["step", "feed"])
def test_golden_replay(path):
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    try:
        dbg = [T.from_numpy(debug_canvas(case)).cuda() for case in cases]
        ts = TrackerSet(c, n, [dict(case["params"], debug=dbg[k]) for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [case["params"] for case in cases])
        T.cuda.synchronize()
        clock = 1.0e12
        puts = 0
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
                assert equal_records(ts.step(batch, clock), tr.step(batch, clock)), i
            elif listed:
                vids = {k: to_device(video(frames[k], 1 + k % 3, k == 1)) for k in listed}
                T.cuda.synchronize()
                assert equal_records(ts.feed(vids, clock, W0, H0), tr.feed(vids, clock, W0, H0)), i
            for k, case in enumerate(cases):
                if i >= len(case["steps"]):
                    continue
                want = case["steps"][i]
                if path == "step" or k in listed:
                    # the device sums camshift's moments in another order: angles agree to 1e-9 relative, as in
                    # every GPU tracker test; positions and sizes exactly
                    assert same_calls(ts.debug_calls(k), want["calls"], 1e-9), (case["name"], i, ts.debug_calls(k))
                assert sha_t(dbg[k]) == want["debug_sha256"], (case["name"], i)
                puts += want["put"]
        assert puts == sum(s["put"] for case in cases for s in case["steps"]) > 0
    finally:
        c.close()
        ref.close()


# ---- mixed canvases -------------------------------------------------------------------------------------------------

def carve(buf, off, dw, dh, pitch):
    T = torch()
    return T.as_strided(buf, (dh, dw, 4), (pitch, 4, 1), off)


def test_mixed_canvases_write_only_the_clipped_image_of_cs_entries():
    """one ht_tracker_feed_canvases call per tick: 160x120, 200x150 and 120x160 canvases; debug canvases smaller,
    larger, narrower and taller, row-padded with a pitch that rules out 16-byte stores, all carved out of one buffer
    of sentinel bytes with gaps; streams 3 and 4 have none"""
    T = torch()
    import make_goldens_params as pg
    canv = [(160, 120), (200, 150), (120, 160), (160, 120), (200, 150), (120, 160)]
    # (debug w, h, pitch) or None
    spec = [(100, 80, 400), (240, 180, 960), (120, 160, 4 * 120 + 36), None, None, (64, 200, 4 * 64 + 4)]
    offs, off = [], 64
    for s in spec:
        offs.append(off)
        if s:
            off += s[2] * s[1] + 64
    buf = T.full((off + 64,), 0x5A, dtype=T.uint8, device="cuda")
    exp = buf.clone()
    views = [carve(buf, o, *s) if s else None for o, s in zip(offs, spec)]
    ctx = Context(max_width=200, max_height=160, max_frames=8)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 6)
        ctx.tracker_start(0, 6)
        ctx.tracker_set_debug(0, views)
        T.cuda.synchronize()
        rng = np.random.default_rng(5)
        written = set()
        for tick in range(40):
            ks = [k for k in range(6) if rng.random() < 0.85] or [0]
            rng.shuffle(ks)
            frames = {k: pg.make_frame("face", tick, *canv[k]) for k in ks}
            vids = [to_device(video(frames[k], 1 + k % 2, k == 2)) for k in ks]
            T.cuda.synchronize()
            recs = ctx.tracker_feed(ks, vids, 1.0e12 + 35.0 * tick, [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            for k, rec in zip(ks, recs):
                if rec["detection"] == "CS" and spec[k]:
                    img = backproj(ctx.debug_model_hist(k), T.from_numpy(frames[k]).cuda())
                    put(carve(exp, offs[k], *spec[k]), img)
                    written.add(k)
            assert T.equal(buf, exp), tick
        assert written == {0, 1, 2, 5}
        assert (buf == 0x5A).any()          # the sentinel bytes between, and past the clipped rows
    finally:
        ctx.close()


# ---- scale ----------------------------------------------------------------------------------------------------------

def test_256_streams_640x480_random_subsets():
    T = torch()
    n, W, H = 256, 640, 480
    rng = np.random.default_rng(23)
    frames = [T.from_numpy(synth.frame(800 + i, W, H, n_faces=1)).cuda() for i in range(16)]
    sizes = [(640, 480), (320, 200), (700, 500), (641, 13), (97, 480), (1000, 3)]
    dbg = [None] * n
    for k in rng.permutation(n)[: n // 2]:
        dw, dh = sizes[int(rng.integers(len(sizes)))]
        dbg[k] = T.full((dh, dw, 4), int(k) & 0xff, dtype=T.uint8, device="cuda")
    exp = [d.clone() if d is not None else None for d in dbg]
    ctx = Context(max_width=W, max_height=H, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        ctx.tracker_set_debug(0, dbg)
        T.cuda.synchronize()
        clock = [1.0e12 + 17.0 * k for k in range(n)]
        checked = 0
        for tick in range(30):
            ks = [k for k in range(n) if rng.random() < 0.85]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            recs = ctx.tracker_feed(ks, [frames[k % 16] for k in ks], [clock[k] for k in ks], W, H)
            for k, rec in zip(ks, recs):
                if rec["detection"] == "CS" and dbg[k] is not None:
                    put(exp[k], backproj(ctx.debug_model_hist(k), frames[k % 16]))
                    checked += 1
            for k in range(n):
                if dbg[k] is not None:
                    assert T.equal(dbg[k], exp[k]), (tick, k)
        assert checked > 200
    finally:
        ctx.close()


# ---- lifetime, launches, rejections ---------------------------------------------------------------------------------

def run(ctx, ticks, t0, n=2):
    """ticks of streams [0, n) on face frames; -> records of the last tick"""
    import make_goldens_params as pg
    recs = None
    for t in range(t0, t0 + ticks):
        recs = ctx.tracker_feed(list(range(n)), [pg.make_frame("face", t, W0, H0)] * n, 1.0e12 + 35.0 * t, W0, H0)
    return recs


def test_lifetime():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        d = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
        ctx.tracker_set_debug(0, [d])
        T.cuda.synchronize()
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]
        assert d.any()

        def cleared_then_written(op, written):
            d.fill_(7)
            T.cuda.synchronize()
            op()
            assert (d == 7).all()                    # the call itself writes nothing
            recs = run(ctx, 1, 30)
            assert recs[0]["detection"] == "CS"
            assert bool((d != 7).any()) == written, op

        cleared_then_written(lambda: ctx.tracker_set_params(0, [dict(calcAngles=True)]), True)
        cleared_then_written(lambda: ctx.tracker_config(), False)          # discards every debug canvas
        ctx.tracker_set_debug(0, [d])
        cleared_then_written(lambda: None, True)
        d.fill_(9)
        T.cuda.synchronize()
        ctx.tracker_stop(0, 1)
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        run(ctx, 15, 40)                                                    # starter, whitebalance, VJ: no writes
        assert (d == 9).all()
        assert run(ctx, 8, 60)[0]["detection"] == "CS" and (d != 9).any()  # the canvas survived stop / reset / start
        ts_ctx = Context(max_width=W0, max_height=H0, max_frames=2)
        try:
            e = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
            ts = TrackerSet(ts_ctx, 2, [dict(debug=e), {}])
            ts.start()
            import make_goldens_params as pg
            for t in range(22):
                ts.feed({0: pg.make_frame("face", t, W0, H0), 1: pg.make_frame("face", t, W0, H0)}, 1.0e12 + 35.0 * t,
                        W0, H0)
            assert ts.current[0]["detection"] == "CS" and e.any()
            ts.set_params(0, {"calcAngles": True})                         # no "debug" key: none
            e.fill_(3)
            T.cuda.synchronize()
            for t in range(22, 26):
                ts.feed({0: pg.make_frame("face", t, W0, H0)}, 1.0e12 + 35.0 * t, W0, H0)
            assert ts.current[0]["detection"] == "CS" and (e == 3).all()
        finally:
            ts_ctx.close()
    finally:
        ctx.close()


def test_launch_count_unchanged_without_debug_canvases():
    T = torch()
    a = Context(max_width=W0, max_height=H0, max_frames=4)
    b = Context(max_width=W0, max_height=H0, max_frames=4)
    try:
        for x in (a, b):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        d = [T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda") for _ in range(2)]
        for t in range(40):
            if t == 10:
                b.tracker_set_debug(1, d)
            if t == 25:
                b.tracker_set_debug(1, [None, None])
            la, lb = a.launch_count, b.launch_count
            ra, rb = run(a, 1, t, 4), run(b, 1, t, 4)
            assert equal_records(ra, rb)
            extra = 2 if 10 <= t < 25 else 0                               # k_debug_table + k_debug_backproj
            assert b.launch_count - lb == a.launch_count - la + extra, t
        assert all(x.any() for x in d)
    finally:
        a.close()
        b.close()


def set_debug_raw(c, first, recs):
    arr = (_lib.DebugCanvas * max(1, len(recs)))(*recs)
    return c._L.ht_tracker_set_debug(c._h, first, len(recs), C.addressof(arr))


def test_rejections_leave_the_settings_in_force():
    T = torch()
    mf = 3
    c = Context(max_width=W0, max_height=H0, max_frames=mf)
    buf = T.full((4 * W0 * H0 * 4,), 0x11, dtype=T.uint8, device="cuda")
    base = buf.data_ptr()
    D = _lib.DebugCanvas
    try:
        assert set_debug_raw(c, 0, [D(base, W0, H0, 0, 0)]) == HT_ERR_STATE
        c.tracker_config()
        c.tracker_reset(0, mf)
        c.tracker_start(0, mf)
        a = carve(buf, 0, W0, H0, 4 * W0)
        b = carve(buf, 2 * W0 * H0 * 4, W0, H0, 4 * W0)
        c.tracker_set_debug(0, [a, None, b])
        host = np.zeros(W0 * H0 * 4, np.uint8)
        far = base + 4 * W0 * H0 * 4 - 64 * 4
        cases = [
            (HT_ERR_ARG, -1, [D(far, 4, 4, 0, 0)]),
            (HT_ERR_ARG, 0, []),
            (HT_ERR_ARG, 2, [D(far, 4, 4, 0, 0), D(far, 4, 4, 0, 0)]),          # past max_frames
            (HT_ERR_ARG, 1, [D(host.ctypes.data, 4, 4, 0, 0)]),                 # host memory
            (HT_ERR_ARG, 1, [D(far + 2, 4, 4, 0, 0)]),                          # not a multiple of 4
            (HT_ERR_ARG, 1, [D(far, 4, 4, 18, 0)]),                             # pitch not a multiple of 4
            (HT_ERR_ARG, 1, [D(far, 4, 4, 12, 0)]),                             # pitch below 4 * width
            (HT_ERR_ARG, 1, [D(base + 4 * W0 * (H0 - 1), 4, 4, 0, 0)]),          # overlaps stream 0's last row
            (HT_ERR_ARG, 0, [D(far, 4, 4, 0, 0), D(far + 32, 4, 1, 0, 0)]),     # two records share bytes
            (HT_ERR_ARG, 2, [D(base + 4 * W0 * H0 - 4, 2, 1, 0, 0)]),           # overlaps stream 0's canvas
            (HT_ERR_SIZE, 1, [D(far, 0, 4, 0, 0)]),
            (HT_ERR_SIZE, 1, [D(far, 4, 0, 0, 0)]),
            (HT_ERR_SIZE, 1, [D(far, 16385, 1, 0, 0)]),
        ]
        for i, (code, first, recs) in enumerate(cases):
            rc = set_debug_raw(c, first, recs)
            assert rc == code, (i, rc, c._L.ht_last_error(c._h))
        assert c._L.ht_tracker_set_debug(c._h, 0, 1, None) == HT_ERR_ARG
        # stream 1 may take the gap between the two canvases; and a canvas may replace its own stream's
        assert set_debug_raw(c, 1, [D(base + W0 * H0 * 4, W0, H0, 0, 0)]) == 0
        assert set_debug_raw(c, 1, [D(None, 0, 0, 0, 0)]) == 0
        T.cuda.synchronize()
        run(c, 24, 0, mf)
        # streams 0 and 2 still write their canvases, stream 1 and the gap are untouched
        assert a.ne(0x11).any() and b.ne(0x11).any()
        assert (buf[W0 * H0 * 4: 2 * W0 * H0 * 4] == 0x11).all() and (buf[3 * W0 * H0 * 4:] == 0x11).all()
    finally:
        c.close()
