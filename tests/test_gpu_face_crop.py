"""GPU: face crops cut by k_face_crop (ht_tracker_set_face_crop, TrackerSet's "faceCrop"), against the C restatement
tests/crop_oracle.c applied to the device's own records and the tick's video (the crop is a function of the record and
the video; the device's angle may differ from the oracle's in its last bits):

  * every case of reference_js_debug.json through step, feed, feed_yuv (NV12, P010, BGR24) and feed through views,
    with crops on, against a crops-off twin: records byte-identical; after every tick each crop is the restatement's
    crop of the tick's record and video, or unchanged on a tick that writes none;
  * host and device videos, mixed canvas sizes and mixed crop sizes carved out of one sentinel buffer: no byte outside
    the crops changes;
  * 1024 streams of 1280x720 NV12 onto 320x240 canvases with 112x112 crops, a seeded sample checked;
  * the crop's lifetime, the launch count, and every rejection of ht_tracker_set_face_crop."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, debug_canvas, make_frame
from test_face_crop_host import event, oracle_crop, so  # noqa: F401  (fixture: the C restatement)
from test_formats_host import fo, oracle_convert  # noqa: F401
from test_gpu_debug import black, carve, run
from test_gpu_feed import equal_records, to_device, video
from test_gpu_formats import api_frame, from_rgba
from test_gpu_views import unorient

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]
SENTINEL = 0x5A
DET = {"VJ": 1, "CS": 2}


def torch():
    import torch as t
    return t


def host(t):
    return t.cpu().numpy()


def expect(so, prev, rec, cw, ch, rgba, o=0, rect=(0, 0, 0, 0), scale=1.0):  # noqa: F811
    """the crop after a tick: the restatement's crop of the tick's record and RGBA8 video (as stored, seen through
    orientation o and rect), or `prev` on a tick that writes none"""
    Sh, Sw = prev.shape[:2]
    e = event(DET.get(rec["detection"], 0), rec["x"], rec["y"], rec["width"], rec["height"], rec["angle"])
    rc, buf, pitch = oracle_crop(so, e, cw, ch, np.ascontiguousarray(rgba), o, rect, Sw, Sh, scale)
    if not rc:
        return prev, False
    return buf.reshape(Sh, pitch)[:, :4 * Sw].reshape(Sh, Sw, 4).copy(), True


CROPS = [(112, 112, 1.0), (64, 96, 1.5), (48, 48, 0.75), (100, 60, 2.0), (33, 17, 1.0)]


def carve_crops(T, specs, extra_pad=(0, 8, 0, 4, 12)):
    """crops (Sw, Sh, pitch) carved out of one buffer of sentinel bytes with gaps -> (buffer, views, offsets)"""
    offs, off = [], 64
    for (Sw, Sh, _), pad in zip(specs, extra_pad):
        offs.append((off, 4 * Sw + pad))
        off += (4 * Sw + pad) * Sh + 64
    buf = T.full((off + 64,), SENTINEL, dtype=T.uint8, device="cuda")
    return buf, [carve(buf, o, s[0], s[1], p) for (o, p), s in zip(offs, specs)], offs


@pytest.mark.parametrize("path", ["step", "feed", "nv12", "p010", "bgr24", "views"])
def test_golden_replay(so, fo, path):  # noqa: F811
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    specs = [CROPS[k % len(CROPS)] for k in range(n)]
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(17)
    try:
        buf, crops, offs = carve_crops(T, specs)
        dbg = [T.from_numpy(debug_canvas(case)).cuda() for case in cases]
        twin = [d.clone() for d in dbg]
        ts = TrackerSet(c, n, [dict(case["params"], debug=dbg[k], faceCrop={"out": crops[k], "scale": specs[k][2]})
                               for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], debug=twin[k]) for k, case in enumerate(cases)])
        T.cuda.synchronize()
        exp_buf = host(buf).copy()
        exp = [np.lib.stride_tricks.as_strided(exp_buf[o:], (s[1], s[0], 4), (p, 4, 1)) for (o, p), s in zip(offs, specs)]
        clock, written, turned = 1.0e12, 0, 0
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
            seen = {}                                        # stream -> (RGBA8 video as stored, orientation, canvas)
            if path == "step":
                batch = T.from_numpy(np.stack(frames)).cuda()
                T.cuda.synchronize()
                ticked = dict(enumerate(ts.step(batch, clock)))
                assert equal_records(list(ticked.values()), tr.step(batch, clock)), i
                seen = {k: (frames[k], 0) for k in ticked}
            elif listed:
                vids, rgba, kw = {}, {}, {}
                for k in listed:
                    v = video(frames[k], 1 + k % 3, False)
                    if path in ("feed", "views"):
                        o = (k + i) % 8 if path == "views" else 0
                        stored = unorient(v, o)
                        vids[k], rgba[k] = to_device(stored), (stored, o)
                    else:
                        fmt, color = {"nv12": ("nv12", "bt709"), "p010": ("p010", "bt2020"), "bgr24": ("bgr24", "bt601")}[path]
                        bf = from_rgba(v, fmt, rng)
                        vids[k], rgba[k] = api_frame(bf, True), (oracle_convert(fo, bf, color), 0)
                        kw = dict(format=fmt, color=color)
                if path == "views":
                    kw = dict(view={k: {"rotate": 90 * (rgba[k][1] & 3), "mirror": bool(rgba[k][1] & 4), "crop": None}
                                    for k in listed})
                T.cuda.synchronize()
                call = "feed" if path in ("feed", "views") else "feed_yuv"
                ticked = getattr(ts, call)(vids, clock, W0, H0, **kw)
                assert equal_records(list(ticked.values()), list(getattr(tr, call)(vids, clock, W0, H0, **kw).values())), i
                seen = rgba
            else:
                ticked = {}
            for k, rec in ticked.items():
                stored, o = seen[k]
                new, wrote = expect(so, exp[k].copy(), rec, W0, H0, stored, o, scale=specs[k][2])
                exp[k][...] = new
                written += wrote
                turned += wrote and o != 0
            assert np.array_equal(host(buf), exp_buf), i
        assert written > 40 and (path != "views" or turned > 20)
        assert (host(buf) == SENTINEL).any()
    finally:
        c.close()
        ref.close()


def test_mixed_canvases_crops_and_memory_write_only_the_crops(so):  # noqa: F811
    """one ht_tracker_feed_canvases call per tick over three canvas sizes, host and device videos in turn, crops of
    five sizes carved out of one sentinel buffer; streams 5 and 6 have no crop"""
    T = torch()
    import make_goldens_params as pg
    canv = [(160, 120), (200, 150), (120, 160), (160, 120), (200, 150), (120, 160), (160, 120)]
    ctx = Context(max_width=200, max_height=160, max_frames=8)
    try:
        buf, crops, offs = carve_crops(T, CROPS)
        ctx.tracker_config()
        ctx.tracker_reset(0, 7)
        ctx.tracker_start(0, 7)
        with pytest.raises(_lib.HtError):                    # a crop may not share bytes with a debug canvas
            ctx.tracker_set_face_crop(0, [{"out": crops[0]}])
            ctx.tracker_set_debug(0, [carve(buf, offs[0][0], 16, 16, 64)])
        ctx.tracker_set_face_crop(0, [{"out": v, "scale": s[2]} for v, s in zip(crops, CROPS)])
        T.cuda.synchronize()
        exp_buf = host(buf).copy()
        exp = [np.lib.stride_tricks.as_strided(exp_buf[o:], (s[1], s[0], 4), (p, 4, 1)) for (o, p), s in zip(offs, CROPS)]
        rng = np.random.default_rng(5)
        written = set()
        for tick in range(40):
            ks = [k for k in range(7) if rng.random() < 0.85] or [0]
            rng.shuffle(ks)
            vids = {k: video(pg.make_frame("face", tick, *canv[k]), 1 + k % 2, k == 2) for k in ks}
            frames = [to_device(vids[k]) if tick % 2 else vids[k] for k in ks]
            T.cuda.synchronize()
            recs = ctx.tracker_feed(ks, frames, 1.0e12 + 35.0 * tick, [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            for k, rec in zip(ks, recs):
                if k < 5:
                    new, wrote = expect(so, exp[k].copy(), rec, *canv[k], vids[k], scale=CROPS[k][2])
                    exp[k][...] = new
                    if wrote:
                        written.add(k)
            assert np.array_equal(host(buf), exp_buf), tick
        assert written == {0, 1, 2, 3, 4}
    finally:
        ctx.close()


def test_1024_streams_of_1280x720_nv12_with_112x112_crops(so, fo):  # noqa: F811
    T = torch()
    n, W, H, CW, CH = 1024, 1280, 720, 320, 240
    rng = np.random.default_rng(31)
    bframes = [from_rgba(synth.frame(700 + i, W, H, n_faces=1), "nv12", rng) for i in range(8)]
    dframes = [api_frame(b, True) for b in bframes]
    rgba = [oracle_convert(fo, b, "bt601") for b in bframes]
    out = T.full((n, 112, 112, 4), SENTINEL, dtype=T.uint8, device="cuda")
    ctx = Context(max_width=CW, max_height=CH, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        ctx.tracker_set_face_crop(0, [{"out": out[k], "scale": 1.0 + (k % 3) * 0.25} for k in range(n)])
        T.cuda.synchronize()
        sample = [int(k) for k in rng.choice(n, 48, replace=False)]
        exp = {k: host(out[k]).copy() for k in sample}
        clock = [1.0e12 + 13.0 * k for k in range(n)]
        written = 0
        for tick in range(30):
            ks = [k for k in range(n) if rng.random() < 0.9]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            recs = ctx.tracker_feed_yuv(ks, [dframes[k % 8] for k in ks], [clock[k] for k in ks], CW, CH, format="nv12")
            for k, rec in zip(ks, recs):
                if k in exp:
                    exp[k], wrote = expect(so, exp[k], rec, CW, CH, rgba[k % 8], scale=1.0 + (k % 3) * 0.25)
                    written += wrote
            for k in sample:
                assert np.array_equal(host(out[k]), exp[k]), (tick, k)
        assert written > 300
    finally:
        ctx.close()


# ---- lifetime, launches, rejections -----------------------------------------------------------------------------------

def test_lifetime():
    T = torch()
    import make_goldens_params as pg
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        out = T.zeros((64, 64, 4), dtype=T.uint8, device="cuda")
        ctx.tracker_set_face_crop(0, [{"out": out, "scale": 1.2}])
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]

        def cut(t):
            """one CS tick on a cleared crop; -> whether the crop was written"""
            out.zero_()
            T.cuda.synchronize()
            recs = run(ctx, 1, t)
            T.cuda.synchronize()
            assert recs[0]["detection"] == "CS" and recs[0]["width"] > 0
            return bool((out[..., 3] > 0).any())

        assert cut(30)
        ctx.tracker_set_params(0, [dict(calcAngles=True)])
        assert cut(31)                                       # set_params keeps it
        snap = ctx.tracker_export([0])
        ctx.tracker_stop(0, 1)
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        ctx.tracker_import([0], snap)
        assert cut(32)                                       # stop / reset / start / import keep it
        ctx.tracker_config()                                 # removes every crop
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        run(ctx, 22, 40)
        assert not cut(62)
        ts_ctx = Context(max_width=W0, max_height=H0, max_frames=2)
        try:
            e = T.zeros((48, 48, 4), dtype=T.uint8, device="cuda")
            ts = TrackerSet(ts_ctx, 2, [dict(faceCrop={"out": e}), {}])
            ts.start()
            for t in range(22):
                ts.feed({0: pg.make_frame("face", t, W0, H0)}, 1.0e12 + 35.0 * t, W0, H0)
            T.cuda.synchronize()
            assert ts.current[0]["detection"] == "CS" and (e[..., 3] > 0).any()
            ts.set_params(0, {})                             # no "faceCrop" key: none
            e.zero_()
            T.cuda.synchronize()
            ts.feed({0: pg.make_frame("face", 22, W0, H0)}, 1.0e12 + 35.0 * 22, W0, H0)
            T.cuda.synchronize()
            assert ts.current[0]["detection"] == "CS" and not (e != 0).any()
        finally:
            ts_ctx.close()
    finally:
        ctx.close()


def test_launch_count():
    """without crops: the launches of a context without them; with a crop on some stream: one more per tick"""
    T = torch()
    a = Context(max_width=W0, max_height=H0, max_frames=4)
    b = Context(max_width=W0, max_height=H0, max_frames=4)
    try:
        for x in (a, b):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        out = T.zeros((32, 32, 4), dtype=T.uint8, device="cuda")
        for t in range(40):
            if t == 10:
                b.tracker_set_face_crop(3, [{"out": out}])
            if t == 25:
                b.tracker_set_face_crop(3, [None])
            la, lb = a.launch_count, b.launch_count
            ra, rb = run(a, 1, t, 4), run(b, 1, t, 4)
            assert equal_records(ra, rb)
            assert b.launch_count - lb == a.launch_count - la + (1 if 10 <= t < 25 else 0), t
    finally:
        a.close()
        b.close()


def set_raw(c, first, crops, n=None):
    arr = (_lib.FaceCrop * max(1, len(crops)))(*crops)
    return c._L.ht_tracker_set_face_crop(c._h, first, len(crops) if n is None else n, C.addressof(arr))


def test_rejections_leave_the_settings_in_force():
    T = torch()
    mf = 3
    c = Context(max_width=W0, max_height=H0, max_frames=mf)
    try:
        buf = T.zeros((3, 40, 40, 4), dtype=T.uint8, device="cuda")
        p = [buf[k].data_ptr() for k in range(3)]
        ok = [_lib.FaceCrop(p[k], 40, 40, 0, 0, 1.0) for k in range(3)]
        assert set_raw(c, 0, ok[:1]) == HT_ERR_STATE
        c.tracker_config()
        c.tracker_reset(0, mf)
        c.tracker_start(0, mf)
        assert set_raw(c, 0, ok) == 0
        hostbuf = (C.c_uint8 * 6400)()
        fc = _lib.FaceCrop
        bad = [(HT_ERR_ARG, -1, ok[:1], None), (HT_ERR_ARG, 0, ok[:1], 0), (HT_ERR_ARG, 2, ok[:2], None),
               (HT_ERR_ARG, 3, ok[:1], None),
               (HT_ERR_ARG, 0, [fc(C.addressof(hostbuf), 40, 40, 0, 0, 1.0)], None),       # host memory
               (HT_ERR_ARG, 0, [fc(p[0] + 2, 20, 20, 0, 0, 1.0)], None),                     # misaligned
               (HT_ERR_ARG, 0, [fc(p[0], 20, 20, 82, 0, 1.0)], None),                        # pitch not a multiple of 4
               (HT_ERR_ARG, 0, [fc(p[0], 20, 20, 76, 0, 1.0)], None),                        # pitch below 4 * width
               (HT_ERR_ARG, 0, [fc(p[0], 20, 20, 0, 0, 0.0)], None),
               (HT_ERR_ARG, 0, [fc(p[0], 20, 20, 0, 0, 16.5)], None),
               (HT_ERR_ARG, 0, [fc(p[0], 20, 20, 0, 0, float("nan"))], None),
               (HT_ERR_SIZE, 0, [fc(p[0], 0, 20, 0, 0, 1.0)], None),
               (HT_ERR_SIZE, 0, [fc(p[0], 20, 2049, 0, 0, 1.0)], None),
               (HT_ERR_ARG, 0, [ok[0], fc(p[0] + 4 * 40 * 39, 40, 2, 0, 0, 1.0)], None),      # overlaps stream 0's
               (HT_ERR_ARG, 1, [fc(p[2] + 64, 10, 10, 0, 0, 1.0)], None)]                     # overlaps stream 2's
        for code, first, crops, n in bad:
            assert set_raw(c, first, crops, n) == code, (first, n, c.last_warning)
        assert c._L.ht_tracker_set_face_crop(c._h, 0, 1, None) == HT_ERR_ARG
        d = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
        c.tracker_set_debug(0, [d])
        assert set_raw(c, 1, [fc(d.data_ptr() + 4096, 10, 10, 0, 0, 1.0)]) == HT_ERR_ARG    # overlaps a debug canvas
        dc = (_lib.DebugCanvas * 1)(_lib.DebugCanvas(p[1] + 400, 4, 4, 0, 0))
        assert c._L.ht_tracker_set_debug(c._h, 1, 1, C.addressof(dc)) == HT_ERR_ARG            # a canvas on a crop
        T.cuda.synchronize()
        run(c, 24, 0, mf)
        T.cuda.synchronize()
        assert all((buf[k][..., 3] > 0).any() for k in range(3))   # every crop is still in force
    finally:
        c.close()
