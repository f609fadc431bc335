"""GPU: NV12 and I420 face crops (ht_tracker_set_face_crop_yuv, Context.tracker_set_face_crop with "format") against a
twin context with RGBA crops of the same sizes and scales: a YUV crop is, bit for bit, the conversion
(tests/crop_yuv_oracle.c) of the RGBA crop the same tick makes (DESIGN.md 2, "Face crops", item 5):

  * every case of reference_js_debug.json through step, feed, feed_yuv (NV12, P010, BGR24) and feed through views,
    NV12 and I420 crops across the four colours: records byte-identical to the twin's, every YUV crop the conversion
    of the twin's RGBA crop after every tick, every other byte of the sentinel buffer (row and plane padding, gaps,
    ticks that write no crop) untouched;
  * RGBA, NV12 and I420 crops of mixed sizes in one sentinel buffer, and a stream switching layout between ticks;
  * 1024 streams of 1280x720 NV12 with NV12 crops, a seeded sample checked;
  * the lifetime, the launch count (YUV crops launch what RGBA crops launch) and every rejection."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, make_frame
from test_face_crop_yuv_host import COLORS, SENTINEL, yo  # noqa: F401  (fixture: the C restatement)
from test_gpu_debug import black, carve, run
from test_gpu_feed import equal_records, to_device, video
from test_gpu_formats import api_frame, from_rgba
from test_gpu_views import unorient

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]


def torch():
    import torch as t
    return t


def host(t):
    return t.cpu().numpy()


class Crops:
    """face crops (fmt, Sw, Sh, scale, color) - NV12, I420 or RGBA - carved out of one sentinel buffer, with row
    padding (odd for YUV planes) and gaps between planes, and their RGBA twins (tight, zeroed) for a twin context"""

    def __init__(self, specs):
        T = torch()
        self.specs, self.layout, at = specs, [], 64
        for k, (fmt, Sw, Sh, _, _) in enumerate(specs):
            rows = {"nv12": [(Sh, Sw), (Sh // 2, Sw)], "i420": [(Sh, Sw), (Sh // 2, Sw // 2), (Sh // 2, Sw // 2)],
                    "rgba": [(Sh, 4 * Sw)]}[fmt]
            planes = []
            for p, (n, b) in enumerate(rows):
                if fmt == "rgba":
                    at, pitch = (at + 3) // 4 * 4, b + 4 * (k % 3)
                else:
                    pitch = b + (k + 3 * p) % 5                   # odd pitches and plane offsets among them
                planes.append((at, pitch, n, b))
                at += pitch * n + 1 + (k + p) % 7
            self.layout.append(planes)
        self.buf = T.full((at + 64,), SENTINEL, dtype=T.uint8, device="cuda")
        self.out = []
        for (fmt, Sw, Sh, _, _), pl in zip(specs, self.layout):
            if fmt == "rgba":
                self.out.append(carve(self.buf, pl[0][0], Sw, Sh, pl[0][1]))
            else:
                self.out.append(tuple(T.as_strided(self.buf, (n, b), (pitch, 1), off) for off, pitch, n, b in pl))
        self.rgba = [T.zeros((Sh, Sw, 4), dtype=T.uint8, device="cuda") for _, Sw, Sh, _, _ in specs]

    def crop(self, k):
        fmt, _, _, scale, color = self.specs[k]
        return {"out": self.out[k], "scale": scale} if fmt == "rgba" else \
            {"out": self.out[k], "format": fmt, "color": color, "scale": scale}

    def twin(self, k):
        return {"out": self.rgba[k], "scale": self.specs[k][3]}

    def expect(self, yo, exp, k, rgba):  # noqa: F811
        """exp (host copy of buf) with crop k set to what a tick makes of the RGBA crop `rgba` (numpy): the
        restatement's conversion, or rgba itself"""
        fmt, Sw, Sh, _, color = self.specs[k]
        rgba = np.ascontiguousarray(rgba)
        if fmt == "rgba":
            off, pitch = self.layout[k][0][:2]
            for r in range(Sh):
                exp[off + r * pitch:off + r * pitch + 4 * Sw] = rgba[r].reshape(-1)
            return
        pl = self.layout[k] + [(0, 0, 0, 0)] * (3 - len(self.layout[k]))
        base = exp.ctypes.data
        yo.hcyo_convert(_lib.YUV_COLORS[color], fmt == "nv12", rgba.ctypes.data, Sw, Sh, 4 * Sw, base + pl[0][0],
                        pl[0][1], base + pl[1][0], pl[1][1], base + pl[2][0] if fmt == "i420" else None, pl[2][1])


def wrote(rec):
    return rec["detection"] == "CS" and rec["width"] > 0 and rec["height"] > 0


SPECS = [("nv12", 112, 112, 1.0, "bt601"), ("i420", 64, 96, 1.5, "bt709"), ("nv12", 48, 48, 0.75, "bt601-full"),
         ("i420", 100, 60, 2.0, "bt709-full"), ("nv12", 34, 18, 1.0, "bt709"), ("i420", 2, 2, 1.0, "bt601")]


@pytest.mark.parametrize("path", ["step", "feed", "nv12", "p010", "bgr24", "views"])
def test_golden_replay_against_rgba_twin(yo, path):  # noqa: F811
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    cr = Crops([SPECS[k % len(SPECS)] for k in range(n)])
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(19)
    try:
        ts = TrackerSet(c, n, [dict(case["params"], faceCrop=cr.crop(k)) for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], faceCrop=cr.twin(k)) for k, case in enumerate(cases)])
        T.cuda.synchronize()
        exp = host(cr.buf).copy()
        clock, written = 1.0e12, 0
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
                ticked = dict(enumerate(ts.step(batch, clock)))
                assert equal_records(list(ticked.values()), tr.step(batch, clock)), i
            elif listed:
                vids, kw = {}, {}
                for k in listed:
                    v = video(frames[k], 1 + k % 3, False)
                    if path in ("feed", "views"):
                        vids[k] = to_device(unorient(v, (k + i) % 8 if path == "views" else 0))
                    else:
                        fmt, color = {"nv12": ("nv12", "bt709"), "p010": ("p010", "bt2020"), "bgr24": ("bgr24", "bt601")}[path]
                        vids[k] = api_frame(from_rgba(v, fmt, rng), True)
                        kw = dict(format=fmt, color=color)
                if path == "views":
                    kw = dict(view={k: {"rotate": 90 * (((k + i) % 8) & 3), "mirror": bool((k + i) % 8 & 4), "crop": None}
                                    for k in listed})
                T.cuda.synchronize()
                call = "feed" if path in ("feed", "views") else "feed_yuv"
                ticked = getattr(ts, call)(vids, clock, W0, H0, **kw)
                assert equal_records(list(ticked.values()), list(getattr(tr, call)(vids, clock, W0, H0, **kw).values())), i
            else:
                ticked = {}
            T.cuda.synchronize()
            for k, rec in ticked.items():
                if wrote(rec):
                    cr.expect(yo, exp, k, host(cr.rgba[k]))
                    written += 1
            assert np.array_equal(host(cr.buf), exp), i
        assert written > 40 and (host(cr.buf) == SENTINEL).any()
    finally:
        c.close()
        ref.close()


def test_mixed_layouts_in_one_buffer_and_a_layout_switch(yo):  # noqa: F811
    """NV12, I420 and RGBA crops of several sizes carved out of one sentinel buffer over mixed canvas sizes; stream 1
    switches between I420, RGBA and NV12 crops of one size and scale (carved out of a second buffer) every 10 ticks
    once it tracks, while its twin keeps one RGBA crop"""
    T = torch()
    import make_goldens_params as pg
    specs = SPECS + [("rgba", 40, 30, 1.0, None), ("rgba", 17, 9, 2.0, None)]
    n = len(specs)
    canv = [(160, 120), (200, 150), (120, 160)] * 3
    cr = Crops(specs)
    alt = Crops([SPECS[1], ("rgba",) + SPECS[1][1:], ("nv12",) + SPECS[1][1:]])
    ctx = Context(max_width=200, max_height=160, max_frames=n)
    ref = Context(max_width=200, max_height=160, max_frames=n)
    try:
        for x in (ctx, ref):
            x.tracker_config()
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
        ctx.tracker_set_face_crop(0, [alt.crop(0) if k == 1 else cr.crop(k) for k in range(n)])
        ref.tracker_set_face_crop(0, [cr.twin(k) for k in range(n)])
        T.cuda.synchronize()
        exp, exp_alt = host(cr.buf).copy(), host(alt.buf).copy()
        rng = np.random.default_rng(5)
        written, active = set(), 0
        for tick in range(55):
            if tick in (25, 35, 45):
                active = (active + 1) % 3
                ctx.tracker_set_face_crop(1, [alt.crop(active)])
            ks = [k for k in range(n) if rng.random() < 0.85] or [0]
            rng.shuffle(ks)
            vids = {k: video(pg.make_frame("face", tick, *canv[k]), 1 + k % 2, k == 2) for k in ks}
            frames = [to_device(vids[k]) if tick % 2 else vids[k] for k in ks]
            T.cuda.synchronize()
            cw, ch = [canv[k][0] for k in ks], [canv[k][1] for k in ks]
            recs = ctx.tracker_feed(ks, frames, 1.0e12 + 35.0 * tick, cw, ch)
            assert equal_records(recs, ref.tracker_feed(ks, frames, 1.0e12 + 35.0 * tick, cw, ch)), tick
            T.cuda.synchronize()
            for k, rec in zip(ks, recs):
                if wrote(rec):
                    written.add((k, active) if k == 1 else k)
                    if k == 1:
                        alt.expect(yo, exp_alt, active, host(cr.rgba[1]))
                    else:
                        cr.expect(yo, exp, k, host(cr.rgba[k]))
            assert np.array_equal(host(cr.buf), exp) and np.array_equal(host(alt.buf), exp_alt), tick
        assert written >= (set(range(n)) - {1}) | {(1, 0), (1, 1), (1, 2)}
    finally:
        ctx.close()
        ref.close()


def test_1024_streams_of_1280x720_nv12_with_nv12_crops(yo):  # noqa: F811
    T = torch()
    n, W, H, CW, CH, S = 1024, 1280, 720, 320, 240, 112
    rng = np.random.default_rng(37)
    bframes = [from_rgba(synth.frame(700 + i, W, H, n_faces=1), "nv12", rng) for i in range(8)]
    dframes = [api_frame(b, True) for b in bframes]
    y = T.full((n, S, S), SENTINEL, dtype=T.uint8, device="cuda")
    uv = T.full((n, S // 2, S), SENTINEL, dtype=T.uint8, device="cuda")
    twin = T.zeros((n, S, S, 4), dtype=T.uint8, device="cuda")
    ctx = Context(max_width=CW, max_height=CH, max_frames=n)
    ref = Context(max_width=CW, max_height=CH, max_frames=n)
    try:
        for x in (ctx, ref):
            x.tracker_config()
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
        ctx.tracker_set_face_crop(0, [{"out": (y[k], uv[k]), "format": "nv12", "color": COLORS[k % 4],
                                       "scale": 1.0 + (k % 3) * 0.25} for k in range(n)])
        ref.tracker_set_face_crop(0, [{"out": twin[k], "scale": 1.0 + (k % 3) * 0.25} for k in range(n)])
        T.cuda.synchronize()
        sample = sorted(int(k) for k in rng.choice(n, 48, replace=False))
        exp = {k: np.concatenate([host(y[k]).reshape(-1), host(uv[k]).reshape(-1)]) for k in sample}
        clock = [1.0e12 + 13.0 * k for k in range(n)]
        written = 0
        for tick in range(30):
            ks = [k for k in range(n) if rng.random() < 0.9]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            args = (ks, [dframes[k % 8] for k in ks], [clock[k] for k in ks], CW, CH)
            recs = ctx.tracker_feed_yuv(*args, format="nv12")
            assert equal_records(recs, ref.tracker_feed_yuv(*args, format="nv12")), tick
            T.cuda.synchronize()
            for k, rec in zip(ks, recs):
                if k in exp and wrote(rec):
                    rgba = np.ascontiguousarray(host(twin[k]))
                    e = exp[k]
                    yo.hcyo_convert(_lib.YUV_COLORS[COLORS[k % 4]], 1, rgba.ctypes.data, S, S, 4 * S, e.ctypes.data, S,
                                    e.ctypes.data + S * S, S, None, 0)
                    written += 1
            for k in sample:
                got = np.concatenate([host(y[k]).reshape(-1), host(uv[k]).reshape(-1)])
                assert np.array_equal(got, exp[k]), (tick, k)
        assert written > 300
    finally:
        ctx.close()
        ref.close()


# ---- lifetime, launches, rejections -----------------------------------------------------------------------------------

def test_lifetime():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        y = T.zeros((64, 64), dtype=T.uint8, device="cuda")
        u, v = T.zeros((32, 32), dtype=T.uint8, device="cuda"), T.zeros((32, 32), dtype=T.uint8, device="cuda")
        ctx.tracker_set_face_crop(0, [{"out": (y, u, v), "format": "i420", "color": "bt709", "scale": 1.2}])
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]

        def cut(t):
            """one CS tick on cleared planes; -> whether the crop was written"""
            for p in (y, u, v):
                p.zero_()
            T.cuda.synchronize()
            recs = run(ctx, 1, t)
            T.cuda.synchronize()
            assert recs[0]["detection"] == "CS" and recs[0]["width"] > 0
            return bool((y > 0).any() and (u > 0).any())

        assert cut(30)
        ctx.tracker_set_params(0, [dict(calcAngles=True)])
        assert cut(31)                                       # set_params keeps it
        snap = ctx.tracker_export([0])
        ctx.tracker_stop(0, 1)
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        ctx.tracker_import([0], snap)
        assert cut(32)                                       # stop / reset / start / import keep it
        ctx.tracker_set_face_crop(0, [None])                 # None removes it
        assert not cut(33)
        ctx.tracker_set_face_crop(0, [{"out": (y, u, v), "format": "i420", "color": "bt709"}])
        assert cut(34)
        ctx.tracker_config()                                 # removes every crop
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        run(ctx, 22, 40)
        assert not cut(62)
    finally:
        ctx.close()


def test_launch_count_equals_rgba_crops():
    """crops off: the launches of a context without crops; YUV crops: exactly those of RGBA crops"""
    T = torch()
    ctxs = [Context(max_width=W0, max_height=H0, max_frames=4) for _ in range(3)]
    try:
        for x in ctxs:
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        a, b, c = ctxs
        rgba = T.zeros((32, 32, 4), dtype=T.uint8, device="cuda")
        y, uv = T.zeros((32, 32), dtype=T.uint8, device="cuda"), T.zeros((16, 32), dtype=T.uint8, device="cuda")
        for t in range(40):
            if t == 10:
                b.tracker_set_face_crop(3, [{"out": rgba}])
                c.tracker_set_face_crop(2, [{"out": (y, uv), "format": "nv12"}])
            if t == 25:
                b.tracker_set_face_crop(3, [None])
                c.tracker_set_face_crop(2, [None])
            before = [x.launch_count for x in ctxs]
            recs = [run(x, 1, t, 4) for x in ctxs]
            assert equal_records(recs[0], recs[1]) and equal_records(recs[0], recs[2])
            d = [x.launch_count - n0 for x, n0 in zip(ctxs, before)]
            assert d[2] == d[1] == d[0] + (1 if 10 <= t < 25 else 0), t
    finally:
        for x in ctxs:
            x.close()


def set_raw(c, first, crops, n=None):
    arr = (_lib.FaceCropYuv * max(1, len(crops)))(*crops)
    return c._L.ht_tracker_set_face_crop_yuv(c._h, first, len(crops) if n is None else n, C.addressof(arr))


def yc(planes, w=20, h=20, fmt=0, color=0, pitch=(0, 0, 0), pad=0, scale=1.0):
    return _lib.FaceCropYuv((C.c_void_p * 3)(*planes), (C.c_int32 * 3)(*pitch), w, h, fmt, color, pad, scale)


def test_rejections_leave_the_settings_in_force():
    T = torch()
    mf = 3
    c = Context(max_width=W0, max_height=H0, max_frames=mf)
    try:
        buf = T.zeros((3, 8192), dtype=T.uint8, device="cuda")
        p = [buf[k].data_ptr() for k in range(3)]
        ok = [yc((p[k], p[k] + 1600, None), 40, 40) for k in range(3)]        # NV12 40 x 40: Y 1600, UV 800 bytes
        assert set_raw(c, 0, ok[:1]) == HT_ERR_STATE
        c.tracker_config()
        c.tracker_reset(0, mf)
        c.tracker_start(0, mf)
        assert set_raw(c, 0, ok) == 0
        hostbuf = (C.c_uint8 * 6400)()
        q = p[0]
        i420 = (q, q + 400, q + 500)
        bad = [(HT_ERR_ARG, -1, ok[:1], None), (HT_ERR_ARG, 0, ok[:1], 0), (HT_ERR_ARG, 2, ok[:2], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), fmt=16)], None),                     # NV21: not a crop format
               (HT_ERR_ARG, 0, [yc(i420, fmt=1, color=8)], None),                           # BT.2020
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), color=4)], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), color=-1)], None),
               (HT_ERR_SIZE, 0, [yc((q, q + 400, None), w=21)], None),                      # odd
               (HT_ERR_SIZE, 0, [yc((q, q + 400, None), h=19)], None),
               (HT_ERR_SIZE, 0, [yc((q, q + 400, None), w=0)], None),
               (HT_ERR_SIZE, 0, [yc((q, q + 400, None), h=2050)], None),
               (HT_ERR_ARG, 0, [yc((q, None, None))], None),                                # missing plane
               (HT_ERR_ARG, 0, [yc((q, q + 400, q + 600))], None),                          # extra plane
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), fmt=1)], None),                      # I420 missing V
               (HT_ERR_ARG, 0, [yc((C.addressof(hostbuf), q + 400, None))], None),          # host memory
               (HT_ERR_ARG, 0, [yc((q, C.addressof(hostbuf), None))], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), pitch=(19, 0, 0))], None),           # pitch below the row
               (HT_ERR_ARG, 0, [yc(i420, fmt=1, pitch=(0, 9, 0))], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), pitch=(-20, 0, 0))], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), pad=1)], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), scale=0.0)], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), scale=16.5)], None),
               (HT_ERR_ARG, 0, [yc((q, q + 400, None), scale=float("nan"))], None),
               (HT_ERR_ARG, 0, [yc((q, q + 399, None))], None),                             # UV overlaps its Y
               (HT_ERR_ARG, 0, [yc((q, q + 400, q + 499), fmt=1)], None),                   # V overlaps U
               (HT_ERR_ARG, 0, [ok[0], yc((p[0] + 2000, p[0] + 2400, None))], None),        # on stream 0's UV
               (HT_ERR_ARG, 1, [yc((p[2] + 64, p[2] + 2400, None))], None)]                  # on stream 2's Y
        for code, first, crops, n in bad:
            assert set_raw(c, first, crops, n) == code, (first, n, c.last_warning)
        assert c._L.ht_tracker_set_face_crop_yuv(c._h, 0, 1, None) == HT_ERR_ARG
        assert set_raw(c, 1, [yc((q + 8, p[1] + 4000, None))]) == HT_ERR_ARG                  # Y on stream 0's Y
        rgba = _lib.FaceCrop(p[1] + 4, 4, 4, 0, 0, 1.0)                                          # RGBA on stream 1's Y
        assert c._L.ht_tracker_set_face_crop(c._h, 2, 1, C.addressof((_lib.FaceCrop * 1)(rgba))) == HT_ERR_ARG
        d = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
        c.tracker_set_debug(0, [d])
        assert set_raw(c, 1, [yc((d.data_ptr() + 4096, p[1] + 4000, None))]) == HT_ERR_ARG     # on a debug canvas
        dc = (_lib.DebugCanvas * 1)(_lib.DebugCanvas(p[1] + 1700, 4, 4, 0, 0))
        assert c._L.ht_tracker_set_debug(c._h, 1, 1, C.addressof(dc)) == HT_ERR_ARG            # a canvas on a UV plane
        for kw in (dict(format="yuyv"), dict(color="bt2020")):
            with pytest.raises((ValueError, _lib.HtError)):
                c.tracker_set_face_crop(0, [dict(dict(out=(buf[0, :400].view(20, 20), buf[0, 400:600].view(10, 20)),
                                                      format="nv12"), **kw)])
        T.cuda.synchronize()
        run(c, 24, 0, mf)
        T.cuda.synchronize()
        assert all((buf[k][:1600] > 0).any() and (buf[k][1600:2400] > 0).any() for k in range(3))   # still in force
    finally:
        c.close()
