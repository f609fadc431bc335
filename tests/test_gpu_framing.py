"""GPU: framing (ht_tracker_set_framing, Context.tracker_set_framing, TrackerSet's "framing" key; DESIGN.md 2, "Face
crops", item 7): a stream's steady face-cam box, moved on the device on every crop tick, and the outputs cut from it:

  * every case of reference_js_debug.json through step, feed, feed_yuv (NV12, P010, BGR24) and feed through views,
    each stream with an RGBA crop and a u8 HWC tensor of the same size and scale, against a twin without framing:
    records byte-identical, every unframed output equal to the twin's (streams that frame only the crop keep a
    tracked tensor), every box after every tick framing.py's replay byte for byte, every framed output the host
    build's crop from that box;
  * 1024 streams on two canvas sizes with mixed crop sizes, a seeded sample checked;
  * the lifetime: lost and refound inside and outside the box, stop / start / reset, import into a framed id, a
    canvas-size change, removal by tracker_config; the launch count; the overlap rule both ways; every rejection."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, framing, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, make_frame
from test_formats_host import fo, oracle_convert  # noqa: F401  (fixture: the format restatement)
from test_gpu_debug import black, run
from test_gpu_feed import equal_records, to_device, video
from test_gpu_formats import api_frame, from_rgba
from test_gpu_views import unorient
from test_views_host import view_of

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]
SIZES = [(112, 112, 1.0), (64, 96, 1.5), (48, 48, 0.75), (100, 60, 2.0), (34, 18, 1.0), (1, 1, 1.0)]


def torch():
    import torch as t
    return t


def host(t):
    return t.cpu().numpy()


def st_lib():
    """the host-only build of ht_api.cu (test_cascade_host's fixture, built once here)"""
    import subprocess
    import tempfile
    from pathlib import Path
    from test_cascade_host import CSRC
    global _ST
    try:
        return _ST
    except NameError:
        pass
    so = Path(tempfile.mkdtemp()) / "libht_selftest.so"
    subprocess.check_call([_lib.nvcc(), "-DHT_HOST_SELFTEST", "-gencode", "arch=compute_90a,code=sm_90a", "-O2",
                           "-std=c++17", "-fmad=false", "-Xcompiler", "-fPIC", "-shared", "-o", str(so),
                           str(CSRC / "ht_api.cu")], stderr=subprocess.DEVNULL)
    L = C.CDLL(str(so))
    L.ht_selftest_face_crop_framed_rgba.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    _ST = L
    return L


def host_crop(box, cw, ch, rgba, Sw, Sh, scale, o=0):
    """the host build's RGBA crop cut from box (a dict) out of an RGBA8 video (h, w, 4) through orientation o"""
    rgba = np.ascontiguousarray(rgba)
    h, w = rgba.shape[:2]
    f = _lib.VideoFrame(rgba.ctypes.data, 0, w, h, 4 * w, 0.0)
    out = np.zeros((Sh, Sw, 4), np.uint8)
    crop = _lib.FaceCrop(out.ctypes.data, Sw, Sh, 4 * Sw, 0, scale)
    b, v = framing.box_struct(box), view_of(o)
    rc = st_lib().ht_selftest_face_crop_framed_rgba(C.addressof(b), cw, ch, C.addressof(f), C.addressof(v),
                                                    C.addressof(crop))
    assert rc == 1
    return out


def wrote(rec):
    return rec["detection"] == "CS" and rec["width"] > 0 and rec["height"] > 0


class Outputs:
    """per stream an RGBA crop, a u8 HWC RGB tensor of the same size and scale, and a framed box"""

    def __init__(self, n, sizes=SIZES):
        T = torch()
        self.spec = [sizes[k % len(sizes)] for k in range(n)]
        self.crop = [T.zeros((Sh, Sw, 4), dtype=T.uint8, device="cuda") for Sw, Sh, _ in self.spec]
        self.tensor = [T.zeros((Sh, Sw, 3), dtype=T.uint8, device="cuda") for Sw, Sh, _ in self.spec]
        self.box = T.zeros((n, 64), dtype=T.uint8, device="cuda")       # 48 bytes each, 64 apart

    def params(self, k, frame=True, tensor=None):
        Sw, Sh, scale = self.spec[k]
        p = {"faceCrop": {"out": self.crop[k], "scale": scale},
             "faceTensor": {"out": self.tensor[k], "layout": "hwc", "channels": "rgb", "scale": scale}}
        if frame:
            p["framing"] = {"out": self.box[k, :48], "alpha": 0.25, "dead_zone": 0.1, "crop": True,
                            "tensor": (k % 2 == 0) if tensor is None else tensor}
        return p

    def boxes(self):
        return [framing.box_from_bytes(host(self.box[k, :48])) for k in range(self.box.shape[0])]


@pytest.mark.parametrize("path", ["step", "feed", "nv12", "p010", "bgr24", "views"])
def test_golden_replay_against_twin_without_framing(fo, path):  # noqa: F811
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    ours, twin = Outputs(n), Outputs(n)
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(29)
    replay = [framing.new_box() for _ in range(n)]
    try:
        ts = TrackerSet(c, n, [dict(case["params"], **ours.params(k)) for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], **twin.params(k, frame=False)) for k, case in enumerate(cases)])
        clock, framed = 1.0e12, 0
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
            rgba_video, orient = {}, {}
            if path == "step":
                batch = T.from_numpy(np.stack(frames)).cuda()
                T.cuda.synchronize()
                ticked = dict(enumerate(ts.step(batch, clock)))
                assert equal_records(list(ticked.values()), tr.step(batch, clock)), i
                rgba_video = {k: frames[k] for k in ticked}
            elif listed:
                vids, kw = {}, {}
                for k in listed:
                    v = video(frames[k], 1 + k % 3, False)
                    o = (k + i) % 8 if path == "views" else 0
                    if path in ("feed", "views"):
                        vids[k] = to_device(unorient(v, o))
                        rgba_video[k], orient[k] = unorient(v, o), o
                    else:
                        fmt, color = {"nv12": ("nv12", "bt709"), "p010": ("p010", "bt2020"), "bgr24": ("bgr24", "bt601")}[path]
                        b = from_rgba(v, fmt, rng)
                        vids[k] = api_frame(b, True)
                        rgba_video[k] = oracle_convert(fo, b, color)
                        kw = dict(format=fmt, color=color)
                if path == "views":
                    kw = dict(view={k: {"rotate": 90 * (orient[k] & 3), "mirror": bool(orient[k] & 4), "crop": None}
                                    for k in listed})
                T.cuda.synchronize()
                call = "feed" if path in ("feed", "views") else "feed_yuv"
                ticked = getattr(ts, call)(vids, clock, W0, H0, **kw)
                assert equal_records(list(ticked.values()), list(getattr(tr, call)(vids, clock, W0, H0, **kw).values())), i
            else:
                ticked = {}
            T.cuda.synchronize()
            for k, rec in ticked.items():
                framing.framing_step(replay[k], rec, W0, H0, 0.25, 0.1)
            got = ours.boxes()
            for k in range(n):
                assert framing.box_to_bytes(got[k]) == framing.box_to_bytes(replay[k]), (i, k)
            for k in range(n):
                Sw, Sh, scale = ours.spec[k]
                if k in ticked and wrote(ticked[k]):
                    want = host_crop(replay[k], W0, H0, rgba_video[k], Sw, Sh, scale, orient.get(k, 0))
                    assert np.array_equal(host(ours.crop[k]), want), (path, i, k)
                    framed += 1
                if k % 2 == 0:      # a framed tensor: the RGB of the framed crop
                    assert T.equal(ours.tensor[k], ours.crop[k][..., :3]), (i, k)
                else:               # crop only: the tensor stays the tracked one
                    assert T.equal(ours.tensor[k], twin.tensor[k]), (i, k)
        assert framed > 30
        assert any(b["updates"] > 5 for b in ours.boxes())
        # a framed box that glides makes a crop other than the tracked one
        assert any(not T.equal(a, b) for a, b in zip(ours.crop, twin.crop))
    finally:
        c.close()
        ref.close()


def test_1024_streams_two_canvases_mixed_crops():
    T = torch()
    n, W, H = 1024, 640, 360
    canv = [(320, 240) if k % 2 else (160, 120) for k in range(n)]
    sizes = [(112, 112, 1.0), (64, 48, 1.5), (224, 224, 1.25), (30, 40, 1.0)]
    outs = Outputs(n, sizes)
    frames = [synth.frame(700 + i, W, H, n_faces=1) for i in range(6)]
    dframes = [T.from_numpy(f).cuda() for f in frames]
    rng = np.random.default_rng(77)
    ctx = Context(max_width=320, max_height=240, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        p = [outs.params(k, tensor=k % 3 == 0) for k in range(n)]
        ctx.tracker_set_face_crop(0, [q["faceCrop"] for q in p])
        ctx.tracker_set_face_tensor(0, [q["faceTensor"] for q in p])
        ctx.tracker_set_framing(0, [q["framing"] for q in p])
        sample = sorted(int(k) for k in rng.choice(n, 48, replace=False))
        replay = {k: framing.new_box() for k in sample}
        clock = [1.0e12 + 7.0 * k for k in range(n)]
        written = 0
        for tick in range(28):
            ks = [k for k in range(n) if rng.random() < 0.9]
            for k in ks:
                clock[k] += 35.0
            fidx = {k: (k + tick // 9) % 6 for k in ks}
            recs = ctx.tracker_feed(ks, [dframes[fidx[k]] for k in ks], [clock[k] for k in ks],
                                    [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            T.cuda.synchronize()
            byk = dict(zip(ks, recs))
            for k in sample:
                if k not in byk:
                    continue
                cw, ch = canv[k]
                framing.framing_step(replay[k], byk[k], cw, ch, 0.25, 0.1)
                assert framing.box_to_bytes(framing.box_from_bytes(host(outs.box[k, :48]))) == \
                    framing.box_to_bytes(replay[k]), (tick, k)
                if wrote(byk[k]):
                    Sw, Sh, scale = outs.spec[k]
                    want = host_crop(replay[k], cw, ch, frames[fidx[k]], Sw, Sh, scale)
                    assert np.array_equal(host(outs.crop[k]), want), (tick, k)
                    written += 1
        assert written > 100
    finally:
        ctx.close()


def box_of(ctx_box):
    return framing.box_from_bytes(host(ctx_box))


def test_lifetime_and_launch_counts():
    T = torch()
    ctx = Context(max_width=2 * W0, max_height=2 * H0, max_frames=2)
    twin = Context(max_width=2 * W0, max_height=2 * H0, max_frames=2)
    b = T.zeros((2, 64), dtype=T.uint8, device="cuda")
    crop = [T.zeros((32, 32, 4), dtype=T.uint8, device="cuda") for _ in range(2)]
    try:
        for x in (ctx, twin):
            x.tracker_config()
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
            x.tracker_set_face_crop(0, [{"out": crop[0]}, None] if x is ctx else [{"out": T.zeros_like(crop[0])}, None])
        run(ctx, 22, 0), run(twin, 22, 0)
        l0, t0 = ctx.launch_count, twin.launch_count
        run(ctx, 1, 22), run(twin, 1, 22)
        assert ctx.launch_count - l0 == twin.launch_count - t0          # no framing: the same launches

        ctx.tracker_set_framing(0, [{"out": b[0, :48]}, {"out": b[1, :48], "crop": False, "tensor": True}])
        T.cuda.synchronize()
        assert box_of(b[0, :48]) == framing.new_box() == box_of(b[1, :48])
        l0, t0 = ctx.launch_count, twin.launch_count
        recs = run(ctx, 1, 23)
        run(twin, 1, 23)
        assert ctx.launch_count - l0 == twin.launch_count - t0 + 1       # one more with a framing
        assert wrote(recs[0]) and box_of(b[0, :48])["valid"] == 1 and box_of(b[0, :48])["updates"] == 1
        assert box_of(b[1, :48])["updates"] == 1                          # a stream without a crop still frames

        def kept(op, t):
            before = box_of(b[0, :48])
            op()
            T.cuda.synchronize()
            assert box_of(b[0, :48]) == before, op
            recs = run(ctx, 1, t)
            after = box_of(b[0, :48])
            assert after["updates"] == before["updates"] + wrote(recs[0]), op
        kept(lambda: ctx.tracker_set_params(0, [dict()]), 24)
        kept(lambda: ctx.tracker_set_face_crop(0, [{"out": crop[0], "scale": 1.5}]), 25)
        rec = ctx.tracker_export([0])
        kept(lambda: ctx.tracker_import([1], rec), 26)
        assert box_of(b[1, :48])["updates"] == 4                         # the framing stayed on id 1
        ctx.tracker_stop(0, 1)
        before = box_of(b[0, :48])
        run(ctx, 3, 27)
        assert box_of(b[0, :48]) == before                               # stopped: no crop ticks
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        run(ctx, 22, 30)                                                 # starter, whitebalance, VJ, then CS again
        again = box_of(b[0, :48])
        assert again["valid"] == 1 and again["updates"] > before["updates"]

        # lost, then refound inside the box (a glide) and outside it (a snap): driven through framing.py's rule on
        # the same records, the device box follows byte for byte
        rep = box_of(b[0, :48])
        import make_goldens_params as pg
        for t, f in ((60, "face"), (61, "empty"), (62, "empty"), (63, "face"), (64, "face")):
            r = ctx.tracker_feed([0], [pg.make_frame(f, t, W0, H0)], 1.0e12 + 35.0 * t, W0, H0)[0]
            framing.framing_step(rep, r, W0, H0, 0.25, 0.1)
            assert framing.box_to_bytes(box_of(b[0, :48])) == framing.box_to_bytes(rep), t

        # a canvas-size change snaps
        for t in range(65, 120):          # lost on the new canvas, then found again there: the first crop tick snaps
            r = ctx.tracker_feed([0], [pg.make_frame("face", t, W0, H0)], 1.0e12 + 35.0 * t, 2 * W0, 2 * H0)[0]
            framing.framing_step(rep, r, 2 * W0, 2 * H0, 0.25, 0.1)
            assert framing.box_to_bytes(box_of(b[0, :48])) == framing.box_to_bytes(rep), t
            if wrote(r):
                break
        assert wrote(r)
        nb = box_of(b[0, :48])
        assert framing.box_to_bytes(nb) == framing.box_to_bytes(rep)
        assert (nb["canvas_w"], nb["canvas_h"]) == (2 * W0, 2 * H0) and (nb["width"], nb["height"]) == (r["width"], r["height"])

        ctx.tracker_config()                                              # removes every framing
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        b.fill_(0x5A)
        T.cuda.synchronize()
        run(ctx, 24, 0)
        assert (host(b) == 0x5A).all()
    finally:
        ctx.close()
        twin.close()


def test_framing_off_launches_nothing_more():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    twin = Context(max_width=W0, max_height=H0, max_frames=2)
    b = T.zeros((48,), dtype=T.uint8, device="cuda")
    try:
        for x in (ctx, twin):
            x.tracker_config()
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
        ctx.tracker_set_framing(0, [{"out": b}])
        ctx.tracker_set_framing(0, [None])                                 # removed again
        run(ctx, 22, 0), run(twin, 22, 0)
        l0, t0 = ctx.launch_count, twin.launch_count
        run(ctx, 2, 22), run(twin, 2, 22)
        assert ctx.launch_count - l0 == twin.launch_count - t0
    finally:
        ctx.close()
        twin.close()


def test_overlap_both_ways_and_rejections():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=4)
    buf = T.zeros((4096,), dtype=T.uint8, device="cuda")
    base = buf.data_ptr()
    L = _lib.lib()

    def setf(recs, first=0):
        arr = (_lib.Framing * len(recs))(*recs)
        return L.ht_tracker_set_framing(ctx._h, first, len(recs), C.addressof(arr))

    def last_error():
        return (L.ht_last_error(ctx._h) or b"").decode()

    def fr(p, alpha=0.25, dz=0.1, outputs=1, pad=0):
        return _lib.Framing(p, alpha, dz, outputs, pad)
    try:
        assert setf([fr(base)]) == HT_ERR_STATE
        ctx.tracker_config()
        assert setf([fr(base)]) == 0
        # a camera on the box, in either order; a crop, a tensor and a debug canvas on it
        cam = dict(scaling=1, fixedPosition=(0, 0, 60), lookAt=(0, 0, 0), fov=45, aspect=1.5, near=1, far=1000)
        with pytest.raises(_lib.HtError, match="framed box"):
            ctx.tracker_set_camera(1, [dict(cam, out=buf[0:224])])
        with pytest.raises(_lib.HtError, match="framed box"):
            ctx.tracker_set_face_crop(1, [{"out": buf[32:32 + 64].view(4, 4, 4)}])
        with pytest.raises(_lib.HtError, match="framed box"):
            ctx.tracker_set_debug(1, [buf[0:64].view(4, 4, 4)])
        with pytest.raises(_lib.HtError, match="framed box"):
            ctx.tracker_set_face_tensor(1, [{"out": buf[40:40 + 12].view(2, 2, 3), "layout": "hwc"}])
        ctx.tracker_set_camera(1, [dict(cam, out=buf[1024:1024 + 224])])
        assert setf([fr(base + 1024 + 216)], 2) == HT_ERR_ARG and "camera" in last_error()
        assert setf([fr(base + 1024 + 224)], 2) == 0
        assert setf([fr(base + 48)], 3) == 0 and setf([fr(base + 40)], 3) == HT_ERR_ARG
        # every rejection, with nothing changed
        before = host(buf).copy()
        host_box = (C.c_char * 64)()
        for bad in (fr(base + 4 + 2048), fr(C.addressof(host_box)), fr(base + 2048, alpha=0.0), fr(base + 2048, alpha=1.5),
                    fr(base + 2048, alpha=float("nan")), fr(base + 2048, dz=-0.01), fr(base + 2048, dz=0.51),
                    fr(base + 2048, dz=float("inf")), fr(base + 2048, outputs=0), fr(base + 2048, outputs=4),
                    fr(base + 2048, outputs=-1), fr(base + 2048, pad=1)):
            assert setf([fr(0), bad]) == HT_ERR_ARG
            assert last_error().startswith("record 1:"), last_error()
        assert setf([fr(base + 2048)], 4) == HT_ERR_ARG                     # a range past max_frames
        assert L.ht_tracker_set_framing(ctx._h, 0, 1, None) == HT_ERR_ARG
        assert L.ht_tracker_set_framing(ctx._h, 0, 0, C.addressof((_lib.Framing * 1)())) == HT_ERR_ARG
        T.cuda.synchronize()
        assert np.array_equal(host(buf), before)
        with pytest.raises(ValueError):
            ctx.tracker_set_framing(0, [{"out": buf[:47]}])
    finally:
        ctx.close()
