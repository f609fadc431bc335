"""GPU: face redaction (ht_tracker_set_redact, Context.tracker_set_redact, TrackerSet's "redact" key; DESIGN.md 2,
"Face redaction"): each stream's tracked face hidden in its own video, on the device, after the tick's crops:

  * every case of reference_js_debug.json through step, feed (RGBA), feed_yuv (NV12, I420, P010, YUYV, BGR24) and
    feed through views, against a twin context without redaction: records byte-identical, crops equal to the twin's
    (cut before the redaction), and every video after its tick the restatement's (tests/redact_oracle.c) redaction of
    its pre-tick copy under the replayed hold; through step the camshift model at every hand-off equals the twin's;
  * 1024 streams on two canvas sizes with mixed modes, cell sizes, scales and holds, a seeded sample checked;
  * the lifetime, the launch count, and every rejection (host video, two redacting records on one frame, bad
    records), each leaving nothing enqueued; streams without a redaction may still share a frame."""
import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, make_frame
from test_gpu_debug import black
from test_gpu_feed import equal_records
from test_gpu_formats import from_rgba
from test_gpu_views import unorient

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]
CODE = {"rgba": -1, "nv12": 0, "i420": 1, "p010": 21, "yuyv": 19, "bgr24": 33}
COLOR = {"nv12": "bt709", "i420": "bt601", "p010": "bt2020", "yuyv": "bt601", "bgr24": "bt601"}


def torch():
    import torch as t
    return t


def oracle():
    global _RO
    try:
        return _RO
    except NameError:
        pass
    so = Path(tempfile.mkdtemp()) / "libredact_oracle.so"
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(so),
                           str(Path(__file__).with_name("redact_oracle.c")), "-lm"])
    L = C.CDLL(str(so))
    L.hro_rect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double,
                           C.c_void_p]
    L.hro_hold.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.hro_redact.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    _RO = L
    return L


class Replay:
    """one stream's redaction replayed by the restatement: its hold, and the redaction of a host copy of a video"""

    def __init__(self, d):
        self.d, self.state = d, (C.c_char * 56)()

    def apply(self, rec, cw, ch, fmt, planes, w, h, o=0):
        """planes: uint8 numpy arrays (rows of their pitch), redacted in place -> whether the tick redacted"""
        det = {"": 0, "VJ": 1, "CS": 2, "WB": 3}[rec["detection"]]
        r = (C.c_double * 7)(det, rec["x"], rec["y"], rec["width"], rec["height"], rec["angle"], rec["confidence"])
        L = oracle()
        if not L.hro_hold(self.state, self.d["hold"], r, cw, ch):
            return False
        box = np.frombuffer(bytes(self.state)[:40], np.float64)
        stored = int(np.frombuffer(bytes(self.state)[40:44], np.int32)[0])
        W, H = (h, w) if o & 1 else (w, h)
        out = (C.c_int32 * 4)()
        if not L.hro_rect((C.c_double * 7)(stored, *box, 1.0), cw, ch, w, h, o, (C.c_int32 * 4)(0, 0, W, H),
                          self.d["block"], self.d["scale"], out):
            return False
        p = (C.c_void_p * 3)(*([q.ctypes.data for q in planes] + [0] * (3 - len(planes))))
        pitch = (C.c_int32 * 3)(*([q.strides[0] for q in planes] + [0] * (3 - len(planes))))
        mode = {"mosaic": 1, "fill": 2}[self.d["mode"]]
        L.hro_redact(CODE[fmt], p, pitch, out, mode, self.d["block"], (C.c_uint8 * 3)(*self.d["fill_rgb"]),
                     (C.c_uint8 * 3)(*self.d["fill_yuv"]))
        return True


def red(k):
    return {"mode": "mosaic" if k % 2 == 0 else "fill", "block": (16, 4, 2, 8)[k % 4], "scale": (1.25, 1.0, 2.0)[k % 3],
            "hold": (10, 0, 3)[k % 3], "fill_rgb": (10, 20, 30), "fill_yuv": (40, 50, 60)}


class DevFrame:
    """byte planes of a frame on the device, and the argument the wrappers take for them"""

    def __init__(self, fmt, planes, w, h):
        T = torch()
        self.fmt, self.w, self.h = fmt, w, h
        self.bases = [T.from_numpy(np.ascontiguousarray(p)).cuda() for p in planes]
        b = self.bases
        if fmt == "rgba":
            self.arg = b[0].view(h, w, 4)
        elif fmt in ("yuyv", "bgr24"):
            c = {"yuyv": 2, "bgr24": 3}[fmt]
            self.arg = b[0].as_strided((h, w, c), (b[0].stride(0), c, 1))
        elif fmt == "p010":
            self.arg = tuple(p.view(T.int16) for p in b)
        else:
            self.arg = tuple(b)

    def host(self):
        return [p.cpu().numpy().copy() for p in self.bases]


def byte_planes(rgba, fmt, rng):
    if fmt == "rgba":
        return [np.ascontiguousarray(rgba).reshape(rgba.shape[0], -1)]
    return list(from_rgba(rgba, fmt, rng)[3])


@pytest.mark.parametrize("path", ["step", "rgba", "nv12", "i420", "p010", "yuyv", "bgr24", "views"])
def test_golden_replay_against_twin_without_redaction(path):
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(31)
    crops = [T.zeros((48, 40, 4), dtype=T.uint8, device="cuda") for _ in range(2 * n)]
    replay = [Replay(red(k)) for k in range(n)]
    try:
        ts = TrackerSet(c, n, [dict(case["params"], faceCrop={"out": crops[k]}, redact=red(k))
                               for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], faceCrop={"out": crops[n + k]}) for k, case in enumerate(cases)])
        clock, redacted, handoffs, seeded = 1.0e12, 0, 0, set()
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
            before, ours, o = {}, {}, {}
            if path == "step":
                batch, twin = T.from_numpy(np.stack(frames)).cuda(), T.from_numpy(np.stack(frames)).cuda()
                T.cuda.synchronize()
                ticked = dict(enumerate(ts.step(batch, clock)))
                assert equal_records(list(ticked.values()), tr.step(twin, clock)), i
                T.cuda.synchronize()
                for k in ticked:
                    before[k] = [frames[k].reshape(H0, -1).copy()]
                    ours[k] = [batch[k].cpu().numpy().reshape(H0, -1)]
                # k_track_init read the frames before they were redacted: the model of every slot that has been
                # seeded (a VJ record that passes the confidence gate hands off on its own frame) equals the twin's.
                # A slot never seeded holds no model yet: its memory is dead state, as for an exported non-CS stream.
                for k, rec in ticked.items():
                    if rec["detection"] == "VJ" and rec["confidence"] > -10:
                        seeded.add(k)
                        handoffs += 1
                for k in sorted(seeded):
                    assert np.array_equal(c.debug_model_hist(k), ref.debug_model_hist(k)), (i, k)
                fmt, size = "rgba", {k: (W0, H0) for k in ticked}
            elif listed:
                fmt = "rgba" if path in ("rgba", "views") else path
                vids, twins, size = {}, {}, {}
                for k in listed:
                    v = np.repeat(np.repeat(frames[k], 1 + k % 3, axis=0), 1 + k % 3, axis=1)
                    o[k] = (k + i) % 8 if path == "views" else 0
                    v = unorient(v, o[k])
                    planes = byte_planes(v, fmt, rng)
                    vids[k], twins[k] = DevFrame(fmt, planes, v.shape[1], v.shape[0]), DevFrame(fmt, planes, v.shape[1], v.shape[0])
                    before[k], size[k] = [p.copy() for p in planes], (v.shape[1], v.shape[0])
                kw = {}
                if path == "views":
                    kw = dict(view={k: {"rotate": 90 * (o[k] & 3), "mirror": bool(o[k] & 4), "crop": None} for k in listed})
                elif fmt != "rgba":
                    kw = dict(format=fmt, color=COLOR[fmt])
                T.cuda.synchronize()
                call = "feed" if fmt == "rgba" else "feed_yuv"
                ticked = getattr(ts, call)({k: vids[k].arg for k in listed}, clock, W0, H0, **kw)
                got = getattr(tr, call)({k: twins[k].arg for k in listed}, clock, W0, H0, **kw)
                assert equal_records(list(ticked.values()), list(got.values())), i
                T.cuda.synchronize()
                ours = {k: vids[k].host() for k in listed}
                for k in listed:                    # the twin's video is untouched
                    assert all(np.array_equal(a, b) for a, b in zip(twins[k].host(), before[k])), (i, k)
            else:
                ticked = {}
            for k, rec in ticked.items():
                w, h = size[k]
                redacted += replay[k].apply(rec, W0, H0, fmt, before[k], w, h, o.get(k, 0))
                assert all(np.array_equal(a, b) for a, b in zip(ours[k], before[k])), (path, i, k)
            for k in range(n):                      # the crops were cut from the unredacted video
                assert T.equal(crops[k], crops[n + k]), (i, k)
        assert redacted > 30
        if path == "step":
            assert handoffs > 0
    finally:
        c.close()
        ref.close()


def test_1024_streams_two_canvases_mixed_blocks_and_modes():
    T = torch()
    n, W, H = 1024, 640, 360
    canv = [(320, 240) if k % 2 else (160, 120) for k in range(n)]
    rng = np.random.default_rng(77)
    frames = [synth.frame(700 + i, W, H, n_faces=1) for i in range(6)]
    dframes = [T.from_numpy(f).cuda() for f in frames]
    ctx = Context(max_width=320, max_height=240, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        ctx.tracker_set_redact(0, [red(k) for k in range(n)])
        sample = sorted(int(k) for k in rng.choice(n, 48, replace=False))
        replay = {k: Replay(red(k)) for k in sample}
        clock = [1.0e12 + 7.0 * k for k in range(n)]
        redacted = 0
        for tick in range(28):
            ks = [k for k in range(n) if rng.random() < 0.9]
            for k in ks:
                clock[k] += 35.0
            fidx = {k: (k + tick // 9) % 6 for k in ks}
            vids = {k: dframes[fidx[k]].clone() for k in ks}     # a redacting stream's own copy of its camera frame
            recs = ctx.tracker_feed(ks, [vids[k] for k in ks], [clock[k] for k in ks],
                                    [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            T.cuda.synchronize()
            byk = dict(zip(ks, recs))
            for k in sample:
                if k in byk:
                    want = [frames[fidx[k]].reshape(H, -1).copy()]
                    redacted += replay[k].apply(byk[k], canv[k][0], canv[k][1], "rgba", want, W, H)
                    assert np.array_equal(vids[k].cpu().numpy().reshape(H, -1), want[0]), (tick, k)
        assert redacted > 100
    finally:
        ctx.close()


def face_tick(r):
    return r["detection"] in ("VJ", "CS") and r["confidence"] != 0 and r["width"] > 0 and r["height"] > 0


def test_lifetime_and_launch_counts():
    T = torch()
    import make_goldens_params as pg
    ctx = Context(max_width=2 * W0, max_height=2 * H0, max_frames=2)
    twin = Context(max_width=2 * W0, max_height=2 * H0, max_frames=2)
    d = dict(red(0), hold=4, mode="fill", block=2, scale=1.0)

    def feed(x, t, kind="face", cw=W0, ch=H0):
        """one tick of streams 0 and 1 on device frames -> (records, stream 0's frame was redacted)"""
        f = pg.make_frame(kind, t, W0, H0)
        dev = [T.from_numpy(f).cuda() for _ in range(2)]
        r = x.tracker_feed([0, 1], dev, 1.0e12 + 35.0 * t, cw, ch)
        T.cuda.synchronize()
        assert np.array_equal(dev[1].cpu().numpy(), f)                     # stream 1 has no redaction
        return r, not np.array_equal(dev[0].cpu().numpy(), f)

    def both(t, kind="face", cw=W0, ch=H0):
        (a, on), (b, _) = feed(ctx, t, kind, cw, ch), feed(twin, t, kind, cw, ch)
        assert equal_records(a, b), t
        return a[0], on
    try:
        for x in (ctx, twin):
            x.tracker_config()
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
        for t in range(22):
            both(t)
        l0, t0 = ctx.launch_count, twin.launch_count
        both(22)
        assert ctx.launch_count - l0 == twin.launch_count - t0          # no redaction: the same launches
        ctx.tracker_set_redact(0, [d])
        ctx.tracker_set_redact(1, [None])
        l0, t0 = ctx.launch_count, twin.launch_count
        r, on = both(23)
        assert ctx.launch_count - l0 == twin.launch_count - t0 + 1       # one more with a redaction
        assert face_tick(r) and on
        ctx.tracker_set_params(0, [dict()]), twin.tracker_set_params(0, [dict()])
        assert both(24)[1]
        for x in (ctx, twin):
            x.tracker_import([0], x.tracker_export([0]))
        assert both(25)[1]
        # lost: the hold redacts the last box on the same canvas
        r, on = both(26, "empty")
        assert not face_tick(r) and r["detection"] in ("CS", "VJ") and on
        for x in (ctx, twin):                                             # an IDLE tick: nothing, and no hold after
            x.tracker_stop(0, 1)
        r, on = both(27)
        assert r["detection"] == "" and not on
        for x in (ctx, twin):
            x.tracker_reset(0, 1)
            x.tracker_start(0, 1)
        seen = [both(t) for t in range(28, 52)]
        assert any(on for _, on in seen)
        for r, on in seen:
            assert on == face_tick(r) or (on and r["detection"] in ("VJ", "CS")), r
        assert face_tick(seen[-1][0])
        # a canvas-size change drops the hold
        r, on = both(52, "empty", 2 * W0, 2 * H0)
        assert on == face_tick(r), r
        if not face_tick(r):
            r, on = both(53, "empty", 2 * W0, 2 * H0)
            assert not on and not face_tick(r)
        for x in (ctx, twin):
            x.tracker_config()                                            # removes every redaction
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
        l0, t0 = ctx.launch_count, twin.launch_count
        for t in range(24):
            assert not both(60 + t)[1]
        assert ctx.launch_count - l0 == twin.launch_count - t0
    finally:
        ctx.close()
        twin.close()


def test_rejections_enqueue_nothing_and_the_next_tick_equals_the_twin():
    T = torch()
    import make_goldens_params as pg
    ctx = Context(max_width=W0, max_height=H0, max_frames=4)
    twin = Context(max_width=W0, max_height=H0, max_frames=4)
    L = _lib.lib()

    def setr(recs, first=0):
        arr = (_lib.FaceRedact * len(recs))(*recs)
        return L.ht_tracker_set_redact(ctx._h, first, len(recs), C.addressof(arr))

    def last_error():
        return (L.ht_last_error(ctx._h) or b"").decode()

    def fr(mode=1, block=16, hold=10, scale=1.25, pads=(0, 0, 0)):
        d = _lib.FaceRedact(mode, block, hold)
        d.pad0, d.pad1, d.pad_ = pads
        d.scale = scale
        return d
    try:
        assert setr([fr()]) == HT_ERR_STATE
        for x in (ctx, twin):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        for bad in (fr(mode=3), fr(mode=-1), fr(block=3), fr(block=0), fr(block=130), fr(hold=-1), fr(hold=65536),
                    fr(scale=0.0), fr(scale=16.5), fr(scale=float("nan")), fr(pads=(1, 0, 0)), fr(pads=(0, 1, 0)),
                    fr(pads=(0, 0, 1))):
            assert setr([fr(), bad]) == HT_ERR_ARG
            assert last_error().startswith("record 1:"), last_error()
        assert setr([fr()], 4) == HT_ERR_ARG
        assert L.ht_tracker_set_redact(ctx._h, 0, 1, None) == HT_ERR_ARG
        assert setr([fr(), fr()]) == 0                                    # streams 0 and 1 redact
        t = 0

        def both(frames_ours, frames_twin, kw_ours=None):
            nonlocal t
            a = ctx.tracker_feed(list(range(4)), frames_ours, 1.0e12 + 35.0 * t, W0, H0)
            b = twin.tracker_feed(list(range(4)), frames_twin, 1.0e12 + 35.0 * t, W0, H0)
            t += 1
            assert equal_records(a, b), t
        face = [pg.make_frame("face", 0, W0, H0)] * 4
        # streams 0, 1 redact and their video is host memory: refused, nothing enqueued
        with pytest.raises(_lib.HtError, match="record 0: stream 0 redacts"):
            ctx.tracker_feed(list(range(4)), face, 1.0e12 + 35.0 * t, W0, H0)
        dev = [T.from_numpy(pg.make_frame("face", 1, W0, H0)).cuda() for _ in range(4)]
        shared = T.from_numpy(pg.make_frame("face", 1, W0, H0)).cuda()
        with pytest.raises(_lib.HtError, match="record 1: its video shares bytes with record 0"):
            ctx.tracker_feed(list(range(4)), [shared, shared, dev[2], dev[3]], 1.0e12 + 35.0 * t, W0, H0)
        with pytest.raises(_lib.HtError, match="frames must be device memory"):
            ctx.tracker_step(np.stack(face), 1.0e12 + 35.0 * t)
        # non-redacting streams may share a frame; the next tick equals the twin's
        for k in range(20):
            f = pg.make_frame("face", 2 + k, W0, H0)
            d = [T.from_numpy(f).cuda() for _ in range(3)]
            e = T.from_numpy(f).cuda()
            both([d[0], d[1], e, e], [f] * 4)
        T.cuda.synchronize()
    finally:
        ctx.close()
        twin.close()
