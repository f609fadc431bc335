"""GPU: best shots (ht_tracker_set_best_shot, Context.tracker_set_best_shot, TrackerSet's "bestShot" key; DESIGN.md 2,
"Best shots"): per track the sharpest crop tick's face, scored and kept on the device.

Each stream carries a best shot and, as its twin, an RGBA face crop of the same size and scale.  After every tick the
host scores the twin crop (bestshot.score) and steps bestshot.step on the tick's record; the state bytes must equal
the mirror's and the image the state names must equal the saved twin crop of the mirror's best tick, byte for byte
(with two images, the previous track's final best must stay in the other one).  A twin context without best shots
gives the same records and crops.

  * every case of reference_js_debug.json through step, feed, feed_yuv (NV12, P010, BGR24) and feed through views, and
    the main.js / lifecycle runs of reference_js_main.json and reference_js_lifecycle.json through step;
  * 1024 streams on two canvas sizes with mixed best-shot sizes, a seeded sample checked;
  * with a redaction the best shot is unredacted; with a framing (crop and tensor) it ignores it;
  * the lifecycle calls, the launch counts, the overlap rule both ways and every rejection."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, bestshot, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, make_frame
from test_gpu_debug import black, run
from test_gpu_feed import equal_records, to_device, video
from test_gpu_formats import api_frame, from_rgba
from test_gpu_views import unorient

pytestmark = pytest.mark.gpu

W0, H0 = GOLD_D["width"], GOLD_D["height"]
SIZES = [(112, 112, 1.0), (64, 96, 1.5), (48, 48, 0.75), (100, 60, 2.0), (34, 18, 1.0), (3, 3, 1.0), (130, 20, 0.5)]


def torch():
    import torch as t
    return t


def host(t):
    return t.cpu().numpy()


class Shots:
    """per stream a best shot (two images for k % 3 != 2, else one; state slots 128 bytes apart) and a twin RGBA crop of
    the same size and scale, with the host mirror of every state"""

    def __init__(self, n, sizes=SIZES):
        T = torch()
        self.n = n
        self.spec = [sizes[k % len(sizes)] for k in range(n)]
        self.two = [k % 3 != 2 for k in range(n)]
        self.img = [[T.full((Sh, Sw, 4), 0x33, dtype=T.uint8, device="cuda") for _ in range(2 if two else 1)]
                    for (Sw, Sh, _), two in zip(self.spec, self.two)]
        self.twin = [T.zeros((Sh, Sw, 4), dtype=T.uint8, device="cuda") for Sw, Sh, _ in self.spec]
        self.state = T.full((n, 128), 0x77, dtype=T.uint8, device="cuda")
        self.mirror = [bestshot.new_state() for _ in range(n)]
        self.saved = [[None, None] for _ in range(n)]     # per image: the twin crop it must hold
        self.checked = self.writes = 0

    def shot(self, k):
        Sw, Sh, scale = self.spec[k]
        return {"out": tuple(self.img[k]) if self.two[k] else self.img[k][0], "state": self.state[k, :96], "scale": scale}

    def crop(self, k):
        return {"out": self.twin[k], "scale": self.spec[k][2]}

    def params(self, k):
        return {"bestShot": self.shot(k), "faceCrop": self.crop(k)}

    def reset(self, k):
        self.mirror[k] = bestshot.new_state()

    def tick(self, ticked, canvas, clock, twin=None):
        """ticked: {stream: record} of one tick; canvas(k) -> (cw, ch); clock(k) -> now_ms; twin: the crops the
        candidates equal (default: the streams' own)"""
        twin = twin or self.twin
        for k, rec in ticked.items():
            cand = host(twin[k]).copy() if bestshot.crop_tick(rec) else None
            s = bestshot.score(cand) if cand is not None else 0
            if bestshot.step(self.mirror[k], rec, s, clock(k), *canvas(k), self.two[k]):
                self.saved[k][self.mirror[k]["buffer"]] = cand
                self.writes += 1

    def check(self, ks=None, where=""):
        st = host(self.state)
        for k in (range(self.n) if ks is None else ks):
            assert st[k, :96].tobytes() == bestshot.state_to_bytes(self.mirror[k]), \
                (where, k, bestshot.state_from_bytes(st[k, :96]), self.mirror[k])
            assert (st[k, 96:] == 0x77).all(), (where, k)
            for b, want in enumerate(self.saved[k]):
                if want is not None:
                    assert np.array_equal(host(self.img[k][b]), want), (where, k, b)
                    self.checked += 1


def drive_debug_golden(path, ts, tr, rng):
    """every case of the debug golden through `path` on TrackerSets ts (best shots) and tr (twin context, crops only)"""
    T = torch()
    cases = GOLD_D["cases"]
    clock = 1.0e12
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
                o = (k + i) % 8 if path == "views" else 0
                if path in ("feed", "views"):
                    vids[k] = to_device(unorient(v, o))
                else:
                    fmt, color = {"nv12": ("nv12", "bt709"), "p010": ("p010", "bt2020"), "bgr24": ("bgr24", "bt601")}[path]
                    vids[k] = api_frame(from_rgba(v, fmt, rng), True)
                    kw = dict(format=fmt, color=color)
            if path == "views":
                kw = dict(view={k: {"rotate": 90 * (((k + i) % 8) & 3), "mirror": bool(((k + i) % 8) & 4), "crop": None}
                                for k in listed})
            T.cuda.synchronize()
            call = "feed" if path in ("feed", "views") else "feed_yuv"
            ticked = getattr(ts, call)(vids, clock, W0, H0, **kw)
            assert equal_records(list(ticked.values()), list(getattr(tr, call)(vids, clock, W0, H0, **kw).values())), i
        else:
            ticked = {}
        T.cuda.synchronize()
        yield i, ticked, clock


@pytest.mark.parametrize("path", ["step", "feed", "nv12", "p010", "bgr24", "views"])
def test_debug_golden_replay(path):
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    shots, twin = Shots(n), Shots(n)
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(31)
    try:
        ts = TrackerSet(c, n, [dict(case["params"], **shots.params(k)) for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], faceCrop=twin.crop(k)) for k, case in enumerate(cases)])
        for i, ticked, clock in drive_debug_golden(path, ts, tr, rng):
            shots.tick(ticked, lambda k: (W0, H0), lambda k: clock)
            shots.check(where=(path, i))
            for k in range(n):
                assert T.equal(shots.twin[k], twin.twin[k]), (i, k)       # the crops are the twin context's
        assert shots.writes > 10 and shots.checked > 50
        assert any(m["track"] >= 1 and m["ended"] >= 1 for m in shots.mirror)
        assert any(m["best_tick"] > 0 for m in shots.mirror)            # some track improved after its first tick
    finally:
        c.close()
        ref.close()


def test_main_and_lifecycle_goldens_through_step():
    from test_gpu_tracker import BATCHES, MS, W as WL, H as HL, black as black_l
    from test_host_lifecycle import case_spec, make_frame as make_frame_l
    T = torch()
    params, streams = BATCHES["default"]
    n = len(streams)
    sizes = [(56, 64, 1.25), (33, 33, 1.0), (3, 7, 4.0)]
    shots, twin = Shots(n, sizes), Shots(n, sizes)
    c = Context(max_width=WL, max_height=HL, max_frames=16)
    ref = Context(max_width=WL, max_height=HL, max_frames=16)
    try:
        ts = TrackerSet(c, n, [dict(params, **shots.params(k)) for k in range(n)])
        tr = TrackerSet(ref, n, [dict(params, faceCrop=twin.crop(k)) for k in range(n)])
        specs = [case_spec(s[0])[0] if isinstance(s, tuple) else None for s in streams]
        steps = max(s[1] + len(sp) for s, sp in zip(streams, specs) if sp) + 2
        for t in range(steps):
            frames = []
            for k, s in enumerate(streams):
                f = black_l()
                if s == "black" and t == 0:
                    ts.start(k), tr.start(k)
                if isinstance(s, tuple) and 0 <= t - s[1] < len(specs[k]):
                    action, kind, tt = specs[k][t - s[1]]
                    if action == "start":
                        ts.start(k), tr.start(k)
                    if action == "stop":
                        ts.stop(k), tr.stop(k)
                    else:
                        f = make_frame_l(kind, tt)
                frames.append(f)
            batch = T.from_numpy(np.stack(frames)).cuda()
            T.cuda.synchronize()
            now = 1.0e12 + MS * t
            recs = ts.step(batch, now_ms=now)
            assert equal_records(recs, tr.step(batch, now_ms=now)), t
            T.cuda.synchronize()
            shots.tick(dict(enumerate(recs)), lambda k: (WL, HL), lambda k: now)
            shots.check(where=t)
        assert shots.writes > 5 and sum(m["ended"] for m in shots.mirror) >= 1
    finally:
        c.close()
        ref.close()


def test_1024_streams_two_canvases_mixed_sizes():
    T = torch()
    n, W, H = 1024, 640, 360
    canv = [(320, 240) if k % 2 else (160, 120) for k in range(n)]
    sizes = [(112, 112, 1.0), (64, 48, 1.5), (224, 224, 1.25), (30, 40, 1.0), (3, 3, 2.0)]
    shots = Shots(n, sizes)
    frames = [synth.frame(900 + i, W, H, n_faces=1) for i in range(6)]
    dframes = [T.from_numpy(f).cuda() for f in frames]
    rng = np.random.default_rng(78)
    ctx = Context(max_width=320, max_height=240, max_frames=n)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, n)
        ctx.tracker_start(0, n)
        ctx.tracker_set_face_crop(0, [shots.crop(k) for k in range(n)])
        ctx.tracker_set_best_shot(0, [shots.shot(k) for k in range(n)])
        sample = sorted(int(k) for k in rng.choice(n, 48, replace=False))
        clock = [1.0e12 + 7.0 * k for k in range(n)]
        for tick in range(30):
            ks = [k for k in range(n) if rng.random() < 0.9]
            for k in ks:
                clock[k] += 35.0
            fidx = {k: (k + tick // 9) % 6 for k in ks}
            recs = ctx.tracker_feed(ks, [dframes[fidx[k]] for k in ks], [clock[k] for k in ks],
                                    [canv[k][0] for k in ks], [canv[k][1] for k in ks])
            T.cuda.synchronize()
            byk = {k: r for k, r in zip(ks, recs) if k in sample}
            shots.tick(byk, lambda k: canv[k], lambda k: clock[k])
            shots.check(sample, where=tick)
        assert shots.writes > 50 and shots.checked > 150
        st = host(shots.state)
        assert sum(bestshot.state_from_bytes(st[k, :96])["track"] > 0 for k in range(n)) > n // 2
    finally:
        ctx.close()


def test_redaction_and_framing_do_not_reach_the_best_shot():
    T = torch()
    n = 4
    shots, twin = Shots(n), Shots(n)
    box = T.zeros((n, 64), dtype=T.uint8, device="cuda")
    tens = [T.zeros((Sh, Sw, 3), dtype=T.uint8, device="cuda") for Sw, Sh, _ in shots.spec]
    ctx = Context(max_width=W0, max_height=H0, max_frames=n)
    ref = Context(max_width=W0, max_height=H0, max_frames=n)
    try:
        for x, s in ((ctx, shots), (ref, twin)):
            x.tracker_config()
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
            x.tracker_set_face_crop(0, [s.crop(k) for k in range(n)])
        ctx.tracker_set_best_shot(0, [shots.shot(k) for k in range(n)])
        # streams 0, 1 redact their faces; 2, 3 frame their crop and tensor
        ctx.tracker_set_redact(0, [{"mode": "fill", "block": 8, "scale": 1.5}, {"mode": "mosaic"}])
        ctx.tracker_set_framing(2, [{"out": box[k, :48], "alpha": 0.25, "crop": True, "tensor": True} for k in (2, 3)])
        ctx.tracker_set_face_tensor(2, [{"out": tens[k], "layout": "hwc", "scale": shots.spec[k][2]} for k in (2, 3)])
        import make_goldens_params as pg
        framed_apart = redacted = 0
        for t in range(40):
            f = pg.make_frame("face", t, W0, H0)
            vids = [T.from_numpy(f.copy()).cuda() for _ in range(n)]   # each stream its own video: redaction writes it
            T.cuda.synchronize()
            now = 1.0e12 + 35.0 * t
            recs = ctx.tracker_feed(list(range(n)), vids, now, W0, H0)
            ref_vids = [T.from_numpy(f.copy()).cuda() for _ in range(n)]
            T.cuda.synchronize()
            assert equal_records(recs, ref.tracker_feed(list(range(n)), ref_vids, now, W0, H0)), t
            T.cuda.synchronize()
            redacted += int(not np.array_equal(host(vids[0]), f))
            framed_apart += int(not T.equal(shots.twin[2], twin.twin[2]))
            shots.tick(dict(enumerate(recs)), lambda k: (W0, H0), lambda k: now, twin=twin.twin)   # the unframed crop
            shots.check(where=t)
        assert redacted > 5 and framed_apart > 5 and shots.writes > 4
    finally:
        ctx.close()
        ref.close()


def state_of(shots, k):
    return bestshot.state_from_bytes(host(shots.state[k, :96]))


def test_lifecycle_and_launch_counts():
    T = torch()
    shots = Shots(2, [(40, 40, 1.0), (24, 30, 1.5)])
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    twin = Context(max_width=W0, max_height=H0, max_frames=2)
    twin_crop = [T.zeros_like(t) for t in shots.twin]
    try:
        for x in (ctx, twin):
            x.tracker_config()
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
        ctx.tracker_set_face_crop(0, [shots.crop(k) for k in range(2)])
        twin.tracker_set_face_crop(0, [{"out": twin_crop[k], "scale": shots.spec[k][2]} for k in range(2)])
        run(ctx, 22, 0), run(twin, 22, 0)
        l0, t0 = ctx.launch_count, twin.launch_count
        run(ctx, 1, 22), run(twin, 1, 22)
        assert ctx.launch_count - l0 == twin.launch_count - t0          # no best shot: the same launches
        ctx.tracker_set_best_shot(0, [shots.shot(0), shots.shot(1)])
        T.cuda.synchronize()
        assert all(state_of(shots, k) == bestshot.new_state() for k in range(2))
        assert (host(shots.state[:, 96:]) == 0x77).all()
        assert all((host(i) == 0x33).all() for i in shots.img[0])        # the images are not touched by the setter
        l0, t0 = ctx.launch_count, twin.launch_count
        recs = run(ctx, 1, 23)
        run(twin, 1, 23)
        assert ctx.launch_count - l0 == twin.launch_count - t0 + 2       # two more with a best shot

        def tick(t, ks=(0, 1), frame="face"):
            import make_goldens_params as pg
            now = 1.0e12 + 35.0 * t
            recs = ctx.tracker_feed(list(ks), [pg.make_frame(frame, t, W0, H0)] * len(ks), now, W0, H0)
            T.cuda.synchronize()
            shots.tick(dict(zip(ks, recs)), lambda k: (W0, H0), lambda k: now)
            shots.check(where=t)
            return recs
        shots.tick(dict(enumerate(recs)), lambda k: (W0, H0), lambda k: 1.0e12 + 35.0 * 23)
        shots.check()
        assert shots.mirror[0]["track"] == 1 and shots.mirror[0]["flags"] & bestshot.BEGAN
        for t in range(24, 30):
            tick(t)
        ctx.tracker_set_params(0, [dict()])                              # kept
        tick(30)
        assert shots.mirror[0]["track"] == 1 and shots.mirror[0]["ticks"] > 1
        before = host(shots.state[0]).copy()
        tick(31, ks=(1,))                                                # stream 0 not listed: nothing moves
        assert np.array_equal(host(shots.state[0]), before)
        ctx.tracker_stop(0, 1)                                           # the next tick of a stopped stream ends it
        T.cuda.synchronize()
        shots.check()
        tick(32)
        assert shots.mirror[0]["ended"] == 1 and shots.mirror[0]["flags"] == bestshot.ENDED
        ctx.tracker_start(0, 1)
        for t in range(33, 60):                                         # starter, whitebalance, VJ, then CS again
            tick(t)
        m = shots.mirror[0]
        assert m["track"] >= 2 and m["buffer"] == (m["track"] - 1) % 2 and shots.saved[0][0] is not None
        ctx.tracker_reset(1, 1)
        tick(60)
        assert shots.mirror[1]["ended"] == shots.mirror[1]["track"]      # a tick after reset ends stream 1's track
        ctx.tracker_start(1, 1)
        for t in range(61, 85):
            tick(t)
        open_ = shots.mirror[0]["track"] != shots.mirror[0]["ended"]
        rec = ctx.tracker_export([0, 1])
        ctx.tracker_import([0, 1], rec)                                  # import ends the open tracks
        T.cuda.synchronize()
        for k in range(2):
            bestshot.end(shots.mirror[k])
        shots.check()
        assert open_ and shots.mirror[0]["flags"] == bestshot.ENDED
        tick(85)
        assert shots.mirror[0]["flags"] & bestshot.BEGAN                # the imported tracker begins a new track
        ctx.tracker_set_best_shot(0, [shots.shot(0)])                   # setting again starts from zero
        shots.reset(0)
        T.cuda.synchronize()
        shots.check([0])
        tick(86)
        assert shots.mirror[0]["track"] == 1
        ctx.tracker_set_best_shot(1, [None])                            # removed: stream 1's state stays as it was
        before = host(shots.state[1]).copy()
        tick(87, ks=(0,))
        run(ctx, 2, 88)
        assert np.array_equal(host(shots.state[1]), before)
        ctx.tracker_config()                                             # removes every best shot
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        shots.state.fill_(0x5A)
        for i in shots.img[0]:
            i.fill_(0x5A)
        T.cuda.synchronize()
        run(ctx, 24, 0)
        assert (host(shots.state) == 0x5A).all() and all((host(i) == 0x5A).all() for i in shots.img[0])
        l0 = ctx.launch_count
        run(ctx, 2, 24)
        d0 = ctx.launch_count - l0
        ctx.tracker_set_best_shot(0, [shots.shot(0)])
        ctx.tracker_set_best_shot(0, [None])                             # set and removed: no launch more
        l0 = ctx.launch_count
        run(ctx, 2, 26)
        assert ctx.launch_count - l0 == d0
    finally:
        ctx.close()
        twin.close()


def test_overlap_both_ways_and_rejections():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=4)
    buf = T.zeros((8192,), dtype=T.uint8, device="cuda")
    base = buf.data_ptr()
    L = _lib.lib()

    def setb(recs, first=0):
        arr = (_lib.BestShot * len(recs))(*recs)
        return L.ht_tracker_set_best_shot(ctx._h, first, len(recs), C.addressof(arr))

    def last_error():
        return (L.ht_last_error(ctx._h) or b"").decode()

    def bs(a, b=None, st=None, w=4, h=4, pitch=0, pad=0, scale=1.0):
        return _lib.BestShot((C.c_void_p * 2)(a, b), st, w, h, pitch, pad, scale)
    try:
        assert setb([bs(base, None, base + 4096)]) == HT_ERR_STATE
        ctx.tracker_config()
        assert setb([bs(base, base + 64, base + 4096)]) == 0                 # images [0, 64), [64, 128); state at 4096
        # every other output on a best-shot image or state is refused, naming it
        cam = dict(scaling=1, fixedPosition=(0, 0, 60), lookAt=(0, 0, 0), fov=45, aspect=1.5, near=1, far=1000)
        with pytest.raises(_lib.HtError, match="best-shot state"):
            ctx.tracker_set_camera(1, [dict(cam, out=buf[4096 - 128:4096 + 96])])
        with pytest.raises(_lib.HtError, match="best-shot image"):
            ctx.tracker_set_face_crop(1, [{"out": buf[32:32 + 64].view(4, 4, 4)}])
        with pytest.raises(_lib.HtError, match="best-shot image"):
            ctx.tracker_set_debug(1, [buf[64:128].view(4, 4, 4)])
        with pytest.raises(_lib.HtError, match="best-shot state"):
            ctx.tracker_set_face_tensor(1, [{"out": buf[4100:4112].view(2, 2, 3), "layout": "hwc"}])
        with pytest.raises(_lib.HtError, match="best-shot image"):
            ctx.tracker_set_framing(1, [{"out": buf[120:168]}])
        # and a best shot on another output, or on another best shot
        ctx.tracker_set_face_crop(1, [{"out": buf[1024:1024 + 64].view(4, 4, 4)}])
        assert setb([bs(base + 1024 + 60, None, base + 5000)], 2) == HT_ERR_ARG and "face crop plane" in last_error()
        assert last_error().startswith("record 0: its best-shot image"), last_error()
        assert setb([bs(base + 2048, None, base + 1024 + 8)], 2) == HT_ERR_ARG and "face crop plane" in last_error()
        assert setb([bs(base + 2048, None, base + 4096 + 88)], 2) == HT_ERR_ARG and "best-shot state" in last_error()
        assert setb([bs(base + 2048, base + 2048 + 60, base + 5000)], 2) == HT_ERR_ARG   # its own two images
        assert setb([bs(base + 2048, base + 2048 + 64, base + 5000)], 2) == 0
        # every rejection, with nothing changed
        T.cuda.synchronize()
        before = host(buf).copy()
        host_img, host_state = (C.c_char * 256)(), (C.c_char * 128)()
        ok = dict(a=base + 6144, st=base + 7168)
        for bad, code in ((bs(base + 6146, None, ok["st"]), HT_ERR_ARG), (bs(ok["a"], base + 6146 + 64, ok["st"]), HT_ERR_ARG),
                          (bs(C.addressof(host_img), None, ok["st"]), HT_ERR_ARG),
                          (bs(ok["a"], C.addressof(host_img), ok["st"]), HT_ERR_ARG),
                          (bs(ok["a"], None, None), HT_ERR_ARG), (bs(ok["a"], None, ok["st"] + 4), HT_ERR_ARG),
                          (bs(ok["a"], None, C.addressof(host_state)), HT_ERR_ARG),
                          (bs(ok["a"], None, ok["st"], w=2), HT_ERR_SIZE), (bs(ok["a"], None, ok["st"], h=2), HT_ERR_SIZE),
                          (bs(ok["a"], None, ok["st"], w=2049), HT_ERR_SIZE),
                          (bs(ok["a"], None, ok["st"], pitch=18), HT_ERR_ARG), (bs(ok["a"], None, ok["st"], pitch=12), HT_ERR_ARG),
                          (bs(ok["a"], None, ok["st"], pad=1), HT_ERR_ARG),
                          (bs(ok["a"], None, ok["st"], scale=0.0), HT_ERR_ARG),
                          (bs(ok["a"], None, ok["st"], scale=16.5), HT_ERR_ARG),
                          (bs(ok["a"], None, ok["st"], scale=float("nan")), HT_ERR_ARG)):
            assert setb([bs(None), bad], 2) == code, last_error()
            assert last_error().startswith("record 1:"), last_error()
        assert setb([bs(ok["a"], None, ok["st"])], 4) == HT_ERR_ARG                    # a range past max_frames
        assert L.ht_tracker_set_best_shot(ctx._h, 0, 1, None) == HT_ERR_ARG
        assert L.ht_tracker_set_best_shot(ctx._h, 0, 0, C.addressof((_lib.BestShot * 1)())) == HT_ERR_ARG
        T.cuda.synchronize()
        assert np.array_equal(host(buf), before)
        # the settings in force still tick: stream 0's state is written by a tick, nothing else in buf
        with pytest.raises(ValueError):
            ctx.tracker_set_best_shot(0, [{"out": buf[:64].view(4, 4, 4), "state": buf[4096:4096 + 95]}])
        with pytest.raises(ValueError):
            ctx.tracker_set_best_shot(0, [{"out": (buf[:64].view(4, 4, 4), buf[64:112].view(4, 3, 4)),
                                           "state": buf[4096:4192]}])
    finally:
        ctx.close()
