"""GPU: tracker records - ht_tracker_export / ht_tracker_import, Context.tracker_export / tracker_import and
TrackerSet.snapshot / restore - moving headtrackr.Tracker streams between ids, contexts and GPUs:

  * golden replays (test_gpu_tracker's and test_gpu_feed's mixed batches through step and feed, the params golden
    through feed with per-record canvases, the debug golden) with every stream moved to the other of two contexts
    before every tick, at a fresh permutation of its ids, through host records on even ticks and device records on
    odd ones; the destination context is configured with other parameters, and each debug canvas stays with its id
    on both contexts (so it is only right if the model histogram travelled and import left the canvas in place);
  * a calcAngles change made by set_params on a CS stream, migrated, takes effect at the next hand-off there;
  * 1024 streams of 640x480 video in steady tracking: migrated at a random permutation and swapped within one
    context, every continuation is the unmoved one's, record for record and byte for byte; a clone into an idle id
    too, up to the last bits of its camshift angle;
  * canonical form, host and device records, the host build's check of device records, launch counts, rejections
    (each leaving every stream as it was), and two GPUs when there are two."""
import ctypes as C
from functools import partial

import numpy as np
import pytest

import test_gpu_canvases
import test_gpu_debug
import test_gpu_feed
import test_gpu_tracker
from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_STATE, HtError
from headtrackr_b200.streams import TrackerSet
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)
from test_migrate_host import MODE, N_DIAG, TRACK, bind, reseal

pytestmark = pytest.mark.gpu

R = _lib.TRACKER_RECORD_BYTES
TM_IDLE, TM_STARTING, TM_WB, TM_VJ, TM_CS = range(5)
# what the destination contexts are configured with: every stream's own parameters must travel in its record
OTHER = {"retryDetection": False, "calcAngles": True, "smoothing": False, "fov": 40.0, "cameraOffset": 3.0}


def torch():
    import torch as t
    return t


def modes(recs):
    return np.ascontiguousarray(recs[:, MODE:MODE + 4]).view(np.int32)[:, 0]


class PingPong:
    """TrackerSet's interface over two contexts.  Before every tick (step or feed) all n streams move, with
    TrackerSet.snapshot / restore, to the other context: a second one with more ids, created here.  They land at a
    fresh random permutation of its ids, or at fixed ids per context when the streams have debug canvases (those stay
    with the ids).  Host records on even ticks, device records on odd ones."""
    made = []

    def __init__(self, context, n, params=None, device_events=False):
        other = Context(max_width=context.max_width, max_height=context.max_height, max_frames=context.max_frames + 8)
        plist = list(params) if isinstance(params, (list, tuple)) else [params] * n
        debug = [(p or {}).get("debug") for p in plist]
        self.fixed = any(d is not None for d in debug)
        self.rng = np.random.default_rng(len(PingPong.made))
        self.n, self.sets, self.ids, self.listeners = n, [], [], []
        for c in (context, other):
            ids = [int(i) for i in self.rng.permutation(c.max_frames)[:n]]
            ps = [dict(OTHER) for _ in range(c.max_frames)]
            for k, i in enumerate(ids):
                ps[i] = plist[k] if c is context else dict(OTHER, debug=debug[k])
            ts = TrackerSet(c, c.max_frames, ps, device_events=device_events)
            ts.addEventListener(partial(self._event, len(self.sets)))
            self.sets.append(ts)
            self.ids.append(ids)
        self.other = other
        self.at, self.ticks, self.modes, self.seeds, self.hints = 0, 0, set(), 0, 0
        PingPong.made.append(self)

    def _event(self, s, i, e):
        if s == self.at and i in self.inv():
            for fn in self.listeners:
                fn(self.inv()[i], e)

    def inv(self):
        return {i: k for k, i in enumerate(self.ids[self.at])}

    def _move(self):
        src, dst = self.at, 1 - self.at
        new = self.ids[dst] if self.fixed else [int(i) for i in self.rng.permutation(self.sets[dst].n)[:self.n]]
        snap = self.sets[src].snapshot(self.ids[src], device=self.ticks % 2 == 1)
        recs = snap["records"].cpu().numpy() if self.ticks % 2 else snap["records"]
        m = modes(recs)
        self.modes |= set(int(v) for v in m)
        tobj = np.ascontiguousarray(recs[:, TRACK + 16:TRACK + 32])
        self.seeds += int(((m == TM_CS) & ~tobj.any(axis=1)).sum())          # CS, tracked by no track() yet
        self.hints += int(((m == TM_VJ) & (recs[:, 32 + 8] == 1)).sum())     # VJ with the "hints" timer running
        self.sets[dst].restore(new, snap)
        self.ids[dst], self.at = new, dst
        self.ticks += 1

    @property
    def cur(self):
        return self.sets[self.at]

    def addEventListener(self, fn):
        self.listeners.append(fn)

    def _ks(self, k):
        return range(self.n) if k is None else [k]

    def start(self, k=None):
        for j in self._ks(k):
            self.cur.start(self.ids[self.at][j])
        return True

    def stop(self, k=None):
        for j in self._ks(k):
            self.cur.stop(self.ids[self.at][j])
        return True

    @property
    def status(self):
        return [self.cur.status[i] for i in self.ids[self.at]]

    @property
    def current(self):
        return [self.cur.current[i] for i in self.ids[self.at]]

    def getFOV(self, k):
        return self.cur.getFOV(self.ids[self.at][k])

    def debug_calls(self, k):
        return self.cur.debug_calls(self.ids[self.at][k])

    def step(self, frames, now_ms=None):
        self._move()
        ids = self.ids[self.at]
        if hasattr(frames, "is_cuda"):
            T = torch()
            full = frames.new_zeros((self.cur.n,) + tuple(frames.shape[1:]))
            full[T.tensor(ids, device=frames.device)] = frames
            T.cuda.synchronize()
        else:
            full = np.zeros((self.cur.n,) + frames.shape[1:], np.uint8)
            full[ids] = frames
        recs = self.cur.step(full, now_ms)
        return [recs[i] for i in ids]

    def feed(self, frames, now_ms=None, width=None, height=None):
        self._move()
        ids = self.ids[self.at]

        def remap(v):
            return {ids[k]: x for k, x in v.items()} if isinstance(v, dict) else v
        recs = self.cur.feed(remap(frames), remap(now_ms), remap(width), remap(height))
        return {k: recs[ids[k]] for k in frames}

    def close(self):
        self.other.close()


@pytest.fixture
def pingpong(monkeypatch):
    for mod in (test_gpu_tracker, test_gpu_feed, test_gpu_canvases, test_gpu_debug):
        monkeypatch.setattr(mod, "TrackerSet", PingPong)
    monkeypatch.setattr(PingPong, "made", [])
    yield PingPong.made
    for p in PingPong.made:
        p.close()


def crossed_every_mode(made):
    p = made[0]
    assert p.ticks >= 10 and set(range(5)) <= p.modes and p.seeds > 0, (p.ticks, p.modes, p.seeds)
    return p


@pytest.mark.parametrize("batch", list(test_gpu_tracker.BATCHES))
def test_step_replay_moving_every_stream_before_every_tick(pingpong, batch):
    test_gpu_tracker.replay(batch, "host")
    p = crossed_every_mode(pingpong)
    if batch == "default":
        assert p.hints > 0


@pytest.mark.parametrize("batch", list(test_gpu_tracker.BATCHES))
def test_feed_replay_moving_every_stream_before_every_tick(pingpong, batch):
    test_gpu_feed.replay(batch, "torch-device")
    crossed_every_mode(pingpong)


def test_params_golden_moving_every_stream_before_every_tick(pingpong):
    """per-record canvases and per-stream parameters; both contexts are configured with OTHER"""
    test_gpu_canvases.test_one_context_replays_every_case_with_its_params_and_canvas("numpy-host")
    crossed_every_mode(pingpong)


@pytest.mark.parametrize("path", ["step", "feed"])
def test_debug_golden_moving_every_stream_before_every_tick(pingpong, path):
    """the canvases hash as the reference's: the model histograms travelled, and import left each canvas in place"""
    test_gpu_debug.test_golden_replay(path)
    assert all(p.ticks > 10 for p in pingpong) and pingpong[0].fixed and not pingpong[1].fixed


# ---- 640x480 video on 320x240 canvases --------------------------------------------------------------------------------

VW, VH, CW, CH = 640, 480, 320, 240


def videos():
    """eight 640x480 synth frames whose one face is at least 64 px wide (32 px on the canvas: detectable)"""
    T = torch()
    frames = []
    for i in range(64):
        f, faces = synth.frame(i, VW, VH, n_faces=1, return_faces=True)
        if faces[0][2] >= 64 and len(frames) < 8:
            frames.append(f)
    return T.from_numpy(np.stack(frames)).cuda()


def tick(ctx, ids, logical, base, t):
    """one feed tick of streams ids, id ids[j] on the video of logical stream logical[j] at time t -> records (bytes)"""
    T = torch()
    v = T.roll(base, shifts=(t % 7) - 3, dims=2)          # the faces move sideways from tick to tick
    T.cuda.synchronize()
    out = T.empty(len(ids) * 144, dtype=T.uint8, device="cuda")
    ctx.tracker_feed(list(ids), [v[k % 8] for k in logical], 1.0e12 + 35.0 * t, CW, CH, out=out)
    ctx.sync()
    return out.view(len(ids), 144).cpu().numpy()


EVENT_ANGLE = 40                                           # ht_tracker_event.angle


def same_but_angle(got, want, off, ignore=(0, 0)):
    """A clone runs at another place of the k_track launch than its original (its tier and cluster size follow its
    rank in the launch), which orders camshift's moment sums differently: the fp64 angle then agrees to 1e-9 relative,
    as in every GPU tracker test, and every other byte exactly (ignore: the checksum, which covers the angle)."""
    mask = np.ones(len(got), bool)
    mask[off:off + 8] = False
    mask[ignore[0]:ignore[1]] = False
    diff = np.flatnonzero((got != want) & mask)
    assert diff.size == 0, diff
    g, w = (float(np.ascontiguousarray(x[off:off + 8]).view(np.float64)[0]) for x in (got, want))
    return g == w or abs(g - w) <= 1e-9 * abs(w)


def test_1024_streams_migrate_clone_and_swap(st):
    T = torch()
    N = 1024
    base = videos()
    a = Context(max_width=CW, max_height=CH, max_frames=N + 8)
    b = Context(max_width=CW, max_height=CH, max_frames=N + 64)
    try:
        a.tracker_config(calcAngles=True)
        a.tracker_start(0, N)
        b.tracker_config(**{k: v for k, v in OTHER.items()})
        ids = list(range(N))
        for t in range(24):
            tick(a, ids, ids, base, t)
        recs = a.tracker_export(ids)
        m = modes(recs)
        assert (m == TM_CS).sum() > N // 2, np.bincount(m)
        # canonical form: a dead camshift section is zeros; device and host records agree; the host build accepts them
        assert not recs[m != TM_CS, TRACK:].any() and recs[m == TM_CS, TRACK:].any(axis=1).all()
        dev = T.empty((N, R), dtype=T.uint8, device="cuda")
        a.tracker_export(ids, out=dev)
        a.sync()
        assert np.array_equal(dev.cpu().numpy(), recs)
        bind(st)
        for j in [int(np.flatnonzero(m == v)[0]) for v in set(m.tolist())]:
            assert st.ht_selftest_tracker_check(np.ascontiguousarray(recs[j]).ctypes.data) == 0
        # migrate at a random permutation of b's ids
        perm = [int(i) for i in np.random.default_rng(1).permutation(N + 64)[:N]]
        b.tracker_import(perm, dev)
        assert np.array_equal(b.tracker_export(perm), recs)               # export(import(r)) == r
        for t in range(24, 34):
            assert np.array_equal(tick(a, ids, ids, base, t), tick(b, perm, ids, base, t)), t
        ra = a.tracker_export(ids)
        assert np.array_equal(ra, b.tracker_export(perm))
        cs = modes(ra) == TM_CS
        angles = np.ascontiguousarray(ra[cs, TRACK + 32:TRACK + 40]).view(np.float64)[:, 0]
        assert np.count_nonzero(angles) > cs.sum() // 2                  # calcAngles travelled
        # clone stream c into the idle id N and swap streams s0, s1, within a; b goes on unmoved
        c = int(np.flatnonzero(cs)[3])
        s0, s1 = int(np.flatnonzero(cs)[10]), int(np.flatnonzero(~cs)[0] if (~cs).any() else np.flatnonzero(cs)[11])
        before = a.launch_count
        a.tracker_import([N], a.tracker_export([c]))
        pair = a.tracker_export([s0, s1])
        a.tracker_import([s1, s0], pair)
        assert a.launch_count - before == 6                                # export 1 launch, import 2, each twice
        assert np.array_equal(a.tracker_export([s1, s0]), pair)
        logical = ids + [c]
        logical[s0], logical[s1] = s1, s0
        for t in range(34, 40):
            ra_t = tick(a, ids + [N], logical, base, t)
            rb_t = tick(b, perm, ids, base, t)
            assert np.array_equal(ra_t[:N], rb_t[logical[:N]]), t
            assert same_but_angle(ra_t[N], rb_t[c], EVENT_ANGLE), t
        got = a.tracker_export(ids + [N])
        want = b.tracker_export([perm[k] for k in logical[:N]])
        assert np.array_equal(got[:N], want)
        assert same_but_angle(got[N], b.tracker_export([perm[c]])[0], TRACK + 32, ignore=(16, 24))
    finally:
        a.close()
        b.close()


def test_calc_angles_set_on_a_cs_stream_takes_effect_at_the_next_hand_off_after_migration():
    base = videos()
    ctxs = [Context(max_width=CW, max_height=CH, max_frames=4) for _ in range(3)]
    try:
        moved, ref, unchanged = [TrackerSet(c, 4) for c in ctxs]          # calcAngles off
        for ts in (moved, ref, unchanged):
            ts.start(1)
        for t in range(24):
            for ts in (moved, ref, unchanged):
                ts.feed({1: base[1]}, 1.0e12 + 35.0 * t, CW, CH)
        assert moved.current[1]["detection"] == "CS"
        moved.set_params(1, {"calcAngles": True})
        ref.set_params(1, {"calcAngles": True})
        dest = Context(max_width=CW, max_height=CH, max_frames=8)
        try:
            there = TrackerSet(dest, 8, dict(calcAngles=False))
            there.restore([5], moved.snapshot([1], device=True))
            recs = {"there": [], "ref": [], "unchanged": []}
            for t in range(24, 60):
                if t == 30:                                               # a new hand-off: stop(), start()
                    there.stop(5), ref.stop(1), unchanged.stop(1)
                    there.start(5), ref.start(1), unchanged.start(1)
                recs["there"].append(there.feed({5: base[1]}, 1.0e12 + 35.0 * t, CW, CH)[5])
                recs["ref"].append(ref.feed({1: base[1]}, 1.0e12 + 35.0 * t, CW, CH)[1])
                recs["unchanged"].append(unchanged.feed({1: base[1]}, 1.0e12 + 35.0 * t, CW, CH)[1])
            assert test_gpu_feed.equal_records(recs["there"], recs["ref"])
            angle = [[r["angle"] for r in recs[k] if r["detection"] == "CS"] for k in ("there", "unchanged")]
            assert angle[0][:6] == angle[1][:6]                            # before the hand-off: as before
            assert angle[0][-1] != angle[1][-1] and recs["there"][-1]["detection"] == "CS"
        finally:
            dest.close()
    finally:
        for c in ctxs:
            c.close()


# ---- launches and rejections ------------------------------------------------------------------------------------------

def small_contexts(k, ticks=20, n=4):
    base = videos()
    cs = [Context(max_width=CW, max_height=CH, max_frames=n) for _ in range(k)]
    for c in cs:
        c.tracker_config()
        c.tracker_start(0, n - 1)
    for t in range(ticks):
        for c in cs:
            tick(c, list(range(n)), list(range(n)), base, t)
    return cs, base


def test_launch_counts():
    (x, y), base = small_contexts(2)
    try:
        ids = [0, 1, 2, 3]
        n0 = x.launch_count
        r = x.tracker_export(ids)
        assert x.launch_count - n0 == 1
        x.tracker_import(ids, r)
        assert x.launch_count - n0 == 3
        for t in range(20, 23):
            nx, ny = x.launch_count, y.launch_count
            assert np.array_equal(tick(x, ids, ids, base, t), tick(y, ids, ids, base, t))
            assert x.launch_count - nx == y.launch_count - ny
    finally:
        x.close()
        y.close()


def raw(c, fn, streams, n, records):
    arr = (C.c_int32 * max(1, len(streams)))(*streams) if streams is not None else None
    return getattr(c._L, fn)(c._h, C.addressof(arr) if arr is not None else None, n, records)


def test_rejections_change_nothing():
    T = torch()
    fresh = Context(max_width=CW, max_height=CH, max_frames=4)
    (c,), _ = small_contexts(1)
    try:
        good = c.tracker_export([0, 1, 2, 3])
        assert set(modes(good).tolist()) >= {TM_IDLE, TM_CS}
        buf = np.zeros((4, R), np.uint8)
        for fn in ("ht_tracker_export", "ht_tracker_import"):
            assert raw(fresh, fn, [0], 1, buf.ctypes.data) == HT_ERR_STATE
        with pytest.raises(HtError) as e:
            fresh.tracker_import([0], good[:1])
        assert e.value.code == HT_ERR_STATE

        def bad_record(off, value, dtype, seal=True):
            r = good.copy()
            r[1, off:off + np.dtype(dtype).itemsize] = np.frombuffer(np.array(value, dtype).tobytes(), np.uint8)
            if seal:
                r[1] = reseal(r[1])
            return r
        flipped = good.copy()
        flipped[1, 5000] ^= 0x10
        dev = T.from_numpy(good.copy()).cuda()
        T.cuda.synchronize()
        misaligned = T.zeros(4 * R + 16, dtype=T.uint8, device="cuda")[4:4 + 4 * R]
        calls = [
            ("ht_tracker_export", [0, 0], 2, buf.ctypes.data), ("ht_tracker_import", [0, 0], 2, good.ctypes.data),
            ("ht_tracker_export", [4], 1, buf.ctypes.data), ("ht_tracker_import", [-1], 1, good.ctypes.data),
            ("ht_tracker_export", [0], 0, buf.ctypes.data), ("ht_tracker_import", [0, 1, 2, 3, 0], 5, good.ctypes.data),
            ("ht_tracker_export", None, 1, buf.ctypes.data), ("ht_tracker_import", [0], 1, None),
            ("ht_tracker_export", [0], 1, None), ("ht_tracker_import", None, 1, good.ctypes.data),
            ("ht_tracker_export", [0], 1, misaligned.data_ptr()), ("ht_tracker_import", [0], 1, misaligned.data_ptr()),
        ]
        for r in (flipped, bad_record(0, 0x31525449, "<u4", False), bad_record(4, 2, "<u4", False),
                  bad_record(MODE, 7, "<i4"), bad_record(N_DIAG, -1, "<i4"), bad_record(MODE + 4, 16, "<i4")):
            calls.append(("ht_tracker_import", [3, 2, 1, 0], 4, r.ctypes.data))
        dev_bad = T.from_numpy(bad_record(N_DIAG, 7, "<i4")).cuda()
        T.cuda.synchronize()
        calls.append(("ht_tracker_import", [3, 2, 1, 0], 4, dev_bad.data_ptr()))
        ids_dev = T.tensor([0], dtype=T.int32, device="cuda")
        assert c._L.ht_tracker_import(c._h, ids_dev.data_ptr(), 1, dev.data_ptr()) == HT_ERR_ARG
        if T.cuda.device_count() >= 2:
            other = T.from_numpy(good.copy()).to("cuda:1")
            T.cuda.synchronize("cuda:1")
            calls += [("ht_tracker_export", [0], 1, other.data_ptr()), ("ht_tracker_import", [0], 1, other.data_ptr())]
        for fn, s, n, p in calls:
            assert raw(c, fn, s, n, p) == HT_ERR_ARG, (fn, s, n)
            assert np.array_equal(c.tracker_export([0, 1, 2, 3]), good), (fn, s, n)
        assert raw(c, "ht_tracker_import", [3, 2, 1, 0], 4, dev_bad.data_ptr()) == HT_ERR_ARG
        msg = c._L.ht_last_error(c._h).decode()
        assert msg.startswith("record 1:") and "head diagonal" in msg, msg
        with pytest.raises(HtError):
            c.tracker_import([0, 1, 2, 3], bad_record(MODE, 9, "<i4"))
        c.tracker_import([3, 2, 1, 0], dev)                                # the same records, well formed
        assert np.array_equal(c.tracker_export([3, 2, 1, 0]), good)
    finally:
        c.close()
        fresh.close()


def test_two_gpus_snapshot_restore():
    T = torch()
    if T.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    N = 256
    base0 = videos()
    base1 = base0.to("cuda:1")
    c0, c1, ref = (Context(max_width=CW, max_height=CH, max_frames=N, device=d) for d in (0, 1, 0))
    try:
        s0, s1, sr = TrackerSet(c0, N, {"calcAngles": True}), TrackerSet(c1, N), TrackerSet(ref, N, {"calcAngles": True})
        s0.start(), sr.start()

        def vids(base, t):
            v = T.roll(base, shifts=(t % 7) - 3, dims=2)
            T.cuda.synchronize(base.device)
            return {k: v[k % 8] for k in range(N)}
        for t in range(24):
            s0.feed(vids(base0, t), 1.0e12 + 35.0 * t, CW, CH)
            sr.feed(vids(base0, t), 1.0e12 + 35.0 * t, CW, CH)
        perm = [int(i) for i in np.random.default_rng(2).permutation(N)]
        s1.restore(perm, s0.snapshot(range(N), device=True))
        for t in range(24, 34):
            got = s1.feed({perm[k]: v for k, v in vids(base1, t).items()}, 1.0e12 + 35.0 * t, CW, CH)
            want = sr.feed(vids(base0, t), 1.0e12 + 35.0 * t, CW, CH)
            assert test_gpu_feed.equal_records([got[perm[k]] for k in range(N)], [want[k] for k in range(N)]), t
            assert [s1.status[perm[k]] for k in range(N)] == sr.status
        assert np.array_equal(c1.tracker_export(perm), ref.tracker_export(range(N)))
    finally:
        for c in (c0, c1, ref):
            c.close()
