"""GPU: video drawn through views (ht_tracker_feed_views, ht_tracker_feed_yuv_views, ht_ingest_views,
ht_ingest_yuv_views; DESIGN.md 2, "Views").

  * the ingest entry points equal hto_draw_image of the numpy-oriented oracle frame for every orientation, format and
    crop, host and device frames, planes carved from one allocation at odd offsets and pitches, and through both thread
    layouts of k_feed_draw_view (upright and transposed views);
  * exact twins of the golden replays: one context feeds V = orient^-1(F) through view o, the other the upright video
    F; records and debug canvases are equal on every tick, with orientations changing every tick and view ticks
    alternating with plain ones; crops of F embedded in a larger frame around which another face sits;
  * four streams cropping one device mosaic equal four plain feeds;
  * 1024 streams of sensor-oriented 1280x720 NV12 rotated onto portrait canvases of four sizes;
  * the identity view is the plain entry points byte for byte, and a view tick launches what a plain tick launches;
  * a sensor-oriented stream that finds no face upright finds and tracks it through its rotation;
  * every rejection names its record, launches nothing and leaves every stream as it was."""
import ctypes as C

import numpy as np
import pytest

import oracle
from headtrackr_b200 import Context, _lib, synth, views
from headtrackr_b200._lib import HT_ERR_ARG, HT_OK
from headtrackr_b200.context import tracker_events_from_bytes
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, debug_canvas
from test_debug_host import make_frame as frame_debug
from test_formats_host import NEW, RGB, fo, oracle_convert, random_frame  # noqa: F401
from test_gpu_canvases import STREAMS, black, canvas_of, make_frame, spec_of
from test_gpu_feed import equal_records, video
from test_gpu_formats import api_frame, carve, from_rgba

pytestmark = pytest.mark.gpu

ALL = ["nv12", "i420"] + NEW


def torch():
    import torch as t
    return t


def orient(a, o):
    r = np.rot90(a, -(o & 3))
    return np.ascontiguousarray(np.fliplr(r) if o & 4 else r)


def unorient(a, o):
    """V with orient(V, o) == a"""
    return np.ascontiguousarray(np.rot90(np.fliplr(a) if o & 4 else a, o & 3))


def view(o, crop=None):
    return {"rotate": 90 * (o & 3), "mirror": bool(o & 4), "crop": crop}


def oracle_view(rgba, o, crop, dw, dh):
    O = orient(rgba, o)
    sx, sy, sw, sh = crop or (0, 0, O.shape[1], O.shape[0])
    out = np.zeros((dh, dw, 4), np.uint8)
    for c in range(4):
        out[..., c] = oracle.draw_image(np.ascontiguousarray(O[..., c]), sx, sy, sw, sh, dw, dh, dw, dh)
    return out


def dev(a):
    return torch().from_numpy(np.ascontiguousarray(a)).cuda()


# ---- ingest ---------------------------------------------------------------------------------------------------------

def crops_of(W, H):
    return [None, (1, 2, W - 3, H - 5), (0, 0, 1, 1), (W - 1, 0, 1, H), (0, H - 1, W, 1), (W // 3, H // 4, W // 2, H // 2)]


@pytest.mark.parametrize("fmt", ALL)
def test_ingest_yuv_views_equal_the_oracle(fo, fmt):
    T = torch()
    rng = np.random.default_rng(len(fmt) * 5 + 1)
    color = "bt601" if fmt in RGB else ("bt709" if fmt != "p010" else "bt2020")
    c = Context(max_width=640, max_height=480, max_frames=4)
    try:
        for (w, h) in ((97, 61), (320, 180)):
            f = random_frame(rng, fmt, w, h)
            rgba = oracle_convert(fo, f, color)
            buf, where = carve(f, rng)
            cf = (f[0], f[1], f[2], tuple(buf[r:r + s[0], o:o + s[1]] for r, o, s in where))
            for o in range(8):
                W, H = (h, w) if o & 1 else (w, h)
                for crop in crops_of(W, H)[o % 2::2] + [None]:
                    sw, sh = (crop[2], crop[3]) if crop else (W, H)
                    # 1:1, down-scaled, up-scaled; widths off a multiple of 4 take the scalar stores
                    for dw, dh in {(sw, sh), (max(1, sw // 3), max(1, sh // 2)), (min(640, 2 * sw + 3), min(480, sh + 7))}:
                        want = oracle_view(rgba, o, crop, dw, dh)
                        got = c.ingest_yuv([api_frame(cf, False)], dw, dh, fmt, color, view=view(o, crop))
                        assert np.array_equal(got[0], want), (fmt, w, o, crop, dw, dh)
                        out = T.zeros((1, dh, dw, 4), dtype=T.uint8, device="cuda")
                        c.ingest_yuv([api_frame(cf, True)], dw, dh, fmt, color, out=out, view=view(o, crop))
                        c.sync()
                        assert np.array_equal(out[0].cpu().numpy(), want), (fmt, w, o, crop, dw, dh, "device")
    finally:
        c.close()


def test_ingest_views_rgba_and_one_call_of_every_orientation():
    T = torch()
    rng = np.random.default_rng(7)
    frames = [rng.integers(0, 256, (h, w, 4), dtype=np.uint8) for w, h in ((1280, 720), (641, 481), (33, 17), (1, 9))]
    c = Context(max_width=320, max_height=320, max_frames=4)
    try:
        recs, vs = [], []
        for i in range(16):
            f, o = frames[i % 4], i % 8
            W, H = (f.shape[0], f.shape[1]) if o & 1 else (f.shape[1], f.shape[0])
            crop = None if i % 3 == 0 else crops_of(W, H)[1 + i % 5] if min(W, H) > 6 else (0, 0, W, H)
            recs.append(f)
            vs.append(view(o, crop))
        for dw, dh in ((320, 240), (240, 320), (65, 33)):
            want = np.stack([oracle_view(f, views.orientation(v), v["crop"], dw, dh) for f, v in zip(recs, vs)])
            # host frames with padded rows, host destination
            padded = [video(f, 1, True) for f in recs]
            assert np.array_equal(c.ingest(padded, dw, dh, view=vs), want), (dw, dh)
            out = T.zeros((len(recs), dh, dw, 4), dtype=T.uint8, device="cuda")
            before = c.launch_count
            c.ingest([dev(f) for f in recs], dw, dh, out=out, view=vs)
            assert c.launch_count - before == 1
            c.sync()
            assert np.array_equal(out.cpu().numpy(), want), (dw, dh)
            # the identity view is ht_ingest
            same = [r for r in recs if r.shape == recs[0].shape]
            assert np.array_equal(c.ingest(same, dw, dh, view=None), c.ingest(same, dw, dh, view=view(0)))
    finally:
        c.close()


# ---- golden replays through views -----------------------------------------------------------------------------------

def embed(F, other, o):
    """F placed in a larger frame filled with the face frame `other`, at an offset -> (the frame, the crop of F in the
    frame's orientation-o coordinates, the video V = orient^-1(frame))"""
    h, w = F.shape[:2]
    reps = (-(-(h + 37) // other.shape[0]), -(-(w + 23) // other.shape[1]), 1)
    E = np.ascontiguousarray(np.tile(other, reps)[:h + 37, :w + 23])
    E[19:19 + h, 11:11 + w] = F
    return (11, 19, w, h), unorient(E, o)


@pytest.mark.parametrize("mode", ["rgba-host", "nv12-device", "crop-device"])
def test_golden_cases_view_tick_equals_upright_tick(fo, mode):
    n = len(STREAMS)
    params = [s[0]["params"] if isinstance(s[0], dict) else {} for s in STREAMS]
    canvases = [canvas_of(s[0]) if isinstance(s[0], dict) else s[1] for s in STREAMS]
    specs = [spec_of(s[0]) if isinstance(s[0], dict) else (None, 1000.0) for s in STREAMS]
    device = mode != "rgba-host"
    rng = np.random.default_rng(61)
    other = synth.frame(5, 200, 160, n_faces=1)
    ca = Context(max_width=200, max_height=160, max_frames=32)
    cb = Context(max_width=200, max_height=160, max_frames=32)
    try:
        ta, tb = TrackerSet(ca, n, params), TrackerSet(cb, n, params)
        pos = [0] * n
        offset = [1.0e12 + 7919.0 * k for k in range(n)]
        seen, orients = set(), set()

        def finished(k):
            return not isinstance(STREAMS[k][0], dict) or pos[k] - STREAMS[k][1] >= len(specs[k][0])

        call = 0
        while not all(finished(k) for k in range(n)) or call < 12:
            chosen = [k for k in range(n) if rng.random() < 0.6] or [int(rng.integers(n))]
            rng.shuffle(chosen)
            listed, va, vb, clocks, vws = [], {}, {}, {}, {}
            plain = call % 3 == 2                   # every third tick feeds the upright video without a view
            for k in chosen:
                s, first = STREAMS[k]
                f = black(*canvases[k])
                if s == "black" and pos[k] == 0:
                    ta.start(k), tb.start(k)
                j = pos[k] - first if isinstance(s, dict) else -1
                if isinstance(s, dict) and 0 <= j < len(specs[k][0]):
                    action, kind, tt = specs[k][0][j]
                    if action == "start":
                        ta.start(k), tb.start(k)
                    if action == "stop":
                        ta.stop(k), tb.stop(k)
                        continue
                    f = make_frame(s, kind, tt)
                listed.append(k)
                clocks[k] = offset[k] + specs[k][1] * (pos[k] + 1)
                F = video(f, 1 + k % 3, False)
                o = (k + call) % 8
                orients.add(o)
                if plain:
                    va[k], vb[k], vws[k] = F, F, view(0)
                elif mode == "rgba-host":
                    va[k], vb[k], vws[k] = unorient(F, o), F, view(o)
                elif mode == "nv12-device":
                    V = unorient(F, o)
                    yf = from_rgba(V, "nv12", rng)
                    va[k], vb[k], vws[k] = api_frame(yf, True), dev(orient(oracle_convert(fo, yf, "bt601"), o)), view(o)
                else:
                    crop, V = embed(F, other, o)
                    va[k], vb[k], vws[k] = dev(V), dev(F), view(o, crop)
            if listed:
                if device:
                    torch().cuda.synchronize()
                cw = {k: canvases[k][0] for k in listed}
                chh = {k: canvases[k][1] for k in listed}
                want = tb.feed(vb, now_ms=clocks, width=cw, height=chh)
                if mode == "nv12-device" and not plain:
                    got = ta.feed_yuv(va, now_ms=clocks, width=cw, height=chh, format="nv12", view=vws)
                else:
                    got = ta.feed(va, now_ms=clocks, width=cw, height=chh, view=vws)
                for k in listed:
                    assert equal_records(got[k], want[k]), (mode, call, k, vws[k], got[k], want[k])
                    assert ta.status[k] == tb.status[k], (mode, call, k)
                    seen.add(want[k]["detection"])
            for k in chosen:
                s, first = STREAMS[k]
                if isinstance(s, dict) and pos[k] - first == len(specs[k][0]) - 1:
                    ta.stop(k), tb.stop(k)
                pos[k] += 1
            call += 1
            assert call < 2000
        assert {"WB", "VJ", "CS"} <= seen, seen
        assert orients == set(range(8))
    finally:
        ca.close()
        cb.close()


def test_debug_cases_view_tick_equals_upright_tick_with_debug_canvases(fo):
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    W0, H0 = GOLD_D["width"], GOLD_D["height"]
    rng = np.random.default_rng(67)
    ca = Context(max_width=W0, max_height=H0, max_frames=8)
    cb = Context(max_width=W0, max_height=H0, max_frames=8)
    try:
        da = [T.from_numpy(debug_canvas(case)).cuda() for case in cases]
        db = [d.clone() for d in da]
        ta = TrackerSet(ca, n, [dict(case["params"], debug=da[k]) for k, case in enumerate(cases)])
        tb = TrackerSet(cb, n, [dict(case["params"], debug=db[k]) for k, case in enumerate(cases)])
        T.cuda.synchronize()
        clock, cs = 1.0e12, 0
        for i in range(max(len(case["steps"]) for case in cases)):
            clock += 35.0
            listed, va, vb, vws = [], {}, {}, {}
            for k, case in enumerate(cases):
                f = black(W0, H0)
                if i < len(case["steps"]):
                    s = case["steps"][i]
                    f = frame_debug(*s["frame"])
                    if s["action"] == "start":
                        ta.start(k), tb.start(k)
                    elif s["action"] == "stop":
                        ta.stop(k), tb.stop(k)
                    if s["action"] != "stop":
                        listed.append(k)
                elif i == len(case["steps"]):
                    ta.stop(k), tb.stop(k)
                o = (k + i) % 8
                yf = from_rgba(unorient(f, o), "i420", rng)
                va[k], vb[k], vws[k] = api_frame(yf, True), dev(orient(oracle_convert(fo, yf, "bt709"), o)), view(o)
            if not listed:
                continue
            T.cuda.synchronize()
            got = ta.feed_yuv({k: va[k] for k in listed}, clock, W0, H0, "i420", "bt709", view={k: vws[k] for k in listed})
            want = tb.feed({k: vb[k] for k in listed}, clock, W0, H0)
            assert equal_records(got, want), i
            cs += sum(want[k]["detection"] == "CS" for k in listed)
            for k in range(n):
                assert T.equal(da[k], db[k]), (i, k)
        assert cs > 0
    finally:
        ca.close()
        cb.close()


def test_mosaic_of_four_golden_videos_equals_four_plain_feeds():
    T = torch()
    cases = GOLD_D["cases"][:4]
    W0, H0 = GOLD_D["width"], GOLD_D["height"]
    ca = Context(max_width=W0, max_height=H0, max_frames=4)
    cb = Context(max_width=W0, max_height=H0, max_frames=4)
    try:
        ta = TrackerSet(ca, 4, [case["params"] for case in cases])
        tb = TrackerSet(cb, 4, [case["params"] for case in cases])
        clock, seen = 1.0e12, set()
        for i in range(max(len(case["steps"]) for case in cases)):
            clock += 35.0
            tiles, listed = [], []
            for k, case in enumerate(cases):
                f = black(W0, H0)
                if i < len(case["steps"]):
                    s = case["steps"][i]
                    f = frame_debug(*s["frame"])
                    if s["action"] == "start":
                        ta.start(k), tb.start(k)
                    elif s["action"] == "stop":
                        ta.stop(k), tb.stop(k)
                    if s["action"] != "stop":
                        listed.append(k)
                tiles.append(f)
            if not listed:
                continue
            mosaic = dev(np.concatenate([np.concatenate(tiles[:2], 1), np.concatenate(tiles[2:], 1)], 0))
            crops = {k: ((k % 2) * W0, (k // 2) * H0, W0, H0) for k in range(4)}
            T.cuda.synchronize()
            got = ta.feed({k: mosaic for k in listed}, clock, W0, H0, view={k: view(0, crops[k]) for k in listed})
            want = tb.feed({k: dev(tiles[k]) for k in listed}, clock, W0, H0)
            assert equal_records(got, want), i
            seen |= {want[k]["detection"] for k in listed}
        assert "CS" in seen, seen
    finally:
        ca.close()
        cb.close()


# ---- at scale -------------------------------------------------------------------------------------------------------

def test_1024_streams_of_sensor_oriented_1280x720_nv12(fo):
    T = torch()
    N = 1024
    rng = np.random.default_rng(71)
    pairs = []
    for i, o in enumerate((1, 3, 5, 7)):                  # a portrait scene in sensor orientation, 1280 x 720
        F = synth.frame(900 + i, 720, 1280, n_faces=1)
        yf = from_rgba(unorient(F, o), "nv12", rng)
        pairs.append((api_frame(yf, True), dev(orient(oracle_convert(fo, yf, "bt601"), o)), view(o)))
    T.cuda.synchronize()
    ca = Context(max_width=360, max_height=640, max_frames=N)
    cb = Context(max_width=360, max_height=640, max_frames=N)
    try:
        for x in (ca, cb):
            x.tracker_config(calcAngles=True)
            x.tracker_reset(0, N)
            x.tracker_start(0, N)
        modes = set()
        mix = [(240, 320), (180, 320), (120, 160), (360, 640)]
        for tick in range(20):
            ks = list(range(N)) if tick < 10 else sorted(rng.choice(N, N - 100, replace=False).tolist())
            rng.shuffle(ks)
            if tick < 10:
                w, h = 240, 320
            else:
                w = [mix[(k + tick) % 4][0] for k in ks]
                h = [mix[(k + tick) % 4][1] for k in ks]
            now = 1.0e12 + 35.0 * tick
            oa = T.empty(len(ks) * 144, dtype=T.uint8, device="cuda")
            ob = T.empty(len(ks) * 144, dtype=T.uint8, device="cuda")
            sel = [pairs[k % 4] for k in ks]
            ca.tracker_feed_yuv(ks, [p[0] for p in sel], now, w, h, out=oa, view=[p[2] for p in sel])
            cb.tracker_feed(ks, [p[1] for p in sel], now, w, h, out=ob)
            ca.sync(), cb.sync()
            a, b = oa.cpu().numpy(), ob.cpu().numpy()
            assert np.array_equal(a, b), tick
            modes |= {r["detection"] for r in tracker_events_from_bytes(a.tobytes())}
        assert {"WB", "VJ", "CS"} <= modes, modes
    finally:
        ca.close()
        cb.close()


def test_identity_view_and_launches_equal_the_plain_entry_points(fo):
    f = synth.frame(11, 320, 240, n_faces=1)
    rng = np.random.default_rng(73)
    yf = from_rgba(f, "nv12", rng)
    rgba = oracle_convert(fo, yf, "bt601")
    T = torch()
    dy, dr = api_frame(yf, True), dev(rgba)
    T.cuda.synchronize()
    cs = [Context(max_width=320, max_height=240, max_frames=4) for _ in range(4)]
    try:
        for x in cs:
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        for t in range(30):
            ks = [3, 0, 2] if t % 3 else [1, 2, 0, 3]
            w, h = (320, 240) if t % 2 else ([320, 160, 200, 160][:len(ks)], [240, 120, 150, 120][:len(ks)])
            o = t % 8
            V = unorient(rgba, o)
            outs, launches = [], []
            for x, call in zip(cs, (
                    lambda x: x.tracker_feed(ks, [dr] * len(ks), 1.0e12 + 35.0 * t, w, h, out=outs[-1]),
                    lambda x: x.tracker_feed(ks, [dr] * len(ks), 1.0e12 + 35.0 * t, w, h, out=outs[-1], view=view(0)),
                    lambda x: x.tracker_feed_yuv(ks, [dy] * len(ks), 1.0e12 + 35.0 * t, w, h, out=outs[-1], view=view(0)),
                    lambda x: x.tracker_feed(ks, [dev(V)] * len(ks), 1.0e12 + 35.0 * t, w, h, out=outs[-1], view=view(o)))):
                outs.append(T.empty(len(ks) * 144, dtype=T.uint8, device="cuda"))
                T.cuda.synchronize()
                before = x.launch_count
                call(x)
                x.sync()
                launches.append(x.launch_count - before)
            assert len(set(launches)) == 1 and launches[0] > 0, (t, launches)
            for i in range(1, 4):
                assert T.equal(outs[i], outs[0]), (t, i)
    finally:
        for x in cs:
            x.close()


def test_sensor_oriented_stream_is_found_only_through_its_rotation(fo):
    """portrait faces in sensor orientation (a quarter turn in memory, either way), one per stream: through their
    rotation every stream has the events of its upright twin on every tick, and some stream whose face the cascade
    never finds through ht_tracker_feed_yuv on the landscape canvas of the video (it only finds upright faces, whatever
    the reason it misses a given one) is found and tracked through its rotation"""
    K = 8
    rng = np.random.default_rng(79)
    frames, twins, vws = {}, {}, {}
    for k in range(K):
        F = synth.frame(31 + k, 240, 320, n_faces=1)
        o = 1 if k % 2 == 0 else 3
        yf = from_rgba(unorient(F, o), "nv12", rng)      # 320 x 240 in memory, shown upright by a quarter turn
        frames[k], twins[k], vws[k] = api_frame(yf, False), orient(oracle_convert(fo, yf, "bt601"), o), view(o)
    cs = [Context(max_width=320, max_height=320, max_frames=K) for _ in range(3)]
    try:
        sets = [TrackerSet(x, K, [{}] * K) for x in cs]
        for s in sets:
            s.start()
        seen_plain, seen_view = [set() for _ in range(K)], [set() for _ in range(K)]
        for t in range(40):
            now = 1.0e12 + 35.0 * t
            plain = sets[0].feed_yuv(frames, now, 320, 240)
            got = sets[1].feed_yuv(frames, now, 240, 320, view=vws)
            want = sets[2].feed(twins, now, 240, 320)
            assert equal_records(got, want), t
            for k in range(K):
                seen_plain[k].add(plain[k]["detection"])
                seen_view[k].add(got[k]["detection"])
        found_by_view_only = [k for k in range(K) if "CS" not in seen_plain[k] and "CS" in seen_view[k]]
        assert found_by_view_only, (seen_plain, seen_view)
    finally:
        for x in cs:
            x.close()


# ---- rejections -----------------------------------------------------------------------------------------------------

def test_rejections_name_the_record_and_change_nothing():
    T = torch()
    MAXF = 4
    rng = np.random.default_rng(83)
    f = dev(synth.frame(9, 320, 240, n_faces=1))
    yf = tuple(dev(p) for p in random_frame(rng, "nv12", 320, 240)[3])
    T.cuda.synchronize()
    c = Context(max_width=320, max_height=240, max_frames=MAXF)
    try:
        c.tracker_config(calcAngles=True)
        c.tracker_reset(0, MAXF)
        c.tracker_start(0, MAXF)
        for t in range(12):
            c.tracker_feed(list(range(MAXF)), [f] * MAXF, 1.0e12 + 35.0 * t, 160, 120, view=view(1))
        before = c.tracker_export(list(range(MAXF)))
        launches = c.launch_count
        vf = _lib.VideoFrame(f.data_ptr(), 0, 320, 240, 0, 1.0e12)
        img = _lib.YuvImage((C.c_void_p * 3)(yf[0].data_ptr(), yf[1].data_ptr(), None), (C.c_int32 * 3)(0, 0, 0), 320, 240,
                            0, 0)

        def V(o, crop=(0, 0, 0, 0), reserved=(0, 0, 0)):
            return _lib.VideoView(o, *crop, (C.c_int32 * 3)(*reserved))
        bad = [V(8), V(-1), V(0, reserved=(0, 1, 0)), V(0, (0, 0, 0, 5)), V(0, (-1, 0, 4, 4)), V(0, (300, 0, 21, 4)),
               V(1, (0, 0, 241, 4)), V(3, (0, 300, 4, 21)), V(0, (0, 0, 320, 241))]
        out = (_lib.TrackerEvent * 2)()
        for i, bv in enumerate(bad):
            vs = (_lib.VideoView * 2)(V(0), bv)
            crecs = (_lib.CanvasFrame * 2)(_lib.CanvasFrame(vf, 160, 120), _lib.CanvasFrame(
                _lib.VideoFrame(f.data_ptr(), 1, 320, 240, 0, 1.0e12), 160, 120))
            rc = c._L.ht_tracker_feed_views(c._h, C.addressof(crecs), C.addressof(vs), 2, 1, C.addressof(out))
            msg = c._L.ht_last_error(c._h).decode()
            assert rc == HT_ERR_ARG and msg.startswith("record 1:"), (i, rc, msg)
            yrecs = (_lib.YuvFrame * 2)(_lib.YuvFrame(img, 0, 160, 120, 0, 1.0e12), _lib.YuvFrame(img, 1, 160, 120, 0, 1.0e12))
            rc = c._L.ht_tracker_feed_yuv_views(c._h, C.addressof(yrecs), C.addressof(vs), 2, 1, C.addressof(out))
            msg = c._L.ht_last_error(c._h).decode()
            assert rc == HT_ERR_ARG and msg.startswith("record 1:"), (i, rc, msg)
            dst = np.zeros((2, 120, 160, 4), np.uint8)
            frames = (_lib.VideoFrame * 2)(vf, vf)
            assert c._L.ht_ingest_views(c._h, C.addressof(frames), C.addressof(vs), 2, 1, dst.ctypes.data, 160, 120) == HT_ERR_ARG
            imgs = (_lib.YuvImage * 2)(img, img)
            assert c._L.ht_ingest_yuv_views(c._h, C.addressof(imgs), C.addressof(vs), 2, 1, dst.ctypes.data, 160, 120) == HT_ERR_ARG
            assert not dst.any()
        crecs = (_lib.CanvasFrame * 1)(_lib.CanvasFrame(vf, 160, 120))
        assert c._L.ht_tracker_feed_views(c._h, C.addressof(crecs), None, 1, 1, C.addressof(out)) == HT_ERR_ARG
        assert "views" in c._L.ht_last_error(c._h).decode()
        assert c.launch_count == launches
        assert np.array_equal(c.tracker_export(list(range(MAXF))), before)
        vs = (_lib.VideoView * 1)(V(7, (10, 20, 100, 200)))
        assert c._L.ht_tracker_feed_views(c._h, C.addressof(crecs), C.addressof(vs), 1, 1, C.addressof(out)) == HT_OK
    finally:
        c.close()
