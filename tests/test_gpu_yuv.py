"""GPU: YUV 4:2:0 video into the tracker (ht_tracker_feed_yuv) and onto canvases (ht_ingest_yuv).

  * ht_ingest_yuv equals hto_draw_image(hto_yuv_to_rgba(frame)) bit for bit: NV12 and I420, every colour space, odd
    and even sizes, 1:1 and scaled, host and device planes (also slices of one larger allocation at odd offsets and
    pitches), host and device destinations;
  * composition: for every case the golden replays of ht_tracker_feed_canvases cover (reference_js_lifecycle, _main,
    _params, _debug), a context ticked with ht_tracker_feed_yuv on YUV video gives exactly the records (and debug
    canvases) of a context ticked with ht_tracker_feed_canvases on hto_yuv_to_rgba of that video - same subsets, clocks,
    canvases and parameters - also when the streams of one context alternate between YUV and RGBA ticks;
  * 1024 streams of 1280x720 NV12 device video, on one canvas size and on four: the same, byte for byte;
  * a YUV tick launches what an RGBA tick of the same layout launches;
  * every rejection names its record and leaves every stream as it was."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_OK
from headtrackr_b200.context import tracker_events_from_bytes
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, debug_canvas
from test_debug_host import make_frame as frame_debug
from test_gpu_canvases import STREAMS, black, canvas_of, make_frame, spec_of
from test_gpu_feed import equal_records, video
from test_yuv_host import (COLORS, SIZES, oracle_convert, oracle_draw, padded_plane, random_frame,  # noqa: F401
                           yo)

pytestmark = pytest.mark.gpu


def torch():
    import torch as t
    return t


def forward(rgba, fmt):
    """test-local RGB -> BT.601 limited-range YUV 4:2:0 (chroma: the mean of each 2 x 2 block), as numpy planes"""
    rgb = rgba[..., :3].astype(np.float64)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    y = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
    u = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
    v = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
    h, w = y.shape

    def sub(c):
        c = np.pad(c, ((0, h % 2), (0, w % 2)), mode="edge")
        return (c[0::2, 0::2] + c[1::2, 0::2] + c[0::2, 1::2] + c[1::2, 1::2]) / 4

    q = [np.clip(np.floor(p + 0.5), 0, 255).astype(np.uint8) for p in (y, sub(u), sub(v))]
    if fmt == "nv12":
        uv = np.empty((q[1].shape[0], 2 * q[1].shape[1]), np.uint8)
        uv[:, 0::2], uv[:, 1::2] = q[1], q[2]
        return (q[0], uv)
    return tuple(q)


def on_device(frame):
    """the planes as CUDA tensors; a row-padded plane (padded_plane) keeps its pitch"""
    T = torch()
    out = []
    for p in frame:
        if p.strides[0] != p.shape[1] and p.base is not None and p.base.ndim == 2:
            out.append(T.from_numpy(np.ascontiguousarray(p.base)).cuda()[:, :p.shape[1]])
        else:
            out.append(T.from_numpy(np.ascontiguousarray(p)).cuda())
    return tuple(out)


def stream_format(k):
    return ("nv12", "i420")[k % 2]


def stream_color(k):
    return "bt709-full" if k % 5 == 3 else "bt601"


# ---- ht_ingest_yuv --------------------------------------------------------------------------------------------------

def carve(frame, rng):
    """the planes of `frame` copied into one larger buffer at odd offsets, each with an odd pitch: slices of it"""
    rows = sum(p.shape[0] for p in frame)
    width = (max(p.shape[1] for p in frame) + 7) | 1     # an odd pitch
    buf = rng.integers(0, 256, (rows + 2, width), dtype=np.uint8)
    out, r = [], 1
    for i, p in enumerate(frame):
        off = 1 + 2 * i                                    # odd column offsets
        buf[r:r + p.shape[0], off:off + p.shape[1]] = p
        out.append((r, off, p.shape))
        r += p.shape[0]
    return buf, out


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
def test_ingest_yuv_equals_the_oracle(yo, fmt):
    T = torch()
    rng = np.random.default_rng(3)
    c = Context(max_width=1280, max_height=720, max_frames=4)
    try:
        for (w, h) in SIZES:
            for ci, color in enumerate(COLORS):
                f = random_frame(rng, w, h, fmt, [(0, 0, 0), (3, 1, 5), (1, 7, 2), (8, 4, 4)][ci])
                rgba = oracle_convert(yo, f, fmt, color)
                for dw, dh in {(w, h), (160, 120), (33, 17)}:
                    want = oracle_draw(rgba, dw, dh)
                    assert np.array_equal(c.ingest_yuv([f], dw, dh, fmt, color)[0], want), (w, h, color, dw, dh)
                    fd = on_device(f)
                    out = T.zeros((1, dh, dw, 4), dtype=T.uint8, device="cuda")
                    c.ingest_yuv([fd], dw, dh, fmt, color, out=out)
                    assert np.array_equal(out[0].cpu().numpy(), want), (w, h, color, dw, dh, "device")
        # planes as slices of one larger allocation (odd offsets and pitches), host and device, with a batch of sizes
        frames = [random_frame(rng, w, h, fmt) for (w, h) in ((641, 481), (33, 17), (1280, 720))]
        want = [oracle_draw(oracle_convert(yo, f, fmt, COLORS[i]), 320, 240) for i, f in enumerate(frames)]
        host, dev = [], []
        for f in frames:
            buf, where = carve(f, rng)
            tb = T.from_numpy(buf).cuda()
            host.append(tuple(buf[r:r + s[0], o:o + s[1]] for r, o, s in where))
            dev.append(tuple(tb[r:r + s[0], o:o + s[1]] for r, o, s in where))
            assert all(p.strides[0] % 2 == 1 for p in host[-1])
        colors = list(COLORS[:3])
        assert np.array_equal(c.ingest_yuv(host, 320, 240, fmt, colors), np.stack(want))
        out = T.zeros((3, 240, 320, 4), dtype=T.uint8, device="cuda")
        c.ingest_yuv(dev, 320, 240, fmt, colors, out=out)
        assert np.array_equal(out.cpu().numpy(), np.stack(want))
        out_host = T.zeros((3, 240, 320, 4), dtype=T.uint8)
        c.ingest_yuv(dev, 320, 240, fmt, colors, out=out_host)           # device planes, host destination
        assert np.array_equal(out_host.numpy(), np.stack(want))
        before = c.launch_count
        c.ingest_yuv(dev, 320, 240, fmt, colors, out=out)
        assert c.launch_count - before == 1
    finally:
        c.close()


# ---- composition with the RGBA path: the golden replays -------------------------------------------------------------

def yuv_pair(yo, rgba, k, device):
    """(the YUV video of stream k made from rgba, hto_yuv_to_rgba of it) - host or device"""
    fmt, color = stream_format(k), stream_color(k)
    y = forward(rgba, fmt)
    if k % 3 == 1:                                         # row-padded planes
        y = tuple(padded_plane(p, 3 + i) for i, p in enumerate(y))
    r = oracle_convert(yo, y, fmt, color)
    if device:
        T = torch()
        return on_device(y), T.from_numpy(r).cuda()
    return y, r


@pytest.mark.parametrize("mode", ["host", "device", "alternate"])
def test_golden_cases_yuv_tick_equals_rgba_tick_of_the_converted_video(yo, mode):
    """every stream of test_gpu_canvases' replay (lifecycle, main and params cases, with their parameters and
    canvases), each call a seeded random subset in shuffled order: ht_tracker_feed_yuv on one context equals
    ht_tracker_feed_canvases on the converted video on another, record for record.  alternate: the YUV context's
    streams take YUV and RGBA ticks in turn (two calls per tick)."""
    n = len(STREAMS)
    params = [s[0]["params"] if isinstance(s[0], dict) else {} for s in STREAMS]
    canvases = [canvas_of(s[0]) if isinstance(s[0], dict) else s[1] for s in STREAMS]
    specs = [spec_of(s[0]) if isinstance(s[0], dict) else (None, 1000.0) for s in STREAMS]
    device = mode != "host"
    rng = np.random.default_rng(29)
    cy = Context(max_width=200, max_height=160, max_frames=32)
    cr = Context(max_width=200, max_height=160, max_frames=32)
    try:
        ty, tr = TrackerSet(cy, n, params), TrackerSet(cr, n, params)
        pos = [0] * n
        offset = [1.0e12 + 7919.0 * k for k in range(n)]
        seen = set()

        def finished(k):
            return not isinstance(STREAMS[k][0], dict) or pos[k] - STREAMS[k][1] >= len(specs[k][0])

        call = 0
        while not all(finished(k) for k in range(n)) or call < 12:
            chosen = [k for k in range(n) if rng.random() < 0.6] or [int(rng.integers(n))]
            rng.shuffle(chosen)
            listed, yv, rv, clocks = [], {}, {}, {}
            for k in chosen:
                s, first = STREAMS[k]
                f = black(*canvases[k])
                if s == "black" and pos[k] == 0:
                    ty.start(k), tr.start(k)
                j = pos[k] - first if isinstance(s, dict) else -1
                if isinstance(s, dict) and 0 <= j < len(specs[k][0]):
                    action, kind, tt = specs[k][0][j]
                    if action == "start":
                        ty.start(k), tr.start(k)
                    if action == "stop":
                        ty.stop(k), tr.stop(k)
                        continue
                    f = make_frame(s, kind, tt)
                listed.append(k)
                clocks[k] = offset[k] + specs[k][1] * (pos[k] + 1)
                yv[k], rv[k] = yuv_pair(yo, video(f, 1 + k % 3, False), k, device)
            if listed:
                if device:
                    torch().cuda.synchronize()         # the library runs on its own stream
                cw = {k: canvases[k][0] for k in listed}
                chh = {k: canvases[k][1] for k in listed}
                fmts = {k: stream_format(k) for k in listed}
                cols = {k: stream_color(k) for k in listed}
                want = tr.feed(rv, now_ms=clocks, width=cw, height=chh)
                if mode == "alternate":
                    ys = [k for k in listed if (k + call) % 2 == 0]
                    got = {}
                    if ys:
                        got.update(ty.feed_yuv({k: yv[k] for k in ys}, {k: clocks[k] for k in ys}, cw, chh, fmts, cols))
                    rs = [k for k in listed if k not in ys]
                    if rs:
                        got.update(ty.feed({k: rv[k] for k in rs}, {k: clocks[k] for k in rs}, cw, chh))
                else:
                    got = ty.feed_yuv(yv, now_ms=clocks, width=cw, height=chh, format=fmts, color=cols)
                for k in listed:
                    assert equal_records(got[k], want[k]), (mode, call, k, got[k], want[k])
                    assert ty.status[k] == tr.status[k], (mode, call, k)
                    seen.add(want[k]["detection"])
            for k in chosen:
                s, first = STREAMS[k]
                if isinstance(s, dict) and pos[k] - first == len(specs[k][0]) - 1:
                    ty.stop(k), tr.stop(k)                   # the case's closing stop()
                pos[k] += 1
            call += 1
            assert call < 2000
        assert {"WB", "VJ", "CS"} <= seen, seen
    finally:
        cy.close()
        cr.close()


def test_debug_cases_yuv_tick_equals_rgba_tick_with_debug_canvases(yo):
    """reference_js_debug's cases, every stream with its debug canvas: records and debug canvases agree after every tick"""
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    W0, H0 = GOLD_D["width"], GOLD_D["height"]
    cy = Context(max_width=W0, max_height=H0, max_frames=8)
    cr = Context(max_width=W0, max_height=H0, max_frames=8)
    try:
        dy = [T.from_numpy(debug_canvas(case)).cuda() for case in cases]
        dr = [d.clone() for d in dy]
        ty = TrackerSet(cy, n, [dict(case["params"], debug=dy[k]) for k, case in enumerate(cases)])
        tr = TrackerSet(cr, n, [dict(case["params"], debug=dr[k]) for k, case in enumerate(cases)])
        T.cuda.synchronize()
        clock, cs = 1.0e12, 0
        for i in range(max(len(case["steps"]) for case in cases)):
            clock += 35.0
            listed, yv, rv = [], {}, {}
            for k, case in enumerate(cases):
                f = black(W0, H0)
                if i < len(case["steps"]):
                    s = case["steps"][i]
                    f = frame_debug(*s["frame"])
                    if s["action"] == "start":
                        ty.start(k), tr.start(k)
                    elif s["action"] == "stop":
                        ty.stop(k), tr.stop(k)
                    if s["action"] != "stop":
                        listed.append(k)
                elif i == len(case["steps"]):
                    ty.stop(k), tr.stop(k)
                yv[k], rv[k] = yuv_pair(yo, video(f, 1 + k % 3, False), k, True)
            if not listed:
                continue
            T.cuda.synchronize()
            got = ty.feed_yuv({k: yv[k] for k in listed}, clock, W0, H0, {k: stream_format(k) for k in listed},
                              {k: stream_color(k) for k in listed})
            want = tr.feed({k: rv[k] for k in listed}, clock, W0, H0)
            assert equal_records(got, want), i
            cs += sum(want[k]["detection"] == "CS" for k in listed)
            for k in range(n):
                assert T.equal(dy[k], dr[k]), (i, k)
        assert cs > 0
    finally:
        cy.close()
        cr.close()


# ---- at scale -------------------------------------------------------------------------------------------------------

def test_1024_streams_of_1280x720_nv12_device_video(yo):
    T = torch()
    N = 1024
    distinct = 8
    rgba = [synth.frame(700 + i, 1280, 720, n_faces=1) for i in range(distinct)]
    nv12 = [forward(f, "nv12") for f in rgba]
    conv = [oracle_convert(yo, f, "nv12", "bt601") for f in nv12]
    yv = [on_device(f) for f in nv12]
    rv = [T.from_numpy(f).cuda() for f in conv]
    T.cuda.synchronize()
    cy = Context(max_width=320, max_height=320, max_frames=N)
    cr = Context(max_width=320, max_height=320, max_frames=N)
    rng = np.random.default_rng(41)
    try:
        for x in (cy, cr):
            x.tracker_config(calcAngles=True)
            x.tracker_reset(0, N)
            x.tracker_start(0, N)
        modes = set()
        mix = [(320, 240), (200, 150), (160, 120), (240, 320)]
        for tick in range(24):
            ks = list(range(N)) if tick < 12 else sorted(rng.choice(N, N - 100, replace=False).tolist())
            rng.shuffle(ks)
            if tick < 12:
                w, h = 320, 240
            else:
                w = [mix[(k + tick) % 4][0] for k in ks]
                h = [mix[(k + tick) % 4][1] for k in ks]
            now = 1.0e12 + 35.0 * tick
            oy = T.empty(len(ks) * 144, dtype=T.uint8, device="cuda")
            orr = T.empty(len(ks) * 144, dtype=T.uint8, device="cuda")
            cy.tracker_feed_yuv(ks, [yv[k % distinct] for k in ks], now, w, h, out=oy)
            cr.tracker_feed(ks, [rv[k % distinct] for k in ks], now, w, h, out=orr)
            cy.sync(), cr.sync()
            a, b = oy.cpu().numpy(), orr.cpu().numpy()
            assert np.array_equal(a, b), tick
            modes |= {r["detection"] for r in tracker_events_from_bytes(a.tobytes())}
        assert {"WB", "VJ", "CS"} <= modes, modes
    finally:
        cy.close()
        cr.close()


def test_launches_equal_an_rgba_tick_of_the_same_layout(yo):
    T = torch()
    f = synth.frame(11, 320, 240, n_faces=1)
    y = on_device(forward(f, "nv12"))
    r = T.from_numpy(oracle_convert(yo, forward(f, "nv12"), "nv12", "bt601")).cuda()
    T.cuda.synchronize()
    cy = Context(max_width=320, max_height=240, max_frames=4)
    cr = Context(max_width=320, max_height=240, max_frames=4)
    try:
        for x in (cy, cr):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        for t in range(30):
            ks = [3, 0, 2] if t % 3 else [1, 2, 0, 3]
            w, h = (320, 240) if t % 2 else ([320, 160, 200, 160][:len(ks)], [240, 120, 150, 120][:len(ks)])
            ly, lr = cy.launch_count, cr.launch_count
            a = cy.tracker_feed_yuv(ks, [y] * len(ks), 1.0e12 + 35.0 * t, w, h)
            b = cr.tracker_feed(ks, [r] * len(ks), 1.0e12 + 35.0 * t, w, h)
            assert equal_records(a, b), t
            assert cy.launch_count - ly == cr.launch_count - lr > 0, t
    finally:
        cy.close()
        cr.close()


# ---- rejections -----------------------------------------------------------------------------------------------------

def test_rejections_name_the_record_and_change_nothing():
    T = torch()
    MAXF = 4
    rng = np.random.default_rng(5)
    f = random_frame(rng, 320, 240, "nv12")
    g = random_frame(rng, 320, 240, "i420")
    fd = on_device(f)
    T.cuda.synchronize()

    def img(frame=f, fmt=0, color=0, w=320, h=240, pitch=(0, 0, 0), third=None):
        ptrs = [p.ctypes.data if isinstance(p, np.ndarray) else p.data_ptr() for p in frame] + [None] * (3 - len(frame))
        if third is not None:
            ptrs[2] = third
        return _lib.YuvImage((C.c_void_p * 3)(*ptrs), (C.c_int32 * 3)(*pitch), w, h, fmt, color)

    def rec(stream, image=None, cw=160, ch=120):
        return _lib.YuvFrame(image if image is not None else img(), stream, cw, ch, 0, 1.0e12)

    def raw(c, recs, on_dev):
        arr = (_lib.YuvFrame * len(recs))(*recs)
        out = (_lib.TrackerEvent * len(recs))()
        return c._L.ht_tracker_feed_yuv(c._h, C.addressof(arr), len(recs), on_dev, C.addressof(out))

    nulled = img()
    nulled.planes[1] = None
    i420_no_v = img(g, fmt=1)
    i420_no_v.planes[2] = None
    y_null = img()
    y_null.planes[0] = None
    cases = [
        (HT_ERR_ARG, [rec(0), rec(1, img(fmt=2))], 0, 1),                       # bad format
        (HT_ERR_ARG, [rec(0, img(color=4))], 0, 0),                             # bad colour
        (HT_ERR_ARG, [rec(0), rec(1, img(color=-1))], 0, 1),
        (HT_ERR_ARG, [rec(0), rec(1), rec(2, nulled)], 0, 2),                   # a missing plane
        (HT_ERR_ARG, [rec(0, i420_no_v)], 0, 0),
        (HT_ERR_ARG, [rec(0), rec(1, y_null)], 0, 1),
        (HT_ERR_ARG, [rec(0, img(third=g[2].ctypes.data))], 0, 0),              # planes[2] for NV12
        (HT_ERR_ARG, [rec(0), rec(1, img(pitch=(319, 0, 0)))], 0, 1),           # short pitches
        (HT_ERR_ARG, [rec(0), rec(1, img(pitch=(0, 319, 0)))], 0, 1),
        (HT_ERR_ARG, [rec(0, img(g, fmt=1, pitch=(0, 160, 159)))], 0, 0),
        (HT_ERR_SIZE, [rec(0), rec(1, img(w=0))], 0, 1),                        # sizes outside 1..16384
        (HT_ERR_SIZE, [rec(0, img(h=16385))], 0, 0),
        (HT_ERR_ARG, [rec(0), rec(0)], 0, 1),                                   # a stream listed twice
        (HT_ERR_ARG, [rec(0), rec(1)], 1, None),                                # host planes, frames_on_device = 1
        (HT_ERR_ARG, [rec(0, img(fd)), rec(1, img(fd))], 0, None),              # device planes, frames_on_device = 0
        (HT_ERR_SIZE, [rec(0), rec(1, cw=20, ch=20)], 0, 1),                    # too small for the pyramid
        (HT_ERR_SIZE, [rec(0), rec(1, cw=321, ch=120)], 0, 1),                  # above max_width
        (HT_ERR_SIZE, [rec(0), rec(1, cw=0, ch=120)], 0, 1),
    ]
    c = Context(max_width=320, max_height=240, max_frames=MAXF)
    try:
        c.tracker_config(calcAngles=True)
        c.tracker_reset(0, MAXF)
        c.tracker_start(0, MAXF)
        v = on_device(forward(synth.frame(9, 320, 240, n_faces=1), "nv12"))
        T.cuda.synchronize()
        for t in range(12):                                   # into tracking, so that the records hold real state
            c.tracker_feed_yuv(list(range(MAXF)), [v] * MAXF, 1.0e12 + 35.0 * t, 160, 120)
        before = c.tracker_export(list(range(MAXF)))
        launches = c.launch_count
        for i, (code, recs, on_dev, idx) in enumerate(cases):
            rc = raw(c, recs, on_dev)
            msg = c._L.ht_last_error(c._h).decode()
            assert rc == code, (i, rc, msg)
            if idx is not None:
                assert msg.startswith(f"record {idx}:"), (i, msg)
        assert c.launch_count == launches
        assert np.array_equal(c.tracker_export(list(range(MAXF))), before)
        assert raw(c, [rec(2, img(fd)), rec(0, img(fd))], 1) == HT_OK         # and the context still works
        # ht_ingest_yuv checks the same records
        out = np.zeros((1, 120, 160, 4), np.uint8)
        arr = (_lib.YuvImage * 1)(img(fmt=2))
        assert c._L.ht_ingest_yuv(c._h, C.addressof(arr), 1, 0, out.ctypes.data, 160, 120) == HT_ERR_ARG
        arr = (_lib.YuvImage * 1)(img())
        assert c._L.ht_ingest_yuv(c._h, C.addressof(arr), 1, 1, out.ctypes.data, 160, 120) == HT_ERR_ARG
        assert c._L.ht_ingest_yuv(c._h, C.addressof(arr), 1, 0, out.ctypes.data, 0, 120) == HT_ERR_SIZE
        assert c._L.ht_ingest_yuv(c._h, C.addressof(arr), 1, 0, out.ctypes.data + 1, 160, 120) == HT_ERR_ARG
        assert not out.any()
    finally:
        c.close()
