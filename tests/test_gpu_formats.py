"""GPU: every ht_yuv_image format and colour into the tracker (ht_tracker_feed_yuv) and onto canvases (ht_ingest_yuv).

  * ht_ingest_yuv equals hto_draw_image(format_oracle(frame)) bit for bit for every format and colour, 1:1 and scaled,
    host and device planes (also slices of one larger allocation at odd offsets and pitches, even ones for P010), host
    and device destinations, and one call mixing every format and size;
  * composition: the golden replays of test_gpu_yuv.py with every stream on its own format and colour (every format,
    with NV12 / I420 and BT.2020), also with streams that change format from tick to tick, against a twin context fed
    the RGBA8 frames the conversion makes: records and debug canvases equal on every tick;
  * 1024 streams of 1280x720 device video spread over the new formats, on one canvas size and on four;
  * a tick of any format mix launches what an RGBA tick of the same layout launches;
  * every new rejection names its record, launches nothing and leaves every stream as it was."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_OK
from headtrackr_b200.context import tracker_events_from_bytes
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, debug_canvas
from test_debug_host import make_frame as frame_debug
from test_formats_host import NEW, RGB, YUV_COLORS, fo, oracle_convert, plane_shapes, random_frame  # noqa: F401
from test_gpu_canvases import STREAMS, black, canvas_of, make_frame, spec_of
from test_gpu_feed import equal_records, video
from test_yuv_host import oracle_draw

pytestmark = pytest.mark.gpu

ALL = NEW + ["nv12", "i420"]


def torch():
    import torch as t
    return t


def colors_of(fmt):
    return ["bt601"] if fmt in RGB else YUV_COLORS


def api_frame(bframe, device):
    """a byte frame of test_formats_host (fmt, w, h, byte planes) as Context takes it: planes (P010: uint16 views) or
    one packed (h, w, c) array, on the host or the device, row strides kept"""
    T = torch() if device else None
    fmt, w, h, planes = bframe

    def move(p):                      # a strided view of a buffer: the buffer goes to the device, the view is re-taken
        if not device:
            return p
        base = np.lib.stride_tricks.as_strided(p, shape=(p.shape[0], p.strides[0]), strides=(p.strides[0], 1))
        return T.from_numpy(np.ascontiguousarray(base)).cuda()[:, :p.shape[1]]
    if fmt in RGB or fmt in ("yuyv", "uyvy"):
        c = {"bgra": 4, "bgr24": 3, "rgb24": 3}.get(fmt, 2)
        p = move(planes[0])
        return p.as_strided((h, w, c), (p.stride(0), c, 1)) if device else \
            np.lib.stride_tricks.as_strided(p, shape=(h, w, c), strides=(p.strides[0], c, 1))
    if fmt == "p010":
        return tuple(move(p).view(T.int16) if device else p.view(np.uint16) for p in planes)
    return tuple(move(p) for p in planes)


def from_rgba(rgba, fmt, rng):
    """a byte frame of `fmt` made from an RGBA frame: the RGB formats by byte order, the YUV ones by a test-local BT.601
    RGB -> YUV (chroma averaged over its block); P010 with random low bits"""
    h, w = rgba.shape[:2]
    cw, ch = (w + 1) // 2, (h + 1) // 2
    if fmt in RGB:
        order = {"bgra": [2, 1, 0, 3], "bgr24": [2, 1, 0], "rgb24": [0, 1, 2]}[fmt]
        return fmt, w, h, (np.ascontiguousarray(rgba[..., order].reshape(h, w * len(order))),)
    rgb = rgba[..., :3].astype(np.float64)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    y = 16 + (65.481 * r + 128.553 * g + 24.966 * b) / 255
    u = 128 + (-37.797 * r - 74.203 * g + 112.0 * b) / 255
    v = 128 + (112.0 * r - 93.786 * g - 18.214 * b) / 255
    q = lambda a: np.clip(np.floor(a + 0.5), 0, 255).astype(np.uint8)     # noqa: E731
    sy = 0 if fmt in ("i444", "i422", "yuyv", "uyvy") else 1
    sx = 0 if fmt == "i444" else 1

    def sub(c):
        c = np.pad(c, ((0, h % 2), (0, w % 2)), mode="edge")
        if sx:
            c = (c[:, 0::2] + c[:, 1::2]) / 2
        if sy:
            c = (c[0::2] + c[1::2]) / 2
        return q(c)
    Y, U, V = q(y), sub(u), sub(v)
    rows, cols = (ch if sy else h), (cw if sx else w)
    U, V = U[:rows, :cols], V[:rows, :cols]
    if fmt in ("i420", "i422", "i444"):
        return fmt, w, h, (Y, np.ascontiguousarray(U), np.ascontiguousarray(V))
    if fmt in ("yuyv", "uyvy"):
        P = np.zeros((h, 4 * cw), np.uint8)
        Yp = np.pad(Y, ((0, 0), (0, 2 * cw - w)))
        yo, uo, vo = (0, 1, 3) if fmt == "yuyv" else (1, 0, 2)
        P[:, yo::2] = Yp
        P[:, uo::4], P[:, vo::4] = U, V
        return fmt, w, h, (P,)
    I = np.empty((ch, 2 * cw), np.uint8)
    first, second = (V, U) if fmt == "nv21" else (U, V)
    I[:, 0::2], I[:, 1::2] = first, second
    if fmt == "p010":
        lift = lambda a: (a.astype(np.uint16) << 8 | rng.integers(0, 128, a.shape, dtype=np.uint16))  # noqa: E731
        return fmt, w, h, tuple(np.ascontiguousarray(lift(a).astype("<u2")).view(np.uint8) for a in (Y, I))
    return fmt, w, h, (Y, I)


# ---- ht_ingest_yuv --------------------------------------------------------------------------------------------------

def carve(bframe, rng):
    """the byte planes of a frame copied into one larger buffer at odd offsets with odd pitches (even ones for P010)"""
    fmt, w, h, planes = bframe
    even = fmt == "p010"
    rows = sum(p.shape[0] for p in planes)
    pitch = max(p.shape[1] for p in planes) + 8
    pitch += (pitch % 2 == 0) != even
    buf = rng.integers(0, 256, (rows + 2, pitch), dtype=np.uint8)
    out, r = [], 1
    for i, p in enumerate(planes):
        off = 2 + 2 * i if even else 1 + 2 * i
        buf[r:r + p.shape[0], off:off + p.shape[1]] = p
        out.append((r, off, p.shape))
        r += p.shape[0]
    return buf, out


@pytest.mark.parametrize("fmt", NEW)
def test_ingest_formats_equal_the_oracle(fo, fmt):
    T = torch()
    rng = np.random.default_rng(len(fmt) + 3)
    c = Context(max_width=1280, max_height=720, max_frames=4)
    try:
        for ci, color in enumerate(colors_of(fmt)):
            for (w, h) in [(1, 1), (3, 5), (33, 17), (641, 481), (1280, 720)][ci % 2::2] + [(64, 48)]:
                f = random_frame(rng, fmt, w, h, extras=(ci, 2 * ci, ci) if fmt != "p010" else (2 * ci,) * 3)
                rgba = oracle_convert(fo, f, color)
                for dw, dh in {(w, h), (160, 120), (33, 17)}:
                    want = oracle_draw(rgba, dw, dh)
                    assert np.array_equal(c.ingest_yuv([api_frame(f, False)], dw, dh, fmt, color)[0], want), (w, h, color)
                    out = T.zeros((1, dh, dw, 4), dtype=T.uint8, device="cuda")
                    c.ingest_yuv([api_frame(f, True)], dw, dh, fmt, color, out=out)
                    c.sync()                                   # a device destination is written on the library's stream
                    assert np.array_equal(out[0].cpu().numpy(), want), (w, h, color, dw, dh, "device")
        # carved out of one allocation at odd offsets and pitches, host and device planes and destinations
        frames = [random_frame(rng, fmt, w, h) for (w, h) in ((641, 481), (33, 17), (1280, 720))]
        colors = [colors_of(fmt)[i % len(colors_of(fmt))] for i in range(3)]
        want = np.stack([oracle_draw(oracle_convert(fo, f, colors[i]), 320, 240) for i, f in enumerate(frames)])
        host, dev = [], []
        for f in frames:
            buf, where = carve(f, rng)
            cf = (f[0], f[1], f[2], tuple(buf[r:r + s[0], o:o + s[1]] for r, o, s in where))
            host.append(api_frame(cf, False))
            dev.append(api_frame(cf, True))
        assert np.array_equal(c.ingest_yuv(host, 320, 240, fmt, colors), want)
        out = T.zeros((3, 240, 320, 4), dtype=T.uint8, device="cuda")
        c.ingest_yuv(dev, 320, 240, fmt, colors, out=out)
        c.sync()
        assert np.array_equal(out.cpu().numpy(), want)
        out_host = T.zeros((3, 240, 320, 4), dtype=T.uint8)
        c.ingest_yuv(dev, 320, 240, fmt, colors, out=out_host)
        assert np.array_equal(out_host.numpy(), want)
    finally:
        c.close()


def test_ingest_one_call_mixes_every_format_and_size(fo):
    T = torch()
    rng = np.random.default_rng(17)
    sizes = [(1280, 720), (641, 481), (320, 240), (33, 17), (160, 120), (7, 3)]
    frames, fmts, colors = [], [], []
    for i, fmt in enumerate(ALL * 2):
        w, h = sizes[i % len(sizes)]
        frames.append(random_frame(rng, fmt, w, h, (i % 3,) * 3 if fmt != "p010" else (2 * (i % 2),) * 3))
        fmts.append(fmt)
        colors.append(colors_of(fmt)[i % len(colors_of(fmt))])
    c = Context(max_width=320, max_height=240, max_frames=4)
    try:
        for dw, dh in ((320, 240), (160, 120)):
            want = np.stack([oracle_draw(oracle_convert(fo, f, colors[i]), dw, dh) for i, f in enumerate(frames)])
            out = T.zeros((len(frames), dh, dw, 4), dtype=T.uint8, device="cuda")
            before = c.launch_count
            c.ingest_yuv([api_frame(f, True) for f in frames], dw, dh, fmts, colors, out=out)
            assert c.launch_count - before == 1
            c.sync()
            assert np.array_equal(out.cpu().numpy(), want)
            assert np.array_equal(c.ingest_yuv([api_frame(f, False) for f in frames], dw, dh, fmts, colors), want)
    finally:
        c.close()


# ---- composition with the RGBA path: the golden replays -------------------------------------------------------------

def stream_format(k, tick, switching):
    return ALL[(k + (tick if switching else 0)) % len(ALL)]


def stream_color(k, fmt):
    cs = colors_of(fmt)
    return cs[k % len(cs)]


def format_pair(fo, rgba, fmt, color, device, rng):
    """(the video of rgba in fmt as Context takes it, format_oracle of it as RGBA8) - host or device"""
    f = from_rgba(rgba, fmt, rng)
    r = oracle_convert(fo, f, color)
    if device:
        return api_frame(f, True), torch().from_numpy(r).cuda()
    return api_frame(f, False), r


@pytest.mark.parametrize("mode", ["host", "device", "switching"])
def test_golden_cases_format_tick_equals_rgba_tick(fo, mode):
    n = len(STREAMS)
    params = [s[0]["params"] if isinstance(s[0], dict) else {} for s in STREAMS]
    canvases = [canvas_of(s[0]) if isinstance(s[0], dict) else s[1] for s in STREAMS]
    specs = [spec_of(s[0]) if isinstance(s[0], dict) else (None, 1000.0) for s in STREAMS]
    device = mode != "host"
    switching = mode == "switching"
    rng = np.random.default_rng(31)
    cy = Context(max_width=200, max_height=160, max_frames=32)
    cr = Context(max_width=200, max_height=160, max_frames=32)
    try:
        ty, tr = TrackerSet(cy, n, params), TrackerSet(cr, n, params)
        pos = [0] * n
        offset = [1.0e12 + 7919.0 * k for k in range(n)]
        seen, used = set(), set()

        def finished(k):
            return not isinstance(STREAMS[k][0], dict) or pos[k] - STREAMS[k][1] >= len(specs[k][0])

        call = 0
        while not all(finished(k) for k in range(n)) or call < 12:
            chosen = [k for k in range(n) if rng.random() < 0.6] or [int(rng.integers(n))]
            rng.shuffle(chosen)
            listed, yv, rv, clocks, fmts, cols = [], {}, {}, {}, {}, {}
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
                fmts[k] = stream_format(k, call, switching)
                cols[k] = stream_color(k, fmts[k])
                used.add((fmts[k], cols[k]))
                yv[k], rv[k] = format_pair(fo, video(f, 1 + k % 3, False), fmts[k], cols[k], device, rng)
            if listed:
                if device:
                    torch().cuda.synchronize()
                cw = {k: canvases[k][0] for k in listed}
                chh = {k: canvases[k][1] for k in listed}
                want = tr.feed(rv, now_ms=clocks, width=cw, height=chh)
                got = ty.feed_yuv(yv, now_ms=clocks, width=cw, height=chh, format=fmts, color=cols)
                for k in listed:
                    assert equal_records(got[k], want[k]), (mode, call, k, fmts[k], got[k], want[k])
                    assert ty.status[k] == tr.status[k], (mode, call, k)
                    seen.add(want[k]["detection"])
            for k in chosen:
                s, first = STREAMS[k]
                if isinstance(s, dict) and pos[k] - first == len(specs[k][0]) - 1:
                    ty.stop(k), tr.stop(k)
                pos[k] += 1
            call += 1
            assert call < 2000
        assert {"WB", "VJ", "CS"} <= seen, seen
        assert {f for f, _ in used} == set(ALL) and any(c.startswith("bt2020") for _, c in used), used
    finally:
        cy.close()
        cr.close()


def test_debug_cases_format_tick_equals_rgba_tick_with_debug_canvases(fo):
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    W0, H0 = GOLD_D["width"], GOLD_D["height"]
    rng = np.random.default_rng(37)
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
            listed, yv, rv, fmts, cols = [], {}, {}, {}, {}
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
                fmts[k] = stream_format(k, i, True)
                cols[k] = stream_color(k, fmts[k])
                yv[k], rv[k] = format_pair(fo, video(f, 1 + k % 3, False), fmts[k], cols[k], True, rng)
            if not listed:
                continue
            T.cuda.synchronize()
            got = ty.feed_yuv({k: yv[k] for k in listed}, clock, W0, H0, {k: fmts[k] for k in listed},
                              {k: cols[k] for k in listed})
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

def test_1024_streams_of_1280x720_device_video_in_every_new_format(fo):
    T = torch()
    N = 1024
    rng = np.random.default_rng(43)
    base = [synth.frame(700 + i, 1280, 720, n_faces=1) for i in range(2)]
    kinds = [(fmt, colors_of(fmt)[i % len(colors_of(fmt))], i % 2) for i, fmt in enumerate(NEW)]
    pairs = [format_pair(fo, base[src], fmt, color, True, rng) for fmt, color, src in kinds]
    T.cuda.synchronize()
    cy = Context(max_width=320, max_height=320, max_frames=N)
    cr = Context(max_width=320, max_height=320, max_frames=N)
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
            sel = [k % len(kinds) for k in ks]
            cy.tracker_feed_yuv(ks, [pairs[i][0] for i in sel], now, w, h, format=[kinds[i][0] for i in sel],
                                color=[kinds[i][1] for i in sel], out=oy)
            cr.tracker_feed(ks, [pairs[i][1] for i in sel], now, w, h, out=orr)
            cy.sync(), cr.sync()
            a, b = oy.cpu().numpy(), orr.cpu().numpy()
            assert np.array_equal(a, b), tick
            modes |= {r["detection"] for r in tracker_events_from_bytes(a.tobytes())}
        assert {"WB", "VJ", "CS"} <= modes, modes
    finally:
        cy.close()
        cr.close()


def test_launches_equal_an_rgba_tick_of_the_same_layout(fo):
    f = synth.frame(11, 320, 240, n_faces=1)
    rng = np.random.default_rng(47)
    pairs = {fmt: format_pair(fo, f, fmt, colors_of(fmt)[-1], True, rng) for fmt in ALL}
    torch().cuda.synchronize()
    cy = Context(max_width=320, max_height=240, max_frames=4)
    cr = Context(max_width=320, max_height=240, max_frames=4)
    try:
        for x in (cy, cr):
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        for t in range(30):
            ks = [3, 0, 2] if t % 3 else [1, 2, 0, 3]
            fm = [ALL[(t + i) % len(ALL)] for i in range(len(ks))]
            w, h = (320, 240) if t % 2 else ([320, 160, 200, 160][:len(ks)], [240, 120, 150, 120][:len(ks)])
            ly, lr = cy.launch_count, cr.launch_count
            a = cy.tracker_feed_yuv(ks, [pairs[m][0] for m in fm], 1.0e12 + 35.0 * t, w, h, format=fm,
                                    color=[colors_of(m)[-1] for m in fm])
            b = cr.tracker_feed(ks, [pairs[m][1] for m in fm], 1.0e12 + 35.0 * t, w, h)
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
    dev = {fmt: tuple(T.from_numpy(np.ascontiguousarray(p)).cuda() for p in random_frame(rng, fmt, 320, 240)[3])
           for fmt in NEW}
    spare = T.zeros(64, dtype=T.uint8, device="cuda")
    T.cuda.synchronize()

    def img(fmt, color=0, planes=None, pitch=None):
        ps = [p.data_ptr() for p in dev[fmt]] + [None] * (3 - len(dev[fmt]))
        if planes:
            for i, v in planes.items():
                ps[i] = v
        return _lib.YuvImage((C.c_void_p * 3)(*ps), (C.c_int32 * 3)(*(pitch or (0, 0, 0))), 320, 240,
                             _lib.YUV_FORMATS[fmt], color)

    def rec(stream, image):
        return _lib.YuvFrame(image, stream, 160, 120, 0, 1.0e12)

    def raw(c, recs):
        arr = (_lib.YuvFrame * len(recs))(*recs)
        out = (_lib.TrackerEvent * len(recs))()
        return c._L.ht_tracker_feed_yuv(c._h, C.addressof(arr), len(recs), 1, C.addressof(out))

    good = rec(0, img("nv21"))
    bad = []
    for fmt in NEW:
        used = len(dev[fmt])
        bad.append(img(fmt, color=1 if fmt in RGB else 9))                     # colour not valid for the format
        bad.append(img(fmt, planes={0: None}))                                 # a required plane missing
        bad.append(img(fmt, planes={used: spare.data_ptr()}) if used < 3 else img(fmt, planes={2: None}))
        tight = plane_shapes(fmt, 320, 240)[0][1]
        bad.append(img(fmt, pitch=(tight - 1, 0, 0)))                          # a pitch below the tight pitch
    bad += [img("p010", planes={1: dev["p010"][1].data_ptr() + 1}), img("p010", pitch=(641, 0, 0)),
            img("p010", pitch=(0, 641, 0)), img("bgra", color=8), img("i444", color=11), img("nv21", color=4)]
    c = Context(max_width=320, max_height=240, max_frames=MAXF)
    try:
        c.tracker_config(calcAngles=True)
        c.tracker_reset(0, MAXF)
        c.tracker_start(0, MAXF)
        vf = T.from_numpy(from_rgba(synth.frame(9, 320, 240, n_faces=1), "yuyv", rng)[3][0]).cuda().reshape(240, 320, 2)
        T.cuda.synchronize()
        for t in range(12):
            c.tracker_feed_yuv(list(range(MAXF)), [vf] * MAXF, 1.0e12 + 35.0 * t, 160, 120, format="yuyv")
        before = c.tracker_export(list(range(MAXF)))
        launches = c.launch_count
        for i, image in enumerate(bad):
            rc = raw(c, [good, rec(1, image)])
            msg = c._L.ht_last_error(c._h).decode()
            assert rc == HT_ERR_ARG, (i, rc, msg)
            assert msg.startswith("record 1:"), (i, msg)
        assert c.launch_count == launches
        assert np.array_equal(c.tracker_export(list(range(MAXF))), before)
        assert raw(c, [rec(2, img("p010")), good, rec(3, img("bgra"))]) == HT_OK     # the context still ticks
        out = np.zeros((1, 120, 160, 4), np.uint8)
        for image in bad[:4]:
            arr = (_lib.YuvImage * 1)(image)
            assert c._L.ht_ingest_yuv(c._h, C.addressof(arr), 1, 1, out.ctypes.data, 160, 120) == HT_ERR_ARG
        assert not out.any()
    finally:
        c.close()
