"""GPU: face tensors (ht_tracker_set_face_tensor, Context.tracker_set_face_tensor / face_tensor_batch): a stream's
face as a model's normalised input is, bit for bit, the conversion (tests/crop_tensor_oracle.c) of the RGBA crop of its
size and scale the same tick makes (DESIGN.md 2, "Face crops", item 6):

  * every case of reference_js_debug.json through step, feed, feed_yuv (NV12, P010, BGR24) and feed through views,
    each stream with an RGBA crop and a tensor of the same size and scale (four dtypes, both layouts, three channel
    modes, padded strides, carved out of one sentinel buffer): records byte-identical to a twin without tensors, crops
    equal to the twin's, every tensor the conversion of that tick's crop, every other byte untouched;
  * an NV12 crop and a tensor on one stream, each the conversion of the twin's RGBA crop;
  * face_tensor_batch over 1024 streams of 1280x720 NV12, a seeded sample checked, with streams.face_written of the
    device records equal to the slots the tick wrote;
  * face_tensor_batch's fill complete before the next tick, with torch's stream busy and the library on its own;
  * the lifetime (a lost and refound face included), the launch count (one k_face_crop for crops, tensors or both) and every rejection."""
import ctypes as C

import numpy as np
import pytest

from headtrackr_b200 import Context, _lib, streams, synth
from headtrackr_b200._lib import HT_ERR_ARG, HT_ERR_SIZE, HT_ERR_STATE
from headtrackr_b200.context import tensor_affine, tracker_events_from_bytes
from headtrackr_b200.streams import TrackerSet
from test_debug_host import GOLD_D, make_frame
from test_face_crop_yuv_host import COLORS, yo  # noqa: F401  (fixture: the YUV restatement)
from test_face_tensor_host import CHANNELS, DTYPES, ESIZE, LAYOUTS, SENTINEL, affine_for, to  # noqa: F401
from test_gpu_debug import black, run
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


def tdtype(d):
    T = torch()
    return {"u8": T.uint8, "f16": T.float16, "bf16": T.bfloat16, "f32": T.float32}[d]


class Tensors:
    """face tensors (dtype, layout, channels, Sw, Sh, scale, pad_row, pad_plane) carved out of one sentinel byte buffer,
    with gaps between them, and the tight RGBA crops of the same sizes"""

    def __init__(self, specs):
        T = torch()
        self.specs, self.place, at = specs, [], 64
        for k, (d, l, c, Sw, Sh, _, pr, pp) in enumerate(specs):
            n, es = (1 if c == "gray" else 3), ESIZE[d]
            if l == "chw":
                row = Sw + pr
                plane = (Sh - 1) * row + Sw + pp if n == 3 else 0
                elems = (n - 1) * plane + (Sh - 1) * row + Sw
            else:
                row, plane = n * Sw + pr, 0
                elems = (Sh - 1) * row + n * Sw
            at = (at + 3) // 4 * 4 + 4 * (k % 3)
            self.place.append((at, row, plane, elems))
            at += elems * es + 1 + k % 5
        self.buf = T.full((at + 64,), SENTINEL, dtype=T.uint8, device="cuda")
        self.out = []
        for (d, l, c, Sw, Sh, _, _, _), (off, row, plane, elems) in zip(specs, self.place):
            es, n = ESIZE[d], 1 if c == "gray" else 3
            flat = self.buf[off:off + elems * es].view(tdtype(d))
            shape, stride = ((n, Sh, Sw), (plane if n == 3 else Sh * row, row, 1)) if l == "chw" else \
                ((Sh, Sw, n), (row, n, 1))
            self.out.append(T.as_strided(flat, shape, stride))
        self.rgba = [T.zeros((Sh, Sw, 4), dtype=T.uint8, device="cuda") for _, _, _, Sw, Sh, _, _, _ in specs]

    def affine(self, k):
        d, _, c = self.specs[k][:3]
        return affine_for(d, c, k)

    def tensor(self, k):
        d, l, c, _, _, scale, _, _ = self.specs[k]
        mul, add = self.affine(k)
        return {"out": self.out[k], "layout": l, "channels": c, "mul": mul, "add": add, "scale": scale}

    def crop(self, k):
        return {"out": self.rgba[k], "scale": self.specs[k][5]}

    def expect(self, to, exp, k, rgba):  # noqa: F811
        """exp (host copy of buf) with tensor k set to the restatement's conversion of the RGBA crop `rgba`"""
        d, l, c, Sw, Sh, _, _, _ = self.specs[k]
        off, row, plane, _ = self.place[k]
        mul, add = self.affine(k)
        rgba = np.ascontiguousarray(rgba)
        to.hcto_convert(rgba.ctypes.data, Sw, Sh, 4 * Sw, DTYPES[d], LAYOUTS[l], CHANNELS[c], (C.c_float * 3)(*mul),
                        (C.c_float * 3)(*add), exp.ctypes.data + off, row, plane)


def wrote(rec):
    return rec["detection"] == "CS" and rec["width"] > 0 and rec["height"] > 0


SPECS = [("f16", "chw", "rgb", 112, 112, 1.0, 0, 0), ("f32", "hwc", "bgr", 64, 96, 1.5, 3, 0),
         ("bf16", "chw", "gray", 48, 48, 0.75, 5, 0), ("u8", "hwc", "rgb", 100, 60, 2.0, 0, 0),
         ("f32", "chw", "bgr", 34, 18, 1.0, 2, 7), ("f16", "hwc", "gray", 1, 1, 1.0, 0, 0),
         ("bf16", "chw", "rgb", 57, 33, 1.25, 1, 3), ("u8", "chw", "gray", 20, 30, 1.0, 4, 0)]


@pytest.mark.parametrize("path", ["step", "feed", "nv12", "p010", "bgr24", "views"])
def test_golden_replay_against_twin_without_tensors(to, path):  # noqa: F811
    T = torch()
    cases = GOLD_D["cases"]
    n = len(cases)
    ts_ = Tensors([SPECS[k % len(SPECS)] for k in range(n)])
    twin = [T.zeros_like(r) for r in ts_.rgba]
    c = Context(max_width=W0, max_height=H0, max_frames=8)
    ref = Context(max_width=W0, max_height=H0, max_frames=8)
    rng = np.random.default_rng(23)
    try:
        ts = TrackerSet(c, n, [dict(case["params"], faceCrop=ts_.crop(k), faceTensor=ts_.tensor(k))
                               for k, case in enumerate(cases)])
        tr = TrackerSet(ref, n, [dict(case["params"], faceCrop={"out": twin[k], "scale": SPECS[k % len(SPECS)][5]})
                                 for k, case in enumerate(cases)])
        T.cuda.synchronize()
        exp = host(ts_.buf).copy()
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
                    ts_.expect(to, exp, k, host(ts_.rgba[k]))
                    written += 1
            assert np.array_equal(host(ts_.buf), exp), i
            assert all(T.equal(a, b) for a, b in zip(ts_.rgba, twin)), i
        assert written > 40 and (host(ts_.buf) == SENTINEL).any()
    finally:
        c.close()
        ref.close()


def test_nv12_crop_and_tensor_on_one_stream(yo, to):  # noqa: F811
    """stream 0 has an NV12 crop and an fp16 CHW tensor, stream 1 a tensor only; the twin has RGBA crops"""
    T = torch()
    ts_ = Tensors([("f16", "chw", "rgb", 48, 40, 1.25, 0, 0), ("f32", "hwc", "bgr", 30, 30, 1.0, 2, 0)])
    y, uv = T.zeros((40, 48), dtype=T.uint8, device="cuda"), T.zeros((20, 48), dtype=T.uint8, device="cuda")
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    ref = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        for x in (ctx, ref):
            x.tracker_config()
            x.tracker_reset(0, 2)
            x.tracker_start(0, 2)
        ctx.tracker_set_face_crop(0, [{"out": (y, uv), "format": "nv12", "color": "bt709", "scale": 1.25}])
        ctx.tracker_set_face_tensor(0, [ts_.tensor(0), ts_.tensor(1)])
        ref.tracker_set_face_crop(0, [ts_.crop(0), ts_.crop(1)])
        exp = host(ts_.buf).copy()
        written = 0
        for t in range(30):
            recs = run(ctx, 1, t)
            assert equal_records(recs, run(ref, 1, t)), t
            T.cuda.synchronize()
            for k in range(2):
                if wrote(recs[k]):
                    ts_.expect(to, exp, k, host(ts_.rgba[k]))
                    written += 1
            if wrote(recs[0]):
                rgba = np.ascontiguousarray(host(ts_.rgba[0]))
                ey, euv = np.zeros((40, 48), np.uint8), np.zeros((20, 48), np.uint8)
                yo.hcyo_convert(_lib.YUV_COLORS["bt709"], 1, rgba.ctypes.data, 48, 40, 4 * 48, ey.ctypes.data, 48,
                                euv.ctypes.data, 48, None, 0)
                assert np.array_equal(host(y), ey) and np.array_equal(host(uv), euv), t
            assert np.array_equal(host(ts_.buf), exp), t
        assert written > 20
    finally:
        ctx.close()
        ref.close()


def test_face_tensor_batch_1024_streams_of_1280x720_nv12(to):  # noqa: F811
    T = torch()
    n, W, H, CW, CH, S = 1024, 1280, 720, 320, 240, 112
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    rng = np.random.default_rng(41)
    bframes = [from_rgba(synth.frame(900 + i, W, H, n_faces=1), "nv12", rng) for i in range(8)]
    dframes = [api_frame(b, True) for b in bframes]
    twin = T.zeros((n, S, S, 4), dtype=T.uint8, device="cuda")
    # the library runs on torch's current stream, so the NaN fill, the tick and face_written's ops are in stream order
    s, prev = T.cuda.Stream(), T.cuda.current_stream()
    T.cuda.set_stream(s)
    ctx = Context(max_width=CW, max_height=CH, max_frames=n, stream=s.cuda_stream)
    ref = Context(max_width=CW, max_height=CH, max_frames=n)
    try:
        for x in (ctx, ref):
            x.tracker_config()
            x.tracker_reset(0, n)
            x.tracker_start(0, n)
        batch = ctx.face_tensor_batch(0, n, S, S, T.float16, "chw", "rgb", mean, std, scale=1.25)
        ref.tracker_set_face_crop(0, [{"out": twin[k], "scale": 1.25} for k in range(n)])
        mul, add = tensor_affine(T.float16, "rgb", mean, std)
        black = np.zeros((S, S, 4), np.uint8)
        want_black = np.zeros((3, S, S), np.uint16)
        to.hcto_convert(black.ctypes.data, S, S, 4 * S, DTYPES["f16"], LAYOUTS["chw"], CHANNELS["rgb"], (C.c_float * 3)(*mul),
                        (C.c_float * 3)(*add), want_black.ctypes.data, S, S * S)
        assert batch.shape == (n, 3, S, S) and batch.dtype == T.float16
        assert (host(batch.view(T.int16)).astype(np.uint16) == want_black).all()   # slots without a face read as black
        sample = sorted(int(k) for k in rng.choice(n, 40, replace=False))
        nan = T.tensor(0x7e00, dtype=T.int16, device="cuda")       # a NaN the conversion never makes
        clock = [1.0e12 + 13.0 * k for k in range(n)]
        written = 0
        for tick in range(30):
            ks = [k for k in range(n) if rng.random() < 0.9]
            rng.shuffle(ks)
            for k in ks:
                clock[k] += 35.0
            batch.view(T.int16).fill_(nan)
            out = T.empty(len(ks) * 144, dtype=T.uint8, device="cuda")
            args = (ks, [dframes[k % 8] for k in ks], [clock[k] for k in ks], CW, CH)
            ctx.tracker_feed_yuv(*args, format="nv12", out=out)
            refs = ref.tracker_feed_yuv(*args, format="nv12")
            mask = streams.face_written(out)
            T.cuda.synchronize()
            assert mask.is_cuda and mask.dtype == T.bool
            recs = tracker_events_from_bytes(host(out).tobytes())
            assert equal_records(recs, refs), tick
            assert np.array_equal(host(mask), streams.face_written(recs))
            assert np.array_equal(host(mask), streams.face_written(host(out)))
            touched = (batch.view(T.int16) != nan).flatten(1).any(1)
            full = (batch.view(T.int16) != nan).flatten(1).all(1)
            want = np.zeros(n, bool)
            want[np.array(ks)[host(mask)]] = True
            assert np.array_equal(host(touched), want) and np.array_equal(host(full), want), tick
            for k, rec in zip(ks, recs):
                if k in sample and wrote(rec):
                    e = np.zeros((3, S, S), np.uint16)
                    rgba = np.ascontiguousarray(host(twin[k]))
                    to.hcto_convert(rgba.ctypes.data, S, S, 4 * S, DTYPES["f16"], LAYOUTS["chw"], CHANNELS["rgb"],
                                    (C.c_float * 3)(*mul), (C.c_float * 3)(*add), e.ctypes.data, S, S * S)
                    assert np.array_equal(host(batch[k].view(T.int16)).astype(np.uint16), e), (tick, k)
                    written += 1
        assert written > 300
    finally:
        ctx.close()
        ref.close()
        T.cuda.set_stream(prev)


def test_face_tensor_batch_is_filled_before_the_next_tick(to):  # noqa: F811
    """the library on its own stream and torch's stream busy when face_tensor_batch fills the batch: the fill has
    landed when it returns, so the next tick's faces are not blackened by it"""
    T = torch()
    S = 40
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        rgba = T.zeros((2, S, S, 4), dtype=T.uint8, device="cuda")
        ctx.tracker_set_face_crop(0, [{"out": rgba[k], "scale": 1.1} for k in range(2)])
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]
        T.cuda.synchronize()
        with T.cuda.stream(T.cuda.Stream()):              # a torch stream of its own, as a model's would be,
            T.cuda._sleep(int(5e8))                        # busy for a while
            batch = ctx.face_tensor_batch(0, 2, S, S, T.float32, "hwc", "bgr", (0.4, 0.5, 0.6), (0.2, 0.3, 0.25), 1.1)
        recs = run(ctx, 1, 22)
        T.cuda.synchronize()
        mul, add = tensor_affine(T.float32, "bgr", (0.4, 0.5, 0.6), (0.2, 0.3, 0.25))
        for k in range(2):
            assert wrote(recs[k])
            e = np.zeros((S, S, 3), np.float32)
            crop = np.ascontiguousarray(host(rgba[k]))
            to.hcto_convert(crop.ctypes.data, S, S, 4 * S, DTYPES["f32"], LAYOUTS["hwc"], CHANNELS["bgr"],
                            (C.c_float * 3)(*mul), (C.c_float * 3)(*add), e.ctypes.data, 3 * S, 0)
            assert np.array_equal(host(batch[k]).view(np.uint32), e.view(np.uint32)), k
    finally:
        ctx.close()


# ---- lifetime, launches, rejections -----------------------------------------------------------------------------------

def test_lifetime_and_independence_from_crops():
    T = torch()
    ctx = Context(max_width=W0, max_height=H0, max_frames=2)
    try:
        ctx.tracker_config()
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        t = T.zeros((3, 40, 40), dtype=T.float32, device="cuda")
        rgba = T.zeros((40, 40, 4), dtype=T.uint8, device="cuda")
        spec = {"out": t, "mean": 0.5, "std": 0.25, "scale": 1.2}
        ctx.tracker_set_face_tensor(0, [spec])
        assert [r["detection"] for r in run(ctx, 22, 0)] == ["CS", "CS"]

        def cut(k):
            """one CS tick on a NaN-filled tensor; -> whether the tensor was written"""
            t.fill_(float("nan"))
            T.cuda.synchronize()
            recs = run(ctx, 1, k)
            T.cuda.synchronize()
            assert recs[0]["detection"] == "CS" and recs[0]["width"] > 0
            return bool(not t.isnan().any())

        assert cut(30)
        ctx.tracker_set_params(0, [dict(calcAngles=True)])
        assert cut(31)                                       # set_params keeps it
        snap = ctx.tracker_export([0])
        ctx.tracker_stop(0, 1)
        ctx.tracker_reset(0, 1)
        ctx.tracker_start(0, 1)
        ctx.tracker_import([0], snap)
        assert cut(32)                                       # stop / reset / start / import keep it
        ctx.tracker_set_face_crop(0, [{"out": rgba, "scale": 1.2}])
        assert cut(33) and (rgba > 0).any()                  # a crop beside it: both written
        ctx.tracker_set_face_crop(0, [None])                 # removing the crop keeps the tensor
        assert cut(34)
        ctx.tracker_set_face_tensor(0, [None])               # None removes it
        assert not cut(35)
        ctx.tracker_set_face_crop(0, [{"out": rgba}])        # and a crop setter does not bring it back
        assert not cut(36)
        ctx.tracker_set_face_tensor(0, [spec])
        assert cut(37)
        import make_goldens_params as pg
        clock = [38]

        def tick(kind):
            """one tick of stream 0 on a NaN-filled tensor: written exactly when the record keeps a face"""
            t.fill_(float("nan"))
            T.cuda.synchronize()
            n = clock[0]
            clock[0] += 1
            rec = ctx.tracker_feed([0], [pg.make_frame(kind, n, W0, H0)], 1.0e12 + 35.0 * n, W0, H0)[0]
            T.cuda.synchronize()
            assert bool(not t.isnan().any()) == wrote(rec) and (wrote(rec) or bool(t.isnan().all())), n
            return rec
        seen = []                                            # a lost face (redetecting, as retryDetection has it)
        while not {"redetecting", "lost"} & set(seen) and clock[0] < 120:
            seen += tick("empty")["status"]
        assert {"redetecting", "lost"} & set(seen), seen
        refound = False                                      # then the face again: the tensor outlived the loss
        while not refound and clock[0] < 200:
            refound = wrote(tick("face"))
        assert refound
        ctx.tracker_config()                                 # removes every tensor
        ctx.tracker_reset(0, 2)
        ctx.tracker_start(0, 2)
        run(ctx, 22, 310)                                    # the frames of ticks 40.. (their jitter repeats every 15)
        assert not cut(332)
    finally:
        ctx.close()


def test_launch_count_one_kernel_for_crops_tensors_or_both():
    T = torch()
    ctxs = [Context(max_width=W0, max_height=H0, max_frames=4) for _ in range(4)]
    try:
        for x in ctxs:
            x.tracker_config()
            x.tracker_reset(0, 4)
            x.tracker_start(0, 4)
        none, crop, tensor, both = ctxs
        rgba = [T.zeros((32, 32, 4), dtype=T.uint8, device="cuda") for _ in range(2)]
        tens = [T.zeros((3, 64, 64), dtype=T.float16, device="cuda") for _ in range(2)]
        for t in range(40):
            if t == 10:
                crop.tracker_set_face_crop(3, [{"out": rgba[0]}])
                tensor.tracker_set_face_tensor(2, [{"out": tens[0]}])
                both.tracker_set_face_crop(1, [{"out": rgba[1]}])
                both.tracker_set_face_tensor(0, [{"out": tens[1]}])
            if t == 25:
                crop.tracker_set_face_crop(3, [None])
                tensor.tracker_set_face_tensor(2, [None])
                both.tracker_set_face_crop(1, [None])
                both.tracker_set_face_tensor(0, [None])
            before = [x.launch_count for x in ctxs]
            recs = [run(x, 1, t, 4) for x in ctxs]
            assert all(equal_records(recs[0], r) for r in recs[1:])
            d = [x.launch_count - n0 for x, n0 in zip(ctxs, before)]
            assert d[1] == d[2] == d[3] == d[0] + (1 if 10 <= t < 25 else 0), t
        T.cuda.synchronize()
        assert all((x > 0).any() for x in rgba) and all(x.abs().sum() > 0 for x in tens)
    finally:
        for x in ctxs:
            x.close()


def set_raw(c, first, tensors, n=None):
    arr = (_lib.FaceTensor * max(1, len(tensors)))(*tensors)
    return c._L.ht_tracker_set_face_tensor(c._h, first, len(tensors) if n is None else n, C.addressof(arr))


def tr_(data, w=20, h=20, dtype=1, layout=0, channels=0, row=None, plane=None, pad=0, mul=(1.0,) * 3, add=(0.0,) * 3,
        scale=1.0):
    n = 1 if channels == 2 else 3
    row = (w if layout == 0 else n * w) if row is None else row
    plane = ((h - 1) * row + w if layout == 0 and n == 3 else 0) if plane is None else plane
    return _lib.FaceTensor(data, row, plane, w, h, dtype, layout, channels, pad, (C.c_float * 3)(*mul),
                           (C.c_float * 3)(*add), scale)


def test_rejections_leave_the_settings_in_force():
    T = torch()
    mf = 3
    c = Context(max_width=W0, max_height=H0, max_frames=mf)
    try:
        buf = T.zeros((3, 16384), dtype=T.uint8, device="cuda")
        p = [buf[k].data_ptr() for k in range(3)]
        ok = [tr_(p[k]) for k in range(3)]                       # f16 CHW RGB 20 x 20: 2400 bytes
        assert set_raw(c, 0, ok[:1]) == HT_ERR_STATE
        c.tracker_config()
        c.tracker_reset(0, mf)
        c.tracker_start(0, mf)
        assert set_raw(c, 0, ok) == 0
        hostbuf = (C.c_uint8 * 8192)()
        q = p[0]
        inf = float("inf")
        bad = [(HT_ERR_ARG, -1, ok[:1], None), (HT_ERR_ARG, 0, ok[:1], 0), (HT_ERR_ARG, 2, ok[:2], None),
               (HT_ERR_ARG, 0, [tr_(q, dtype=4)], None), (HT_ERR_ARG, 0, [tr_(q, dtype=-1)], None),
               (HT_ERR_ARG, 0, [tr_(q, layout=2)], None), (HT_ERR_ARG, 0, [tr_(q, channels=3)], None),
               (HT_ERR_SIZE, 0, [tr_(q, w=0)], None), (HT_ERR_SIZE, 0, [tr_(q, h=2049)], None),
               (HT_ERR_ARG, 0, [tr_(q + 1)], None),                                      # f16 not 2-byte aligned
               (HT_ERR_ARG, 0, [tr_(q + 2, dtype=3)], None),                             # f32 not 4-byte aligned
               (HT_ERR_ARG, 0, [tr_(C.addressof(hostbuf))], None),                       # host memory
               (HT_ERR_ARG, 0, [tr_(q, row=19)], None),                                  # row below S_w
               (HT_ERR_ARG, 0, [tr_(q, layout=1, row=59)], None),                        # HWC row below 3 S_w
               (HT_ERR_ARG, 0, [tr_(q, row=1 << 41)], None),
               (HT_ERR_ARG, 0, [tr_(q, plane=399)], None),                               # plane below the plane
               (HT_ERR_ARG, 0, [tr_(q, layout=1, plane=1200)], None),                    # HWC plane must be 0
               (HT_ERR_ARG, 0, [tr_(q, channels=2, plane=400)], None),                   # gray plane must be 0
               (HT_ERR_ARG, 0, [tr_(q, pad=1)], None),
               (HT_ERR_ARG, 0, [tr_(q, mul=(inf, 1.0, 1.0))], None),
               (HT_ERR_ARG, 0, [tr_(q, add=(0.0, 0.0, float("nan")))], None),
               (HT_ERR_ARG, 0, [tr_(q, dtype=0, mul=(0.5, 1.0, 1.0))], None),            # U8 takes mul 1
               (HT_ERR_ARG, 0, [tr_(q, dtype=0, add=(0.0, 1.0, 0.0))], None),            # and add 0
               (HT_ERR_ARG, 0, [tr_(q, scale=0.0)], None), (HT_ERR_ARG, 0, [tr_(q, scale=16.5)], None),
               (HT_ERR_ARG, 0, [tr_(q, scale=float("nan"))], None),
               (HT_ERR_ARG, 0, [ok[0], tr_(p[0] + 2000)], None),                          # on stream 0's tensor
               (HT_ERR_ARG, 1, [tr_(p[2] + 64, dtype=3)], None)]                          # on stream 2's
        for code, first, ts, n in bad:
            assert set_raw(c, first, ts, n) == code, (first, n, c.last_warning)
        assert c._L.ht_tracker_set_face_tensor(c._h, 0, 1, None) == HT_ERR_ARG
        assert set_raw(c, 0, [tr_(q, dtype=0, channels=2, mul=(1.0, 7.0, 7.0), add=(0.0, 3.0, 3.0))]) == 0  # unused
        assert set_raw(c, 0, ok[:1]) == 0
        # per-plane spans: streams' planes interleaved like a (3, S, H, W) batch are accepted
        il = [tr_(p[2] + 800 * k, plane=2400) for k in range(3)]
        assert set_raw(c, 0, il) == 0
        assert set_raw(c, 0, ok) == 0
        crop = _lib.FaceCrop(p[1] + 4, 4, 4, 0, 0, 1.0)                                            # RGBA on stream 1's
        assert c._L.ht_tracker_set_face_crop(c._h, 2, 1, C.addressof((_lib.FaceCrop * 1)(crop))) == HT_ERR_ARG
        yuv = _lib.FaceCropYuv((C.c_void_p * 3)(p[1] + 900, p[2] + 8000, None), (C.c_int32 * 3)(), 4, 4, 0, 0, 0, 1.0)
        assert c._L.ht_tracker_set_face_crop_yuv(c._h, 2, 1, C.addressof((_lib.FaceCropYuv * 1)(yuv))) == HT_ERR_ARG
        dc = (_lib.DebugCanvas * 1)(_lib.DebugCanvas(p[1] + 1700, 4, 4, 0, 0))
        assert c._L.ht_tracker_set_debug(c._h, 1, 1, C.addressof(dc)) == HT_ERR_ARG                # a canvas on a tensor
        d = T.zeros((H0, W0, 4), dtype=T.uint8, device="cuda")
        c.tracker_set_debug(0, [d])
        assert set_raw(c, 1, [tr_(d.data_ptr() + 4096)]) == HT_ERR_ARG                           # a tensor on a canvas
        r = T.zeros((8, 8, 4), dtype=T.uint8, device="cuda")
        c.tracker_set_face_crop(2, [{"out": r}])
        assert set_raw(c, 1, [tr_(r.data_ptr() + 64, w=2, h=2)]) == HT_ERR_ARG                    # a tensor on a crop
        c.tracker_set_face_crop(2, [None])
        for bad_py in (dict(out=T.zeros((3, 8, 8), dtype=T.int32, device="cuda")),
                       dict(out=T.zeros((8, 8, 3), dtype=T.float16, device="cuda")),                # HWC shape, CHW layout
                       dict(out=T.zeros((3, 8, 8), dtype=T.float16, device="cuda"), channels="gray"),
                       dict(out=T.zeros((3, 8, 8), dtype=T.uint8, device="cuda"), mean=0.5, std=0.5),
                       dict(out=T.zeros((3, 8, 8), dtype=T.float16, device="cuda"), mean=0.5, mul=1.0),
                       dict(out=T.zeros((3, 8, 8), dtype=T.float16, device="cuda"), layout="nchw")):
            with pytest.raises((ValueError, _lib.HtError)):
                c.tracker_set_face_tensor(0, [bad_py])
        T.cuda.synchronize()
        run(c, 24, 0, mf)
        T.cuda.synchronize()
        assert all((buf[k][:2400] > 0).any() for k in range(3))                                   # still in force
    finally:
        c.close()
