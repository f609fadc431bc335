"""CPU: the one overlap rule of the per-stream outputs, against a brute-force restatement.

The streams of a tick run concurrently, so no byte range a tick writes may share a byte with another: each debug
canvas (one span over its rows), each plane of each face crop, each channel plane (CHW) or whole tensor (HWC) of each
face tensor, and each camera (DESIGN.md 2).  ht_selftest_tick_writes resolves ABI records through the setters' own
record functions and returns the verdict of the function every setter calls.  Here every span is restated from the ABI
records, turned into its set of byte addresses, and every pair of spans is intersected.
"""
import ctypes as C
import itertools
import random

import pytest

from headtrackr_b200 import _lib
from test_cascade_host import st  # noqa: F401  (fixture: the host-only build of ht_api.cu)

DEBUG, CROP, TENSOR, CAMERA = range(4)     # the kinds ht_selftest_tick_writes reports
NV12, I420 = 0, 1                          # HT_YUV_NV12, HT_YUV_I420
ES = {_lib.HT_TENSOR_U8: 1, _lib.HT_TENSOR_F16: 2, _lib.HT_TENSOR_BF16: 2, _lib.HT_TENSOR_F32: 4}


def spans(stream):
    """[(kind, start, end)] of one stream's records, restated from the ABI: a span runs from a plane's first byte to
    its last row's last byte"""
    out = []
    d = stream.get("debug")
    if d:
        pitch = d.pitch or 4 * d.width
        out.append((DEBUG, d.rgba, d.rgba + (d.height - 1) * pitch + 4 * d.width))
    c = stream.get("crop")
    if c:
        pitch = c.pitch or 4 * c.width
        out.append((CROP, c.rgba, c.rgba + (c.height - 1) * pitch + 4 * c.width))
    y = stream.get("yuv")
    if y:
        w, h = y.width, y.height
        rows = [(w, h), (w, h // 2)] if y.format == NV12 else [(w, h), (w // 2, h // 2), (w // 2, h // 2)]
        for p, (row, n) in enumerate(rows):
            pitch = y.pitch[p] or row
            out.append((CROP, y.planes[p], y.planes[p] + (n - 1) * pitch + row))
    t = stream.get("tensor")
    if t:
        es = ES[t.dtype]
        ch = 1 if t.channels == _lib.HT_TENSOR_GRAY else 3
        if t.layout == _lib.HT_TENSOR_HWC:
            out.append((TENSOR, t.data, t.data + ((t.height - 1) * t.row_stride + ch * t.width) * es))
        else:
            for k in range(ch):
                a = t.data + k * t.plane_stride * es
                out.append((TENSOR, a, a + ((t.height - 1) * t.row_stride + t.width) * es))
    if stream.get("camera"):
        out.append((CAMERA, stream["camera"], stream["camera"] + _lib.CAMERA_BYTES))
    return out


def brute(streams):
    """every pair of spans that share a byte: [((kind, stream), (kind, stream))]"""
    flat = [(k, s, set(range(a, b))) for s, x in enumerate(streams) for k, a, b in spans(x)]
    return [((k0, s0), (k1, s1)) for (k0, s0, b0), (k1, s1, b1) in itertools.combinations(flat, 2) if b0 & b1]


def verdict(st, streams):
    n = len(streams)
    dbg, crops, yuv = (_lib.DebugCanvas * n)(), (_lib.FaceCrop * n)(), (_lib.FaceCropYuv * n)()
    tensors, cams, clash = (_lib.FaceTensor * n)(), (C.c_void_p * n)(), (C.c_int32 * 4)()
    for s, x in enumerate(streams):
        for arr, key in ((dbg, "debug"), (crops, "crop"), (yuv, "yuv"), (tensors, "tensor")):
            if x.get(key):
                arr[s] = x[key]
        cams[s] = x.get("camera")
    hit = st.ht_selftest_tick_writes(n, dbg, crops, yuv, tensors, cams, clash)
    return hit, ((clash[0], clash[1]), (clash[2], clash[3]))


def check(st, streams):
    """the library's verdict is the brute force's, and a reported pair is one that shares a byte -> the verdict"""
    hit, pair = verdict(st, streams)
    pairs = brute(streams)
    assert hit == (len(pairs) > 0), (hit, pairs)
    if hit:
        assert pair in pairs or pair[::-1] in pairs, (pair, pairs)
    return hit


@pytest.fixture(scope="module")
def tw(st):
    st.ht_selftest_tick_writes.argtypes = [C.c_int] + [C.c_void_p] * 6
    return st


def random_stream(rng, space):
    at = lambda align=1: rng.randrange(64, space, align)   # noqa: E731  (0 would be NULL)
    x = {}
    if rng.random() < 0.5:
        w, h = rng.randint(1, 6), rng.randint(1, 4)
        x["debug"] = _lib.DebugCanvas(at(4), w, h, rng.choice([0, 4 * w + 4 * rng.randint(0, 3)]), 0)
    if rng.random() < 0.3:
        w, h = rng.randint(1, 6), rng.randint(1, 4)
        x["crop"] = _lib.FaceCrop(at(4), w, h, rng.choice([0, 4 * w + 4 * rng.randint(0, 3)]), 0, 1.0)
    elif rng.random() < 0.4:
        w, h, nv12 = 2 * rng.randint(1, 4), 2 * rng.randint(1, 3), rng.random() < 0.5
        rows = (w, w, 0) if nv12 else (w, w // 2, w // 2)
        planes = (at(), at(), None if nv12 else at())
        pitch = tuple(rng.choice([0, r + rng.randint(0, 5)]) if r else 0 for r in rows)
        x["yuv"] = _lib.FaceCropYuv(planes, pitch, w, h, NV12 if nv12 else I420, 0, 0, 1.0)
    if rng.random() < 0.5:
        dtype, hwc, gray = rng.choice(list(ES)), rng.random() < 0.5, rng.random() < 0.3
        w, h = rng.randint(1, 5), rng.randint(1, 4)
        row = (1 if gray else 3) * w if hwc else w
        row_stride = row + rng.randint(0, 4)
        plane = 0 if hwc or gray else (h - 1) * row_stride + w + rng.randint(0, 8)
        x["tensor"] = _lib.FaceTensor(at(ES[dtype]), row_stride, plane, w, h, dtype,
                                      _lib.HT_TENSOR_HWC if hwc else _lib.HT_TENSOR_CHW,
                                      _lib.HT_TENSOR_GRAY if gray else _lib.HT_TENSOR_RGB, 0, (1.0,) * 3, (0.0,) * 3, 1.0)
    if rng.random() < 0.4:
        x["camera"] = at(16)
    return x


def test_random_layouts_equal_the_brute_force(tw):
    rng = random.Random(2026)
    kinds, verdicts = set(), [0, 0]
    for trial in range(3000):
        space = rng.choice([1024, 4096, 16384])
        streams = [random_stream(rng, space) for _ in range(rng.randint(1, 4))]
        verdicts[check(tw, streams)] += 1
        kinds |= {tuple(sorted((a[0], b[0]))) for a, b in brute(streams)}
    assert kinds == set(itertools.combinations_with_replacement(range(4), 2)), kinds   # every pair of kinds clashed
    assert min(verdicts) > 300, verdicts


def test_hand_cases(tw):
    H, W, S = 4, 6, 3
    base = 1 << 20
    # the CHW channel planes of a (3, S, H, W) float16 batch: stream i's planes interleave with the others'
    batch = [{"tensor": _lib.FaceTensor(base + 2 * i * H * W, W, S * H * W, W, H, _lib.HT_TENSOR_F16, _lib.HT_TENSOR_CHW,
                                        _lib.HT_TENSOR_RGB, 0, (1.0,) * 3, (0.0,) * 3, 1.0)} for i in range(S)]
    assert check(tw, batch) == 0
    # the same slices as HWC tensors would cover one another
    hwc = [{"tensor": _lib.FaceTensor(base + 2 * i * H * W, S * 3 * W, 0, W, H, _lib.HT_TENSOR_F16, _lib.HT_TENSOR_HWC,
                                      _lib.HT_TENSOR_RGB, 0, (1.0,) * 3, (0.0,) * 3, 1.0)} for i in range(S)]
    assert check(tw, hwc) == 1
    q = base
    nv12 = lambda uv: _lib.FaceCropYuv((q, uv, None), (0, 0, 0), 20, 20, NV12, 0, 0, 1.0)   # noqa: E731
    i420 = lambda v: _lib.FaceCropYuv((q, q + 400, v), (0, 0, 0), 20, 20, I420, 0, 0, 1.0)  # noqa: E731
    assert check(tw, [{"yuv": nv12(q + 400)}]) == 0
    assert check(tw, [{"yuv": nv12(q + 399)}]) == 1                      # UV on its own Y
    assert verdict(tw, [{"yuv": nv12(q + 399)}])[1] == ((CROP, 0), (CROP, 0))
    assert check(tw, [{"yuv": i420(q + 500)}]) == 0
    assert check(tw, [{"yuv": i420(q + 499)}]) == 1                      # V on U
    # a camera inside a debug canvas, a crop or a tensor of another stream, and just past each
    canvas = _lib.DebugCanvas(base, 64, 4, 0, 0)                          # 1024 bytes
    crop = _lib.FaceCrop(base, 64, 4, 0, 0, 1.0)
    tensor = _lib.FaceTensor(base, 256, 0, 256, 1, _lib.HT_TENSOR_F32, _lib.HT_TENSOR_CHW, _lib.HT_TENSOR_GRAY, 0,
                             (1.0,) * 3, (0.0,) * 3, 1.0)
    for key, rec, kind in (("debug", canvas, DEBUG), ("crop", crop, CROP), ("tensor", tensor, TENSOR)):
        for cam, want in ((base + 512, 1), (base + 1024 - 16, 1), (base - 224, 0), (base - 208, 1), (base + 1024, 0)):
            streams = [{key: rec}, {"camera": cam}]
            assert check(tw, streams) == want, (key, cam - base)
            if want:
                assert sorted(verdict(tw, streams)[1]) == sorted([(kind, 0), (CAMERA, 1)])
    # two cameras of one tick, 224 bytes each
    assert check(tw, [{"camera": base}, {"camera": base + 224}]) == 0
    assert check(tw, [{"camera": base}, {"camera": base + 208}]) == 1
